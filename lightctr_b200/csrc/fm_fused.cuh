// lightctr_b200/csrc/fm_fused.cuh -- order-free FM step kernels (cfg.deterministic == 0), sm_90a.
//
// Reference semantics: Train_FM_Algo::batchGradCompute + accumWVGrad + ApplyGrad (train/train_fm_algo.cpp:63-126).
// The in-order kernels of fm.cu reproduce the reference's arithmetic SEQUENCE (needed for multi-epoch 1e-5 parity);
// these kernels compute the same expressions with shuffle-tree sums (the reference's own multi-threaded Hogwild mode
// is order-free too, SURVEY 8c) and are the throughput path:
//
//   batch layout (built once per batch at upload, depends only on the batch):
//     uniq[U]        the distinct feature ids of the batch ("pull_map" keys, distributed_algo_abst.h:181-190)
//     ent_slot[nnz]  position of each entry's fid in uniq  -> gradients live in a BATCH-COMPACT buffer
//                    G[U][rowlen + 4]  (row = [gV (rowlen) | gW | pad]: one 16 B-aligned record per distinct feature)
//   fm_fused_kernel   warp = sample.  One gather of the sample's V rows (K/4 lanes x 16 B per row, all rows of the
//                     sample in flight, kept in REGISTERS), shuffle-tree sumVX / |Vx|^2 / Wx, sigmoid, loss; the
//                     gradient rows are formed from the register-resident rows and leave as 16 B vector REDs into G.
//                     One gather per step instead of two; no fid-indexed dense update_g; no touched map.
//   apply_compact_kernel  the per-coordinate updater over G: coalesced gradient read, gather/scatter of the U parameter
//                     and state rows, G re-zeroed in the same pass (replaces compact_touched + apply of opt.cu).
// HBM/L2-bound integer + fp32 work: no tensor cores by design.
//
// What bounds the scatter (scripts/lab/fm_lab.cu): fp32 REDs into L2 run at a high rate when the target rows are spread,
// but ops on ONE address serialise -- the hottest id of a Criteo-shaped batch sits in every row, so the pass costs time in
// proportion to the rows however few bytes move (a W-only RED pass takes as long as the full V+W pass).  Hence HOT slots:
// ids whose multiplicity in a sample of the batch predicts >= ~128 occurrences get kHotRep replica rows (Ghot) that the
// warps address round-robin; the updater folds the replicas.  The threshold and kHotRep were tuned on B200s and have not
// been re-measured on H100s.  The same serialisation hits
// plain byte stores, so the mark kernel only writes marks it does not already see set.
#pragma once
#include "opt.cuh"

namespace lctr {

constexpr int kHotSampleRows = 512;
// stride (floats) of a compact gradient row [gV (k) | gW | pad]: power of two >= k + 1 (rows never straddle a 128 B line)
__host__ __device__ constexpr int grad_stride(int k) { return k < 8 ? 8 : (k < 16 ? 16 : (k < 32 ? 32 : 64)); }

__device__ __forceinline__ uint32_t ldg_u32_pinned(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// ---------------------------------------------------------------------------------------------------------------
// slot map of a batch: mark -> compact (+ fid -> slot table) -> assign.  Integer work; runs on the upload stream.
// ---------------------------------------------------------------------------------------------------------------
// Each CTA walks a CONTIGUOUS range of entries and keeps a direct-mapped tag table of the ids it has already marked:
// the hot ids of the small-vocabulary fields recur in every row, and tens of thousands of byte stores (or loads) aimed
// at the same few 128 B lines serialise in one L2 slice; the filter forwards each id once per CTA.
// The mark of id f lives at position (f % 128) * T + f / 128 (T = ceil(F / 128)): ids that are neighbours in value --
// the dense, hot low end of every field's vocabulary -- land T bytes apart, i.e. in different lines and L2 slices.
constexpr int kMarkTags = 2048;
__host__ __device__ inline size_t mark_rows(size_t F) { return (F + 127) / 128; }
__global__ void __launch_bounds__(256)
slotmap_mark_kernel(const uint32_t* __restrict__ fid, const int64_t* __restrict__ hdr, int64_t nnz_arg,
                    uint8_t* __restrict__ mark, size_t T) {
    __shared__ uint32_t tag[kMarkTags];
    const int64_t nnz = hdr ? hdr[1] : nnz_arg;
    for (int i = threadIdx.x; i < kMarkTags; i += blockDim.x) tag[i] = 0xffffffffu;
    __syncthreads();
    const int64_t per = (nnz + gridDim.x - 1) / gridDim.x;
    const int64_t b = (int64_t)blockIdx.x * per, e = min(nnz, b + per);
    for (int64_t i0 = b + threadIdx.x; i0 < e; i0 += 4 * blockDim.x) {  // four index loads in flight per thread
        uint32_t f[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t i = i0 + (int64_t)u * blockDim.x;
            f[u] = i < e ? ldg_u32_pinned(fid + i) : 0xffffffffu;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (f[u] == 0xffffffffu) continue;
            const uint32_t h = f[u] & (kMarkTags - 1);
            if (tag[h] != f[u]) {  // racy inside the CTA, benign: at worst a duplicate store
                tag[h] = f[u];
                mark[(size_t)(f[u] & 127u) * T + (f[u] >> 7)] = 1;
            }
        }
    }
}

// scans the byte map (128 * T positions) 16 marks per lane, clears it, appends the ids of the set positions to `uniq` (one
// warp-aggregated atomicAdd per non-empty 512-position tile) and records slot_of[fid] = slot
__global__ void __launch_bounds__(256)
slotmap_compact_kernel(uint8_t* __restrict__ mark, size_t T, uint32_t* __restrict__ uniq, unsigned int* __restrict__ n_uniq,
                       uint32_t* __restrict__ slot_of) {
    const size_t F = 128 * T;  // positions
    const int lane = threadIdx.x & 31;
    const size_t warp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
    const size_t ntiles = (F + 511) / 512;
    for (size_t tile = warp; tile < ntiles; tile += nwarps) {
        const size_t base = tile * 512 + (size_t)lane * 16;
        uint4 m = make_uint4(0, 0, 0, 0);
        if (base + 16 <= F) {
            m = *reinterpret_cast<const uint4*>(mark + base);
        } else if (base < F) {
            unsigned char tmp[16];
            for (int i = 0; i < 16; i++) tmp[i] = base + i < F ? mark[base + i] : 0;
            m = *reinterpret_cast<uint4*>(tmp);
        }
        const bool any = (m.x | m.y | m.z | m.w) != 0;
        if (!__any_sync(kFull, any)) continue;
        unsigned bits = 0;
        {
            const unsigned wv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int b = 0; b < 4; b++)
                    if ((wv[i] >> (8 * b)) & 0xffu) bits |= 1u << (i * 4 + b);
        }
        if (any) {
            if (base + 16 <= F) *reinterpret_cast<uint4*>(mark + base) = make_uint4(0, 0, 0, 0);
            else for (int i = 0; i < 16 && base + i < F; i++) mark[base + i] = 0;
        }
        const int mycnt = __popc(bits);
        int incl = mycnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += t;
        }
        const int total = __shfl_sync(kFull, incl, 31);
        unsigned int gbase = 0;
        if (lane == 31) gbase = atomicAdd(n_uniq, (unsigned int)total);
        gbase = __shfl_sync(kFull, gbase, 31);
        unsigned int pos = gbase + (unsigned int)(incl - mycnt);
        while (bits) {
            const int bit = __ffs(bits) - 1;
            bits &= bits - 1;
            const size_t ps = base + bit;
            const uint32_t f = (uint32_t)(((ps % T) << 7) | (ps / T));
            uniq[pos] = f;
            if (slot_of) slot_of[f] = pos;
            pos++;
        }
    }
}

// multiplicity estimate: counts the slots of the entries of the first kHotSampleRows rows
__global__ void __launch_bounds__(256)
slotmap_sample_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid, const int64_t* __restrict__ hdr,
                      int64_t rows_arg, const uint32_t* __restrict__ slot_of, unsigned int* __restrict__ cnt) {
    const int64_t rows = hdr ? hdr[0] : rows_arg;
    const int64_t ns = row_ptr[rows < kHotSampleRows ? rows : kHotSampleRows];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(&cnt[slot_of[fid[i]]], 1u);
}

// hot_of[slot] = index of the slot's replica block (or ~0): sampled count >= max(3, 128 * sampled_rows / rows), i.e. an
// expected multiplicity of >= ~128 in the whole batch; clears cnt.  n_hot must be zero on entry.
__global__ void __launch_bounds__(256)
slotmap_hot_kernel(unsigned int* __restrict__ cnt, const unsigned int* __restrict__ n_uniq, const int64_t* __restrict__ hdr,
                   int64_t rows_arg, uint32_t* __restrict__ hot_of, uint32_t* __restrict__ hot_slot,
                   unsigned int* __restrict__ n_hot) {
    const int64_t rows = hdr ? hdr[0] : rows_arg;
    const int64_t srows = rows < kHotSampleRows ? rows : kHotSampleRows;
    const unsigned thr = (unsigned)max((int64_t)3, (128 * srows + rows - 1) / max(rows, (int64_t)1));
    const unsigned n = *n_uniq;
    const int lane = threadIdx.x & 31;
    for (unsigned b0 = (blockIdx.x * blockDim.x + threadIdx.x) - lane; b0 < n; b0 += gridDim.x * blockDim.x) {
        const unsigned i = b0 + lane;
        const bool hot = i < n && cnt[i] >= thr;
        const unsigned m = __ballot_sync(kFull, hot);
        unsigned base = 0;
        if (m && lane == 0) base = atomicAdd(n_hot, (unsigned)__popc(m));
        base = __shfl_sync(kFull, base, 0);
        if (i < n) {
            const unsigned h = base + (unsigned)__popc(m & ((1u << lane) - 1u));
            const bool take = hot && h < (unsigned)kHotMax;
            hot_of[i] = take ? h : 0xffffffffu;
            if (take) hot_slot[h] = i;
            cnt[i] = 0;
        }
    }
}

// ent_slot[i]: the slot of entry i, or kHotBit | replica-block index when the slot is hot
// ent_pslot (optional): always the plain slot -- the row of the entry's parameters in a batch-compact cache (multi-GPU)
__global__ void __launch_bounds__(256)
slotmap_assign_kernel(const uint32_t* __restrict__ fid, const int64_t* __restrict__ hdr, int64_t nnz_arg,
                      const uint32_t* __restrict__ slot_of, const uint32_t* __restrict__ hot_of,
                      uint32_t* __restrict__ ent_slot, uint32_t* __restrict__ ent_pslot) {
    const int64_t nnz = hdr ? hdr[1] : nnz_arg;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t sl = slot_of[fid[i]];
        const uint32_t h = hot_of ? hot_of[sl] : 0xffffffffu;
        if (ent_slot) ent_slot[i] = h != 0xffffffffu ? (kHotBit | h) : sl;
        if (ent_pslot) ent_pslot[i] = sl;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// fused forward (+ RED backward)
// ---------------------------------------------------------------------------------------------------------------
// MODE 0: FM forward only (pred, sumVX, d = pred - label, statistics).  MODE 1: FM forward + RED backward into G / Ghot.
// MODE 2: NFM forward (train_nfm_algo.cpp:78-94): wide part, sumVX and the bi-interaction z = 0.5 (sumVX^2 - sum (xV)^2) for
// the dense layers.  MODE 3: NFM backward (accumWideGrad / accumDeepGrad, :126-159) from the dense layers' input delta dz:
// the rows are gathered again (L2 hits), sumVX comes back from memory, gradients leave as REDs like MODE 1.
// pidx: per-entry index of the PARAMETER row (the fid; or the slot when the rows live in a batch-compact cache),
// gidx: per-entry gradient row: slot, or kHotBit | replica block (slotmap_assign_kernel).  SAME_IDX: pidx == gidx.
//
// Persistent warps: warp w of the grid takes samples w, w + NW, w + 2 NW, ...; the row_ptr pairs of its next 32 samples
// are fetched with one load, and the index loads of sample t+1 are issued before sample t's rows are consumed, so that
// per sample only ONE dependent round trip (the row gather itself) is exposed instead of three (row_ptr -> indices ->
// rows).
// RW: the slot's row weights rw scale the head and the per-occurrence L2 terms of MODE 1 and MODE 3
template <int K, bool HAS_VAL, int MODE, bool SAME_IDX, int MINB = 4, bool RW = false>
__global__ void __launch_bounds__(128, MINB)
fm_fused_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ pidx, const uint32_t* __restrict__ gidx,
                const float* __restrict__ val, const float* __restrict__ label, const float* __restrict__ W,
                const float* __restrict__ V, float* __restrict__ pred, float* __restrict__ sumvx, float* __restrict__ dvec,
                float* __restrict__ G, float* __restrict__ Ghot, int GS, float l2, int64_t rb, int64_t re_arg,
                const int64_t* __restrict__ hdr, double* partial, unsigned int* done, double* out_slot, int do_stats,
                const unsigned long long* wait_flags = nullptr, int n_wait = 0, unsigned long long wait_epoch = 0,
                float* __restrict__ zbuf = nullptr /* MODE 2: z out, MODE 3: dz in; [re - rb][K] */,
                float* __restrict__ wide = nullptr /* MODE 2: wide part out [rows] */,
                const float* __restrict__ rw = nullptr /* RW: [rows] */) {
    constexpr bool FWD = MODE != 3, BWD = MODE == 1 || MODE == 3, NFM = MODE >= 2;
    static_assert(K % 4 == 0 && K <= 32 && (K / 4 & (K / 4 - 1)) == 0, "fused FM step: K in {4, 8, 16, 32}");
    // programmatic dependent launch: a kernel launched behind this one with the serialisation attribute (the compact
    // updater, launch_apply_compact) may start its CTAs as soon as ours retire; it synchronises on our COMPLETION itself
    // (cudaGridDependencySynchronize) before it touches G.  Without the attribute this is a no-op.
    cudaTriggerProgrammaticLaunchCompletion();
    if (wait_flags) {  // multi-GPU: the owners' rows of this step must have landed in the cache (dist.cu)
        if (threadIdx.x < n_wait) {
            const volatile unsigned long long* f = wait_flags + threadIdx.x;
            while (*f < wait_epoch) __nanosleep(40);
            __threadfence();  // the flags and the delivered rows live in this GPU's memory: device scope suffices on the acquire side
        }
        __syncthreads();
    }
    constexpr int LPR = K / 4;                           // lanes per V row (one float4 each)
    constexpr int GR = 32 / LPR;                         // rows per gather instruction
    constexpr int NPASS = K <= 8 ? 8 : (K == 16 ? 4 : 2);  // 32-entry passes whose rows stay in registers
    const int lane = threadIdx.x & 31;
    const int q = lane % LPR, g = lane / LPR;
    const int64_t re = hdr ? hdr[0] : re_arg;
    const int64_t NW = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t gwarp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int rep = (int)(gwarp & (kHotRep - 1));
    double loss = 0.0, correct = 0.0;

    for (int64_t c0 = rb + gwarp; c0 < re; c0 += 32 * NW) {
        // row_ptr pairs of this warp's next (up to) 32 samples: lane l <-> sample c0 + l * NW
        const int64_t myr = c0 + (int64_t)lane * NW;
        long long mb = 0;
        int mn = 0;
        if (myr < re) {
            mb = row_ptr[myr];
            mn = (int)(row_ptr[myr + 1] - mb);
        }
        const int cnt = (int)min((int64_t)32, (re - c0 + NW - 1) / NW);
        uint32_t pf[NPASS], gs[NPASS];
        float xs[NPASS];
        {   // indices of sample 0 of the chunk
            const long long b = __shfl_sync(kFull, mb, 0);
            const int n = __shfl_sync(kFull, mn, 0);
#pragma unroll
            for (int p = 0; p < NPASS; p++) {
                const int i = p * 32 + lane;
                const bool ok = i < n;
                pf[p] = ok ? ldg_u32_pinned(pidx + b + i) : 0u;
                gs[p] = SAME_IDX ? pf[p] : ((ok && BWD) ? ldg_u32_pinned(gidx + b + i) : 0u);
                xs[p] = ok ? (HAS_VAL ? ldg_f32_pinned(val + b + i) : 1.f) : 0.f;
            }
        }
        // launched programmatically dependent (NFM backward behind the dense kernels): everything above is batch data; the
        // parameters, dz and the predictions are read from here on.  A no-op for an ordinary launch.
        cudaGridDependencySynchronize();
        for (int t = 0; t < cnt; t++) {
            const int64_t r = c0 + (int64_t)t * NW;
            const long long b = __shfl_sync(kFull, mb, t);
            const int n = __shfl_sync(kFull, mn, t);
            // ---- every row gather of the sample, back to back
            float4 v[NPASS][LPR];
            float ws[NPASS];
#pragma unroll
            for (int p = 0; p < NPASS; p++) {
                if (p * 32 < n) {  // warp-uniform
                    ws[p] = ldg_f32_pinned(W + pf[p]);  // lane-own W (index 0 beyond n: harmless, x = 0)
#pragma unroll
                    for (int it = 0; it < LPR; it++) {
                        const uint32_t fj = __shfl_sync(kFull, pf[p], it * GR + g);
                        v[p][it] = ldg_f4_pinned(V + (size_t)fj * K + 4 * q);
                    }
                } else {
                    ws[p] = 0.f;
#pragma unroll
                    for (int it = 0; it < LPR; it++) v[p][it] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            // ---- indices of the NEXT sample: in flight while this one is reduced
            uint32_t npf[NPASS], ngs[NPASS];
            float nxs[NPASS];
            {
                const int tn = t + 1 < cnt ? t + 1 : t;
                const long long bn = __shfl_sync(kFull, mb, tn);
                const int nn_raw = __shfl_sync(kFull, mn, tn);
                const int nn = t + 1 < cnt ? nn_raw : 0;
#pragma unroll
                for (int p = 0; p < NPASS; p++) {
                    const int i = p * 32 + lane;
                    const bool ok = i < nn;
                    npf[p] = ok ? ldg_u32_pinned(pidx + bn + i) : 0u;
                    ngs[p] = SAME_IDX ? npf[p] : ((ok && BWD) ? ldg_u32_pinned(gidx + bn + i) : 0u);
                    nxs[p] = ok ? (HAS_VAL ? ldg_f32_pinned(val + bn + i) : 1.f) : 0.f;
                }
            }
            // ---- interaction sums (order-free): s = sum x V (this lane's 4 factors over its rows), sq = sum |xV|^2
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 sqv = make_float4(0.f, 0.f, 0.f, 0.f);  // NFM: per-factor sum (xV)^2
            float sq = 0.f, wsum = 0.f;
            if (FWD) {
#pragma unroll
                for (int p = 0; p < NPASS; p++) {
                    if (p * 32 < n) {
                        wsum = __fmaf_rn(ws[p], HAS_VAL ? xs[p] : (p * 32 + lane < n ? 1.f : 0.f), wsum);  // fm_pred += W[fid] * X   train_fm_algo.cpp:74
#pragma unroll
                        for (int it = 0; it < LPR; it++) {
                            const float xj = HAS_VAL ? __shfl_sync(kFull, xs[p], it * GR + g)
                                                     : (p * 32 + it * GR + g < n ? 1.f : 0.f);  // 0 beyond n
                            const float4 tt = make_float4(v[p][it].x * xj, v[p][it].y * xj, v[p][it].z * xj, v[p][it].w * xj);
                            s.x += tt.x; s.y += tt.y; s.z += tt.z; s.w += tt.w;      // sumVX += tmp            :77
                            if (NFM) {
                                sqv.x = __fmaf_rn(tt.x, tt.x, sqv.x); sqv.y = __fmaf_rn(tt.y, tt.y, sqv.y);
                                sqv.z = __fmaf_rn(tt.z, tt.z, sqv.z); sqv.w = __fmaf_rn(tt.w, tt.w, sqv.w);
                            } else {
                                sq = __fmaf_rn(tt.x, tt.x, sq); sq = __fmaf_rn(tt.y, tt.y, sq);
                                sq = __fmaf_rn(tt.z, tt.z, sq); sq = __fmaf_rn(tt.w, tt.w, sq);  // dot(tmp, tmp)  :78
                            }
                        }
                    }
                }
                for (int base = NPASS * 32; base < n; base += 32) {  // samples longer than the register window
                    const int i = base + lane;
                    const bool ok = i < n;
                    const uint32_t f = ok ? __ldg(pidx + b + i) : 0u;
                    const float x = ok ? (HAS_VAL ? __ldg(val + b + i) : 1.f) : 0.f;
                    wsum = __fmaf_rn(__ldg(W + f), x, wsum);
                    float4 vv[LPR];
#pragma unroll
                    for (int it = 0; it < LPR; it++) {
                        const uint32_t fj = __shfl_sync(kFull, f, it * GR + g);
                        vv[it] = ldg_f4(V + (size_t)fj * K + 4 * q);
                    }
#pragma unroll
                    for (int it = 0; it < LPR; it++) {
                        const float xj = __shfl_sync(kFull, x, it * GR + g);
                        const float4 tt = make_float4(vv[it].x * xj, vv[it].y * xj, vv[it].z * xj, vv[it].w * xj);
                        s.x += tt.x; s.y += tt.y; s.z += tt.z; s.w += tt.w;
                        if (NFM) {
                            sqv.x = __fmaf_rn(tt.x, tt.x, sqv.x); sqv.y = __fmaf_rn(tt.y, tt.y, sqv.y);
                            sqv.z = __fmaf_rn(tt.z, tt.z, sqv.z); sqv.w = __fmaf_rn(tt.w, tt.w, sqv.w);
                        } else {
                            sq = __fmaf_rn(tt.x, tt.x, sq); sq = __fmaf_rn(tt.y, tt.y, sq);
                            sq = __fmaf_rn(tt.z, tt.z, sq); sq = __fmaf_rn(tt.w, tt.w, sq);
                        }
                    }
                }
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {  // over the row groups: every lane ends with the full sumVX of its 4 factors
                    s.x += __shfl_xor_sync(kFull, s.x, o); s.y += __shfl_xor_sync(kFull, s.y, o);
                    s.z += __shfl_xor_sync(kFull, s.z, o); s.w += __shfl_xor_sync(kFull, s.w, o);
                    if (NFM) {
                        sqv.x += __shfl_xor_sync(kFull, sqv.x, o); sqv.y += __shfl_xor_sync(kFull, sqv.y, o);
                        sqv.z += __shfl_xor_sync(kFull, sqv.z, o); sqv.w += __shfl_xor_sync(kFull, sqv.w, o);
                    }
                }
                wsum = warp_sum(wsum);
                if (lane < LPR) *reinterpret_cast<float4*>(sumvx + (size_t)r * K + 4 * q) = s;  // FM_Algo_Abst::sumVX (:145)
            }
            float d = 0.f;
            float4 dz4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!NFM) {
                sq = warp_sum(sq);
                float dot = s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w;  // |sumVX|^2 over the LPR lanes of a row group
#pragma unroll
                for (int o = 1; o < LPR; o <<= 1) dot += __shfl_xor_sync(kFull, dot, o);
                const float fm = wsum - 0.5f * sq + 0.5f * dot;             // :78, :82
                const float pr = ref_sigmoid(fm);                           // :84
                const float y = __ldg(label + r);
                d = row_head<RW>(pr, y, rw, r);                             // LogisticGradW  fm_algo_abst.h:159-161
                if (lane == 0) {
                    pred[r] = pr;
                    if (dvec) dvec[r] = d;
                    if (do_stats) {
                        double l1, c1;
                        loss_terms(pr, y, l1, c1);
                        loss += l1;
                        correct += c1;
                    }
                }
            } else if (MODE == 2) {
                // z = sum -0.5 (xV)^2 + 0.5 sumVX^2 per factor (train_nfm_algo.cpp:87-94); wide part = sum W x (:83)
                if (lane < LPR) {
                    const float4 z4 = make_float4(0.5f * (s.x * s.x - sqv.x), 0.5f * (s.y * s.y - sqv.y),
                                                  0.5f * (s.z * s.z - sqv.z), 0.5f * (s.w * s.w - sqv.w));
                    *reinterpret_cast<float4*>(zbuf + (size_t)(r - rb) * K + 4 * q) = z4;
                }
                if (lane == 0) wide[r] = wsum;
            } else {  // MODE 3
                s = __ldg(reinterpret_cast<const float4*>(sumvx + (size_t)r * K + 4 * q));
                dz4 = __ldg(reinterpret_cast<const float4*>(zbuf + (size_t)(r - rb) * K + 4 * q));
                d = row_head<RW>(__ldg(pred + r), __ldg(label + r), rw, r);
            }
            if (BWD) {
                const float l2r = row_l2<RW>(l2, rw, r);
                // ---- backward from the register-resident rows (train_fm_algo.cpp:101-116; NFM: train_nfm_algo.cpp:126-159),
                // vector REDs into G / Ghot.  FM: gV = (sumVX - xV) gradW + l2 V;  NFM: gV = (sumVX - xV) (dz x) + l2 V
#pragma unroll
                for (int p = 0; p < NPASS; p++) {
                    if (p * 32 < n) {
#pragma unroll
                        for (int it = 0; it < LPR; it++) {
                            const int j = it * GR + g;
                            const float xj = HAS_VAL ? __shfl_sync(kFull, xs[p], j) : 1.f;
                            const float wj = __shfl_sync(kFull, ws[p], j);
                            const uint32_t sj = __shfl_sync(kFull, gs[p], j);
                            if (p * 32 + j < n) {
                                const float gw = __fmaf_rn(d, xj, l2r * wj);                       // :108
                                const float4 vv = v[p][it];
                                const float4 mu = NFM ? make_float4(dz4.x * xj, dz4.y * xj, dz4.z * xj, dz4.w * xj) : make_float4(gw, gw, gw, gw);
                                float4 gv;
                                gv.x = __fmaf_rn(__fmaf_rn(-xj, vv.x, s.x), mu.x, l2r * vv.x);     // :112-115
                                gv.y = __fmaf_rn(__fmaf_rn(-xj, vv.y, s.y), mu.y, l2r * vv.y);
                                gv.z = __fmaf_rn(__fmaf_rn(-xj, vv.z, s.z), mu.z, l2r * vv.z);
                                gv.w = __fmaf_rn(__fmaf_rn(-xj, vv.w, s.w), mu.w, l2r * vv.w);
                                float* dst = (sj & kHotBit) ? Ghot + ((size_t)(sj & ~kHotBit) * kHotRep + rep) * GS
                                                            : G + (size_t)sj * GS;
                                red_add_v4(dst + 4 * q, gv);
                                if (q == 0) red_add_f32(dst + K, gw);                             // :109
                            }
                        }
                    }
                }
                for (int base = NPASS * 32; base < n; base += 32) {
                    const int i = base + lane;
                    const bool ok = i < n;
                    const uint32_t f = ok ? __ldg(pidx + b + i) : 0u;
                    const uint32_t sl = ok ? __ldg(gidx + b + i) : 0u;
                    const float x = ok ? (HAS_VAL ? __ldg(val + b + i) : 1.f) : 0.f;
                    const float w = __ldg(W + f);
#pragma unroll
                    for (int it = 0; it < LPR; it++) {
                        const int j = it * GR + g;
                        const uint32_t fj = __shfl_sync(kFull, f, j);
                        const uint32_t sj = __shfl_sync(kFull, sl, j);
                        const float xj = __shfl_sync(kFull, x, j);
                        const float wj = __shfl_sync(kFull, w, j);
                        if (base + j < n) {
                            const float4 vv = ldg_f4(V + (size_t)fj * K + 4 * q);
                            const float gw = __fmaf_rn(d, xj, l2r * wj);
                            const float4 mu = NFM ? make_float4(dz4.x * xj, dz4.y * xj, dz4.z * xj, dz4.w * xj) : make_float4(gw, gw, gw, gw);
                            float4 gv;
                            gv.x = __fmaf_rn(__fmaf_rn(-xj, vv.x, s.x), mu.x, l2r * vv.x);
                            gv.y = __fmaf_rn(__fmaf_rn(-xj, vv.y, s.y), mu.y, l2r * vv.y);
                            gv.z = __fmaf_rn(__fmaf_rn(-xj, vv.z, s.z), mu.z, l2r * vv.z);
                            gv.w = __fmaf_rn(__fmaf_rn(-xj, vv.w, s.w), mu.w, l2r * vv.w);
                            float* dst = (sj & kHotBit) ? Ghot + ((size_t)(sj & ~kHotBit) * kHotRep + rep) * GS
                                                        : G + (size_t)sj * GS;
                            red_add_v4(dst + 4 * q, gv);
                            if (q == 0) red_add_f32(dst + K, gw);
                        }
                    }
                }
            }
#pragma unroll
            for (int p = 0; p < NPASS; p++) { pf[p] = npf[p]; gs[p] = ngs[p]; xs[p] = nxs[p]; }
        }
    }
    if (do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

// ---------------------------------------------------------------------------------------------------------------
// updater over the batch-compact gradient buffer
// ---------------------------------------------------------------------------------------------------------------
// AdagradUpdater_Num::update / FTRLUpdater::update / AdamUpdater_Num::update ... restricted to the batch's features
// (exactly equivalent to the reference's dense sweep: every updater skips g == 0, SURVEY 8a-7).  Row i of G belongs to
// feature uniq[i]; LPR lanes per row, GR rows per warp step, U steps in flight.  Zeroes G on the way (the memset of
// gradientUpdater.h:149).
template <int K, int OPT>
__global__ void __launch_bounds__(256, 3)
apply_compact_kernel(const uint32_t* __restrict__ uniq, const unsigned int* __restrict__ n_uniq, float* __restrict__ G,
                     const uint32_t* __restrict__ hot_of, const uint32_t* __restrict__ hot_slot,
                     const unsigned int* __restrict__ n_hot, float* __restrict__ Ghot, int GS, int main_blocks,
                     float* __restrict__ W, float* __restrict__ V, float* __restrict__ s1W, float* __restrict__ s1V,
                     float* __restrict__ s2W, float* __restrict__ s2V, OptParams P_in, const OptParams* __restrict__ P_dev) {
    constexpr int LPR = K / 4, GR = 32 / LPR, U = 2;
    OptParams P = P_dev ? *P_dev : P_in;
    P.opt = OPT;
    constexpr bool two = OPT == LCTR_OPT_FTRL || OPT == LCTR_OPT_ADAM || OPT == LCTR_OPT_ADADELTA || OPT == LCTR_OPT_PS_DCASGD ||
                         OPT == LCTR_OPT_PS_DCASGDA;
    const int lane = threadIdx.x & 31;
    // ---- hot slots: the blocks BEYOND main_blocks, one warp per hot slot (the two kinds of work have equally long
    // dependent-load chains, so they run side by side instead of one after the other).  The kHotRep replica rows form a
    // [kHotRep][GS] tile: lane = column, so every load is one fully coalesced row and all rows are requested at once;
    // column c < K is gV[c], column K is gW.  The warp folds, updates and re-zeroes.
    if ((int)blockIdx.x >= main_blocks) {
        const unsigned hwarp = (blockIdx.x - main_blocks) * (blockDim.x >> 5) + (threadIdx.x >> 5);
        const unsigned nhw = (gridDim.x - main_blocks) * (blockDim.x >> 5);
        const unsigned nh = min(*n_hot, (unsigned)kHotMax);
        for (unsigned h = hwarp; h < nh; h += nhw) {
            const uint32_t slot = __ldg(hot_slot + h);
            const uint32_t f = __ldg(uniq + slot);
            float* tile = Ghot + (size_t)h * kHotRep * GS;
#pragma unroll
            for (int c0 = 0; c0 < K + 1; c0 += 32) {  // K = 32: columns 0..31, then column 32
                const int ncol = GS < 32 ? GS : 32;             // columns covered per pass
                const int col = c0 + lane % ncol;
                const int grp = lane / ncol, ngrp = 32 / ncol;  // GS < 32: several replica rows per load
                float wv = 0.f, av = 0.f, bv = 0.f;
                const bool mine = grp == 0 && col <= K;
                const size_t o = col < K ? (size_t)f * K + col : (size_t)f;
                if (mine) {  // parameters and updater state: not written by the gradient kernel, requested before the dependency
                    wv = col < K ? V[o] : W[o];
                    av = col < K ? s1V[o] : s1W[o];
                    if (two) bv = col < K ? s2V[o] : s2W[o];
                }
                cudaGridDependencySynchronize();  // the gradient kernel has completed (returns at once after the first time)
                float t[kHotRep];
#pragma unroll
                for (int i = 0; i < kHotRep; i++)
                    t[i] = (i < kHotRep / ngrp) ? __ldcg(tile + (size_t)(grp + i * ngrp) * GS + col) : 0.f;
                float sum = 0.f;
#pragma unroll
                for (int i = 0; i < kHotRep; i++) {
                    sum += t[i];
                    if (i < kHotRep / ngrp) tile[(size_t)(grp + i * ngrp) * GS + col] = 0.f;
                }
                for (int o2 = ncol; o2 < 32; o2 <<= 1) sum += __shfl_xor_sync(kFull, sum, o2);
                if (mine) {  // (every entry of a hot slot carries kHotBit, so its ordinary row G[slot] stays zero)
                    update_one(P, col < K ? P.corrV : P.corrW, wv, sum, av, bv);
                    if (col < K) { V[o] = wv; s1V[o] = av; if (two) s2V[o] = bv; }
                    else { W[o] = wv; s1W[o] = av; if (two) s2W[o] = bv; }
                }
            }
        }
        cudaGridDependencySynchronize();
        return;
    }
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = (unsigned)main_blocks * (blockDim.x >> 5);
    // ---- ordinary slots
    const int q = lane % LPR, g = lane / LPR;
    const unsigned total = *n_uniq;
    for (unsigned b0 = warp * (GR * U); b0 < total; b0 += nwarps * (GR * U)) {
        uint32_t f[U];
        bool ok[U];
        float4 g4[U], v4[U], a4[U], b4[U];
        float gw[U], w[U], a[U], bb[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const unsigned idx = b0 + u * GR + g;
            ok[u] = idx < total && !(hot_of && __ldg(hot_of + idx) != 0xffffffffu);
            f[u] = ok[u] ? __ldg(uniq + idx) : 0u;
            g4[u] = v4[u] = a4[u] = b4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            gw[u] = w[u] = a[u] = bb[u] = 0.f;
            if (ok[u]) {  // parameters and state first: the gradient kernel does not write them
                const size_t o = (size_t)f[u] * K + 4 * q;
                v4[u] = *reinterpret_cast<const float4*>(V + o);
                a4[u] = *reinterpret_cast<const float4*>(s1V + o);
                if (two) b4[u] = *reinterpret_cast<const float4*>(s2V + o);
                if (q == 0) {
                    w[u] = W[f[u]]; a[u] = s1W[f[u]];
                    if (two) bb[u] = s2W[f[u]];
                }
            }
        }
        cudaGridDependencySynchronize();  // G is complete from here on (immediate after the first iteration)
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (ok[u]) {
                const float* grow = G + (size_t)(b0 + u * GR + g) * GS;
                g4[u] = *reinterpret_cast<const float4*>(grow + 4 * q);
                if (q == 0) gw[u] = grow[K];
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (!ok[u]) continue;
            const unsigned idx = b0 + u * GR + g;
            float* grow = G + (size_t)idx * GS;
            const size_t o = (size_t)f[u] * K + 4 * q;
            update_one(P, P.corrV, v4[u].x, g4[u].x, a4[u].x, b4[u].x);
            update_one(P, P.corrV, v4[u].y, g4[u].y, a4[u].y, b4[u].y);
            update_one(P, P.corrV, v4[u].z, g4[u].z, a4[u].z, b4[u].z);
            update_one(P, P.corrV, v4[u].w, g4[u].w, a4[u].w, b4[u].w);
            *reinterpret_cast<float4*>(V + o) = v4[u];
            *reinterpret_cast<float4*>(s1V + o) = a4[u];
            if (two) *reinterpret_cast<float4*>(s2V + o) = b4[u];
            *reinterpret_cast<float4*>(grow + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q == 0) {
                update_one(P, P.corrW, w[u], gw[u], a[u], bb[u]);
                W[f[u]] = w[u]; s1W[f[u]] = a[u];
                if (two) s2W[f[u]] = bb[u];
                grow[K] = 0.f;
            }
        }
    }
    cudaGridDependencySynchronize();
}

}  // namespace lctr
