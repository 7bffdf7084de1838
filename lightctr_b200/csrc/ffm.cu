// lightctr_b200/csrc/ffm.cu -- field-aware FM forward + backward fused per sample, sm_90a.
//
// Reference semantics: Train_FFM_Algo::batchGradCompute / accumWVGrad (train/train_ffm_algo.cpp:51-118):
//     pred   = sum_i W[f_i] x_i + sum_{i<j} <V[f_i, fld_j], V[f_j, fld_i]> x_i x_j
//     gV[f_i, fld_j] += x_i x_j d V[f_j, fld_i] + l2 V[f_i, fld_j]      (and symmetric), d = p - y,
//     one l2 term PER PAIR (quirk, SURVEY 8a-9); whole row skipped when d == 0 (:81-83).
// The reference walks all n(n-1)/2 pairs.  Here the pair sum is factored through per-sample
// field-pair sums  T[a][b] = sum_{j in field b} x_j R_j[a]   (R_j = the Fc*k-float row of f_j,
// [a] = its k-slice for field a):
//     sum_{i<j} ... = 1/2 ( sum_{a,b} <T[a][b], T[b][a]>  -  sum_i x_i^2 |R_i[fld_i]|^2 )
//     gV[f_i][b]   = d x_i ( T[fld_i][b] - [b == fld_i] x_i R_i[fld_i] ) + l2 c_{i,b} R_i[b],
//                    c_{i,b} = #(features of the sample in field b) - [b == fld_i]
// which is algebraically identical (same terms, re-associated) and costs O(n Fc k) instead of
// O(n^2 k) per sample.  Each embedding row is read as ONE contiguous Fc*k*4-byte segment
// (624 B at Fc=39,k=4), fully coalesced across the CTA; T lives in shared memory with
// thread-owned slots (no shared atomics); gradients leave as 16 B vector REDs that are
// contiguous per row.  HBM-bound by the row gather: no tensor cores by design.
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace lctr {

template <int VEC>
struct VT {
    float a[VEC];
};
template <int VEC>
__device__ __forceinline__ VT<VEC> vload(const float* p) {
    VT<VEC> r;
    if (VEC == 4) { float4 t = ldg_f4(p); r.a[0] = t.x; r.a[1 % VEC] = t.y; r.a[2 % VEC] = t.z; r.a[3 % VEC] = t.w; }
    else if (VEC == 2) { float2 t = __ldg(reinterpret_cast<const float2*>(p)); r.a[0] = t.x; r.a[1 % VEC] = t.y; }
    else r.a[0] = __ldg(p);
    return r;
}
template <int VEC>
__device__ __forceinline__ void vred(float* p, const VT<VEC>& v) {
    if (VEC == 4) red_add_v4(p, make_float4(v.a[0], v.a[1 % VEC], v.a[2 % VEC], v.a[3 % VEC]));
    else {
#pragma unroll
        for (int c = 0; c < VEC; c++) red_add_f32(p + c, v.a[c]);
    }
}

constexpr int FFM_UNROLL = 4;      // gradient phase: entries per group
constexpr int FFM_GATHER_U = 16;   // forward gather: rows in flight per CTA
constexpr int kFfmStage = 256;     // entries staged in shared memory per chunk

// TMA bulk reduce-add of a contiguous fp32 segment from shared to global memory (one request per embedding row
// instead of Fc*k/4 vector REDs): cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32
__device__ __forceinline__ void bulk_reduce_add_f32(float* gdst, const float* ssrc, uint32_t bytes) {
    const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                 :: "l"(gdst), "r"(saddr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One CTA per sample; thread t < A owns slot t (VEC floats of the row; A = Fc*k/VEC).
// GROUPED (with TRAIN): the gradient phase is replaced by storing the sample's field-pair tile T (as [a][b][k], so that
// {T[a][b]}_b -- what an entry of field a needs -- is one contiguous row) and its per-field counts; the feature-grouped
// backward of ffm_grouped.cu consumes them.
template <int VEC, bool HAS_VAL, bool TRAIN, bool BULK, bool GROUPED = false>
__global__ void ffm_fused_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                                 const uint16_t* __restrict__ field, const float* __restrict__ val,
                                 const float* __restrict__ label, const float* __restrict__ W,
                                 const float* __restrict__ V, int Fc, int k, float* __restrict__ pred,
                                 float* __restrict__ gW, float* __restrict__ gV, uint8_t* __restrict__ touched,
                                 float l2, int64_t rb, double* partial, unsigned int* done, double* out_slot,
                                 int do_stats, float* __restrict__ Tbuf, uint16_t* __restrict__ cntbuf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int A = Fc * k / VEC;   // slots per row
    const int PPF = k / VEC;      // slots (parts) per field
    VT<VEC>* S = reinterpret_cast<VT<VEC>*>(smem_raw);                       // S[col b][slot a] = T[a][b]
    int* cnt = reinterpret_cast<int*>(smem_raw + (size_t)Fc * A * VEC * 4);  // features per field
    float* red = reinterpret_cast<float*>(cnt + Fc);                         // [3][32] block reduction scratch + bcast
    uint32_t* st_f = reinterpret_cast<uint32_t*>(red + 80);                  // staged entries of the sample
    float* st_x = reinterpret_cast<float*>(st_f + kFfmStage);
    uint16_t* st_fl = reinterpret_cast<uint16_t*>(st_x + kFfmStage);
    // BULK: FFM_UNROLL staging rows (A slots each, 16 B aligned) for the TMA reduce of the gradient rows
    VT<VEC>* stage = reinterpret_cast<VT<VEC>*>(smem_raw + (((size_t)Fc * A * VEC * 4 + (size_t)Fc * 4 + 80 * 4 + (size_t)kFfmStage * 10 + 15) / 16) * 16);
    const int t = threadIdx.x;
    const int64_t r = rb + blockIdx.x;
    const int64_t b0 = row_ptr[r], e0 = row_ptr[r + 1];
    const size_t rowlen = (size_t)Fc * k;
    const bool own = t < A;
    const int my_field = own ? t / PPF : -1, my_part = own ? t % PPF : 0;

    for (int i = t; i < Fc * A; i += blockDim.x) {
#pragma unroll
        for (int c = 0; c < VEC; c++) S[i].a[c] = 0.f;
    }
    for (int i = t; i < Fc; i += blockDim.x) cnt[i] = 0;
    __syncthreads();

    // ---- phase 1: gather rows, accumulate T, wide sum, diagonal ---------------------------------
    // The sample's (fid, field, x) triples are staged in shared memory with one coalesced load per kFfmStage entries, so
    // that the row gathers of FFM_GATHER_U entries can be issued back to back (FFM_GATHER_U * Fc*k*4 bytes in flight per
    // CTA) instead of waiting on a dependent index load per group.
    float wsum = 0.f, dsq = 0.f;
    for (int64_t c0 = b0; c0 < e0; c0 += kFfmStage) {
        const int nst = (int)min((int64_t)kFfmStage, e0 - c0);
        __syncthreads();  // previous chunk fully consumed
        for (int i = t; i < nst; i += blockDim.x) {
            st_f[i] = __ldg(fid + c0 + i);
            st_fl[i] = __ldg(field + c0 + i);
            st_x[i] = HAS_VAL ? __ldg(val + c0 + i) : 1.f;
        }
        __syncthreads();
        for (int i = 0; i < nst; i += FFM_GATHER_U) {
            VT<VEC> v[FFM_GATHER_U];
            float wv[FFM_GATHER_U];
#pragma unroll
            for (int u = 0; u < FFM_GATHER_U; u++) {
                const bool ok = i + u < nst;
                if (ok && own) v[u] = vload<VEC>(V + (size_t)st_f[i + u] * rowlen + (size_t)t * VEC);
                else {
#pragma unroll
                    for (int c = 0; c < VEC; c++) v[u].a[c] = 0.f;
                }
                wv[u] = (ok && t == 0) ? __ldg(W + st_f[i + u]) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < FFM_GATHER_U; u++) {
                if (i + u >= nst) break;
                const int flu = st_fl[i + u];
                const float xu = st_x[i + u];
                if (own) {
                    VT<VEC>& dst = S[flu * A + t];
#pragma unroll
                    for (int c = 0; c < VEC; c++) {
                        const float tv = v[u].a[c] * xu;
                        dst.a[c] += tv;
                        if (my_field == flu) dsq += tv * tv;
                    }
                }
                if (t == 0) {
                    wsum += wv[u] * xu;  // fm_pred += W[fid] * X  (train_ffm_algo.cpp:60)
                    cnt[flu] += 1;
                }
            }
        }
    }
    __syncthreads();

    // ---- phase 2: P = sum_{a,b} <T[a][b], T[b][a]> ------------------------------------------------
    float P = 0.f;
    if (own) {
        for (int b = 0; b < Fc; b++) {
            if (cnt[b] == 0) continue;
            const VT<VEC> u1 = S[b * A + t];                           // T[my_field][b], my part
            const VT<VEC> u2 = S[my_field * A + b * PPF + my_part];    // T[b][my_field], same part
#pragma unroll
            for (int c = 0; c < VEC; c++) P += u1.a[c] * u2.a[c];
        }
    }
    // block reduce (P, dsq)
    {
        const int lane = t & 31, wid = t >> 5, nw = (blockDim.x + 31) >> 5;
        float a = warp_sum(P), d2 = warp_sum(dsq);
        if (lane == 0) { red[wid] = a; red[32 + wid] = d2; }
        __syncthreads();
        if (wid == 0) {
            float aa = lane < nw ? red[lane] : 0.f, dd = lane < nw ? red[32 + lane] : 0.f;
            aa = warp_sum(aa);
            dd = warp_sum(dd);
            if (lane == 0) {
                const float fm_pred = (float)((double)wsum + 0.5 * ((double)aa - (double)dd));
                const float p = ref_sigmoid(fm_pred);
                pred[r] = p;
                red[64] = p;
            }
        }
        __syncthreads();
    }
    const float p = red[64];
    double loss = 0.0, correct = 0.0;
    if (TRAIN) {
        const float y = label[r];
        const float d = p - y;
        if (d != 0.f) {  // train_ffm_algo.cpp:81-83: rows with pred == label contribute nothing at all
            if (t == 0 && do_stats) loss_terms(p, y, loss, correct);
            if (GROUPED) {
                // ---- phase 3': T tile -> global, transposed through shared memory so that the stores are coalesced
                const int FP = Fc * PPF;  // slots per [a] row
                VT<VEC>* dst = reinterpret_cast<VT<VEC>*>(Tbuf) + (size_t)r * Fc * A;
                for (int o = t; o < Fc * A; o += blockDim.x) {
                    const int a = o / FP, rem = o - a * FP, b = rem / PPF, part = rem - b * PPF;
                    dst[o] = S[b * A + a * PPF + part];  // T[a][b]
                }
                for (int b = t; b < Fc; b += blockDim.x) cntbuf[(size_t)r * Fc + b] = (uint16_t)min(cnt[b], 65535);
            } else {
            // ---- phase 3: gradients ------------------------------------------------------------------
            const int my_cnt = own ? cnt[my_field] : 0;
            for (int64_t i = b0; i < e0; i += FFM_UNROLL) {
                uint32_t f[FFM_UNROLL];
                int fl[FFM_UNROLL];
                float x[FFM_UNROLL];
                VT<VEC> v[FFM_UNROLL];
#pragma unroll
                for (int u = 0; u < FFM_UNROLL; u++) {
                    const bool ok = i + u < e0;
                    f[u] = ok ? __ldg(fid + i + u) : 0u;
                    fl[u] = ok ? (int)__ldg(field + i + u) : 0;
                    x[u] = ok ? (HAS_VAL ? __ldg(val + i + u) : 1.f) : 0.f;
                    if (ok && own) v[u] = vload<VEC>(V + (size_t)f[u] * rowlen + (size_t)t * VEC);
                    else {
#pragma unroll
                        for (int c = 0; c < VEC; c++) v[u].a[c] = 0.f;
                    }
                }
                if (BULK) {  // staging rows of the previous iteration must have been read by the TMA
                    if (t == 0) bulk_wait_read_all();
                    __syncthreads();
                }
#pragma unroll
                for (int u = 0; u < FFM_UNROLL; u++) {
                    if (i + u >= e0) break;
                    if (own) {
                        const int c_ib = my_cnt - (my_field == fl[u] ? 1 : 0);
                        VT<VEC> g;
#pragma unroll
                        for (int c = 0; c < VEC; c++) g.a[c] = 0.f;
                        if (c_ib > 0) {
                            const VT<VEC> tt = S[my_field * A + fl[u] * PPF + my_part];  // T[fld_i][my_field]
                            const float sx = d * x[u];
                            const float lc = l2 * (float)c_ib;
#pragma unroll
                            for (int c = 0; c < VEC; c++) {
                                float tv = tt.a[c];
                                if (my_field == fl[u]) tv -= x[u] * v[u].a[c];
                                g.a[c] = sx * tv + lc * v[u].a[c];
                            }
                            if (!BULK) vred<VEC>(gV + (size_t)f[u] * rowlen + (size_t)t * VEC, g);
                        }
                        if (BULK) stage[u * A + t] = g;
                    }
                    if (t == 0) {
                        red_add_f32(gW + f[u], d * x[u] + l2 * __ldg(W + f[u]));  // train_ffm_algo.cpp:98
                        if (touched) touched[f[u]] = 1;
                    }
                }
                if (BULK) {
                    fence_proxy_async_smem();
                    __syncthreads();
                    if (t == 0) {
#pragma unroll
                        for (int u = 0; u < FFM_UNROLL; u++)
                            if (i + u < e0)
                                bulk_reduce_add_f32(gV + (size_t)f[u] * rowlen, reinterpret_cast<const float*>(stage + u * A),
                                                    (uint32_t)(rowlen * sizeof(float)));
                        bulk_commit();
                    }
                }
            }
            if (BULK) {
                if (t == 0) bulk_wait_read_all();
                __syncthreads();
            }
            }  // !GROUPED
        }
    }
    if (TRAIN && do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

// ------------------------------------------------------------------------------------------------------------
// TMA-staged fused step (k % 4 == 0, training): the default RED-mode kernel
// ------------------------------------------------------------------------------------------------------------
// Same arithmetic as ffm_fused_kernel, different data movement: an embedding row is ONE contiguous, 16 B-aligned
// Fc*k*4-byte segment (624 B at Fc=39,k=4; 1248 B at k=8), exactly what cp.async.bulk (the TMA's non-tensor bulk copy)
// moves with a single instruction.  The rows of a chunk of up to CR entries of the sample (the whole sample, typically)
// are requested at once -- one bulk copy per row, all completing on ONE mbarrier armed with the chunk's byte count -- so
// CR whole rows are in flight per CTA at no register cost and without per-thread load instructions, and the gradient
// phase reads the rows from shared memory again instead of gathering them a second time.
// (A ring of single rows fed by a producer warp pays two mbarrier hand-shakes per row, more than the 16 B of work a
// consumer thread has per row.)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "LAB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra LAB_WAIT;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy of `bytes` (multiple of 16, both sides 16 B aligned), completion counted on `bar`
__device__ __forceinline__ void bulk_load(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// TRAIN = false: the forward-only instance of lctr_score (phases 1 and 2, the pCTR; no statistics, no gradient)
template <bool HAS_VAL, bool TRAIN>
__global__ void ffm_tma_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                               const uint16_t* __restrict__ field, const float* __restrict__ val,
                               const float* __restrict__ label, const float* __restrict__ W, const float* __restrict__ V,
                               int Fc, int k, float* __restrict__ pred, float* __restrict__ gW, float* __restrict__ gV,
                               uint8_t* __restrict__ touched, float l2, int64_t rb, double* partial, unsigned int* done,
                               double* out_slot, int do_stats, int CR /* rows per chunk */) {
    extern __shared__ __align__(16) unsigned char smem_raw[];  // (dynamic shared memory starts 1024 B aligned)
    const int A = Fc * k / 4;     // 16 B slots per row
    const int PPF = k / 4;        // slots per field
    const uint32_t rowbytes = (uint32_t)A * 16u;
    const uint32_t stage_bytes = (rowbytes + 127u) / 128u * 128u;
    unsigned char* rows = smem_raw;                                                         // [CR][stage_bytes]
    float4* S = reinterpret_cast<float4*>(smem_raw + (size_t)CR * stage_bytes);             // S[col b][slot a] = T[a][b]
    int* cnt = reinterpret_cast<int*>(S + (size_t)Fc * A);
    float* red = reinterpret_cast<float*>(cnt + Fc);                                        // [80]
    uint32_t* st_f = reinterpret_cast<uint32_t*>(red + 80);
    float* st_x = reinterpret_cast<float*>(st_f + CR);
    float* st_w = st_x + CR;
    uint16_t* st_fl = reinterpret_cast<uint16_t*>(st_w + CR);
    uint64_t* bar = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(st_fl + CR) + 7) & ~(uintptr_t)7);
    const int t = threadIdx.x;
    const int64_t r = rb + blockIdx.x;
    const int64_t b0 = row_ptr[r], e0 = row_ptr[r + 1];
    const size_t rowlen = (size_t)Fc * k;
    const bool own = t < A;
    const int my_field = own ? t / PPF : -1, my_part = own ? t % PPF : 0;

    if (t == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = t; i < Fc * A; i += blockDim.x) S[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = t; i < Fc; i += blockDim.x) cnt[i] = 0;

    uint32_t uses = 0;  // completed phases of `bar`: its parity
    // stage the indices of entries [c0, c0 + nst), then request their rows (one bulk copy each) and wait for all of them
    auto load_chunk = [&](int64_t c0, int nst) {
        __syncthreads();  // the previous chunk's rows and indices are no longer read; barrier init / S zeroing done
        for (int i = t; i < nst; i += blockDim.x) {
            const uint32_t f = __ldg(fid + c0 + i);
            st_f[i] = f;
            st_fl[i] = __ldg(field + c0 + i);
            st_x[i] = HAS_VAL ? __ldg(val + c0 + i) : 1.f;
            st_w[i] = __ldg(W + f);
        }
        __syncthreads();
        if (t == 0) mbar_arrive_expect_tx(bar, (uint32_t)nst * rowbytes);
        for (int i = t; i < nst; i += blockDim.x)
            bulk_load(rows + (size_t)i * stage_bytes, V + (size_t)st_f[i] * rowlen, rowbytes, bar);
        mbar_wait(bar, uses & 1u);
        uses++;
    };

    // ---- phase 1: T accumulation, wide sum, diagonal ---------------------------------------------------------------
    float wsum = 0.f, dsq = 0.f;
    for (int64_t c0 = b0; c0 < e0; c0 += CR) {
        const int nst = (int)min((int64_t)CR, e0 - c0);
        load_chunk(c0, nst);
        if (own) {
            for (int i = 0; i < nst; i++) {
                const int flu = st_fl[i];
                const float xu = st_x[i];
                const float4 v = reinterpret_cast<const float4*>(rows + (size_t)i * stage_bytes)[t];
                float4& dst = S[flu * A + t];
                const float4 tv = make_float4(v.x * xu, v.y * xu, v.z * xu, v.w * xu);
                dst.x += tv.x; dst.y += tv.y; dst.z += tv.z; dst.w += tv.w;
                if (my_field == flu) dsq += tv.x * tv.x + tv.y * tv.y + tv.z * tv.z + tv.w * tv.w;
            }
        }
        if (t == 0) {
            for (int i = 0; i < nst; i++) {
                wsum += st_w[i] * st_x[i];  // fm_pred += W[fid] * X  (train_ffm_algo.cpp:60)
                cnt[st_fl[i]] += 1;
            }
        }
    }
    __syncthreads();

    // ---- phase 2: P = sum_{a,b} <T[a][b], T[b][a]> ------------------------------------------------------------------
    float P = 0.f;
    if (own) {
        for (int b = 0; b < Fc; b++) {
            if (cnt[b] == 0) continue;
            const float4 u1 = S[b * A + t];
            const float4 u2 = S[my_field * A + b * PPF + my_part];
            P += u1.x * u2.x + u1.y * u2.y + u1.z * u2.z + u1.w * u2.w;
        }
    }
    {
        const int lane = t & 31, wid = t >> 5, nw = (blockDim.x + 31) >> 5;
        float a = warp_sum(P), d2 = warp_sum(dsq);
        if (lane == 0) { red[wid] = a; red[32 + wid] = d2; }
        __syncthreads();
        if (wid == 0) {
            float aa = lane < nw ? red[lane] : 0.f, dd = lane < nw ? red[32 + lane] : 0.f;
            aa = warp_sum(aa);
            dd = warp_sum(dd);
            if (lane == 0) {
                const float fm_pred = (float)((double)wsum + 0.5 * ((double)aa - (double)dd));
                const float p = ref_sigmoid(fm_pred);
                pred[r] = p;
                red[64] = p;
            }
        }
        __syncthreads();
    }
    if (!TRAIN) return;
    const float p = red[64];
    double loss = 0.0, correct = 0.0;
    const float y = label[r];
    const float d = p - y;
    if (d != 0.f) {  // train_ffm_algo.cpp:81-83: rows with pred == label contribute nothing at all
        if (t == 0 && do_stats) loss_terms(p, y, loss, correct);
        // ---- phase 3: gradients, from the rows still in shared memory (one chunk) or streamed a second time -----------
        const int my_cnt = own ? cnt[my_field] : 0;
        const bool resident = e0 - b0 <= CR;
        for (int64_t c0 = b0; c0 < e0; c0 += CR) {
            const int nst = (int)min((int64_t)CR, e0 - c0);
            if (!resident) load_chunk(c0, nst);
            if (own) {
                for (int i = 0; i < nst; i++) {
                    const int flu = st_fl[i];
                    const int c_ib = my_cnt - (my_field == flu ? 1 : 0);
                    if (c_ib <= 0) continue;
                    const float xu = st_x[i];
                    const float4 v = reinterpret_cast<const float4*>(rows + (size_t)i * stage_bytes)[t];
                    const float4 tt = S[my_field * A + flu * PPF + my_part];  // T[fld_i][my_field]
                    const float sx = d * xu, lc = l2 * (float)c_ib;
                    float tx = tt.x, ty = tt.y, tz = tt.z, tw = tt.w;
                    if (my_field == flu) { tx -= xu * v.x; ty -= xu * v.y; tz -= xu * v.z; tw -= xu * v.w; }
                    const float4 g = make_float4(sx * tx + lc * v.x, sx * ty + lc * v.y, sx * tz + lc * v.z, sx * tw + lc * v.w);
                    red_add_v4(gV + (size_t)st_f[i] * rowlen + (size_t)t * 4, g);
                }
            }
            // wide gradients by the threads past the row slots (or thread 0 when there are none)
            const int w0 = A < (int)blockDim.x ? A : 0, wn = A < (int)blockDim.x ? (int)blockDim.x - A : 1;
            if (t >= w0 && t < w0 + wn) {
                for (int i = t - w0; i < nst; i += wn) {
                    const uint32_t f = st_f[i];
                    red_add_f32(gW + f, d * st_x[i] + l2 * st_w[i]);  // train_ffm_algo.cpp:98
                    if (touched) touched[f] = 1;
                }
            }
        }
    }
    if (do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

// FM_Predict, field-aware branch (predict/fm_predict.cpp:34-53) in the reference's OWN order -- no field-pair factorisation:
// warp = sample; for entry i the lanes form the pair terms field_w * X * X2 of 32 partners j at a time (each dot product in
// the avx lane order of common/avx.h:102-127), and the scalar chain fm_pred += ... is replayed in j order through shuffles,
// so the float sequence is exactly the reference's double loop.  O(n^2 k) per sample: the parity predictor
// (cfg.deterministic == 1); the factorised forward above is the throughput predictor.
template <bool HAS_VAL>
__global__ void __launch_bounds__(256)
ffm_predict_inorder_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                           const uint16_t* __restrict__ field, const float* __restrict__ val, const float* __restrict__ W,
                           const float* __restrict__ V, int Fc, int k, float* __restrict__ pred, int64_t rows) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int64_t b = row_ptr[r], e = row_ptr[r + 1];
    const size_t rs = (size_t)Fc * k;
    float fm = 0.f;
    for (int64_t i = b; i < e; i++) {
        const size_t f1 = fid[i];
        const int fl1 = field[i];
        const float X = HAS_VAL ? val[i] : 1.f;
        fm = fm + W[f1] * X;                                                   // fm_predict.cpp:40
        for (int64_t j0 = i + 1; j0 < e; j0 += 32) {
            const int64_t j = j0 + lane;
            float t = 0.f;
            if (j < e) {
                const size_t f2 = fid[j];
                const int fl2 = field[j];
                const float* a = V + f1 * rs + (size_t)fl2 * k;                // getV_field(fid, field2, 0)   :47
                const float* c = V + f2 * rs + (size_t)fl1 * k;                // getV_field(fid2, field, 0)   :48
                const float fw = avx_dot_seq([&](int q) { return a[q]; }, [&](int q) { return c[q]; }, k);
                t = fw * X;
                t = t * (HAS_VAL ? val[j] : 1.f);                              // field_w * X * X2             :49
            }
            const int cnt = (int)min((int64_t)32, e - j0);
            for (int l = 0; l < cnt; l++) fm = fm + __shfl_sync(kFull, t, l);  // fm_pred += ... in j order
        }
    }
    if (lane == 0) pred[r] = ref_sigmoid(fm);                                  // :56
}

int launch_ffm_predict_inorder(lctr_ctx* c, Slot& s) {
    if (s.rows <= 0) return 0;
    LCTR_CHECK(s.has_field, "FFM batch uploaded without the field array");
    const unsigned grid = (unsigned)((s.rows + 7) / 8);
    return launch(c, {grid, 256, 0, c->stream}, s.has_val ? ffm_predict_inorder_kernel<true> : ffm_predict_inorder_kernel<false>,
                  s.row_ptr, s.fid, s.field, s.val, c->cW, c->cV, (int)c->cfg.field_cnt, (int)c->cfg.factor_cnt, s.pred, s.rows);
}

// the CTA-per-sample kernel's instance (bulk: the TMA bulk reduce-add of the gradient rows, 4-wide training rows only)
template <int VEC, bool HV, bool TR>
static auto ffm_kernel(bool bulk) {
    return bulk ? ffm_fused_kernel<VEC, HV, TR, (VEC == 4) && TR> : ffm_fused_kernel<VEC, HV, TR, false>;
}
template <int VEC>
static auto ffm_kernel(bool hv, bool train, bool bulk) {
    return hv ? (train ? ffm_kernel<VEC, true, true>(bulk) : ffm_kernel<VEC, true, false>(bulk))
              : (train ? ffm_kernel<VEC, false, true>(bulk) : ffm_kernel<VEC, false, false>(bulk));
}

// train: the kernel of a train step (stats: with its statistics); otherwise the forward-only CTA-per-sample kernel.  score:
// the kernel a train step would choose, in its forward-only instance (lctr_score: the pCTR of the step, no statistics, no
// gradient)
static int ffm_launch(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool train, bool stats, bool grouped = false,
                      bool score = false) {
    const int k = (int)c->cfg.factor_cnt, Fc = (int)c->cfg.field_cnt;
    const int64_t rows = re - rb;
    if (rows <= 0) return 0;
    LCTR_CHECK(s.has_field, "FFM batch uploaded without the field array");
    const int vec = (k % 4 == 0) ? 4 : ((k % 2 == 0) ? 2 : 1);
    const int A = Fc * k / vec;
    LCTR_CHECK(A <= 1024, "FFM row of %d slots exceeds one CTA (Fc=%d k=%d)", A, Fc, k);
    const int tpb = std::max(64, (A + 31) / 32 * 32);
    // TMA bulk reduce-add of whole gradient rows is built but off by default: on B200s it was no faster than the vector
    // REDs (both end in the same L2 reductions); not re-measured on H100s.
    static const bool use_bulk = getenv("LCTR_FFM_BULK") && atoi(getenv("LCTR_FFM_BULK")) == 1;
    const bool bulk = use_bulk && train && vec == 4 && (Fc * k * 4) % 16 == 0;
    const size_t smem = ((size_t)Fc * A * vec * 4 + (size_t)Fc * 4 + 80 * 4 + (size_t)kFfmStage * 10 + 15) / 16 * 16 +
                        (bulk ? (size_t)FFM_UNROLL * A * vec * 4 : 0);
    LCTR_CHECK(smem <= 227 * 1024, "FFM field-pair tile needs %zu B shared memory (> 227 KB): Fc=%d k=%d", smem, Fc, k);
    double* out_slot = c->stats + 2 * (c->step % kStatRing);
    ProfScope prof(c, PROF_FFM_FUSED);
    if (grouped) {
        LCTR_CHECK(train && vec == 4 && c->ffm_T && c->ffm_cnt, "grouped FFM step needs k %% 4 == 0 and the tile buffer");
        return launch(c, {(unsigned)rows, (unsigned)tpb, smem, c->stream},
                      s.has_val ? ffm_fused_kernel<4, true, true, false, true> : ffm_fused_kernel<4, false, true, false, true>,
                      s.row_ptr, s.fid, s.field, s.val, s.label, c->cW, c->cV, Fc, k, s.pred, c->cgW, c->cgV, nullptr, c->cfg.l2_reg, rb,
                      c->stat_partial, c->stat_done, out_slot, stats ? 1 : 0, c->ffm_T, c->ffm_cnt);
    }
    // LCTR_FFM_TMA=1 selects the TMA-staged kernel (cp.async.bulk rows + mbarrier).  It is parity-green but NOT the
    // default: both kernels are issue-bound rather than memory-bound, and staging whole rows in shared memory cuts the
    // instruction count but leaves 2 CTAs = 4 warps per SM next to the field-pair tile, against 16 warps of the
    // register-staged kernel, which was the faster of the two on B200s.  The choice has not been re-measured on H100s.
    static const bool use_tma = getenv("LCTR_FFM_TMA") && atoi(getenv("LCTR_FFM_TMA")) == 1;
    const bool tr = train && !score;  // the instance: forward + backward, or forward only
    if (use_tma && train && vec == 4 && !bulk) {
        // rows per chunk: as many as leave 3 (narrow rows) or 2 CTAs per SM, at least 40, at most 96
        const size_t stage_bytes = ((size_t)A * 16 + 127) / 128 * 128;
        const size_t fixed = (size_t)Fc * A * 16 + (size_t)Fc * 4 + 80 * 4 + 64 + 1024;
        int CR = 0;
        for (int ncta = 3; ncta >= 1 && CR < 40; ncta--) {
            const size_t budget = (size_t)227 * 1024 / ncta;
            CR = budget > fixed ? (int)((budget - fixed) / (stage_bytes + 14)) : 0;
        }
        CR = std::min(CR, 96);
        LCTR_CHECK(CR >= 8, "FFM field-pair tile + row buffer do not fit 227 KB shared memory: Fc=%d k=%d", Fc, k);
        const size_t smem2 = (size_t)CR * (stage_bytes + 14) + fixed;
        const int tpb2 = std::max(64, (A + 31) / 32 * 32);
        auto tma = s.has_val ? (tr ? ffm_tma_kernel<true, true> : ffm_tma_kernel<true, false>)
                             : (tr ? ffm_tma_kernel<false, true> : ffm_tma_kernel<false, false>);
        return launch(c, {(unsigned)rows, (unsigned)tpb2, smem2, c->stream}, tma, s.row_ptr, c->cfg.world > 1 ? s.ent_pslot : s.fid, s.field, s.val, s.label, c->cW, c->cV, Fc, k, s.pred, c->cgW,
                      c->cgV, c->cfg.world > 1 ? nullptr : c->touched.get(), c->cfg.l2_reg, rb, c->stat_partial, c->stat_done, out_slot,
                      stats && tr ? 1 : 0, CR);
    }
    // default for k % 4 == 0: the warp-per-sample kernel of ffm_warp.cu (LCTR_FFM_WARP=0 keeps the CTA-per-sample kernel below)
    if (train && !bulk && vec == 4) {
        const int rc = launch_ffm_warp(c, s, rb, re, stats && tr, tr);
        if (rc >= 0) return rc;
    }
    // (a forward-only instance of the bulk kernel is the plain one: ffm_kernel takes the bulk path with training only)
    auto kern = vec == 4 ? ffm_kernel<4>(s.has_val, tr, bulk) : vec == 2 ? ffm_kernel<2>(s.has_val, tr, bulk)
                                                                 : ffm_kernel<1>(s.has_val, tr, bulk);
    return launch(c, {(unsigned)rows, (unsigned)tpb, smem, c->stream}, kern, s.row_ptr, c->cfg.world > 1 ? s.ent_pslot : s.fid,
                  s.field, s.val, s.label, c->cW, c->cV, Fc, k, s.pred, c->cgW, c->cgV, c->cfg.world > 1 ? nullptr : c->touched.get(),
                  c->cfg.l2_reg, rb, c->stat_partial, c->stat_done, out_slot, stats && tr ? 1 : 0, nullptr, nullptr);
}

// forward + backward are one fused kernel (stats: a train step; otherwise forward only)
int launch_ffm_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats) {
    return ffm_launch(c, s, rb, re, /*train=*/stats, stats);
}
// forward half of the feature-grouped step: predictions, loss, and the T tiles for ffm_grouped.cu
int launch_ffm_forward_tiles(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    return ffm_launch(c, s, rb, re, true, true, true);
}
// lctr_score: the pCTR a train step computes, by the forward code of the kernel it runs.  The feature-grouped step's
// kernel (deterministic = 2) is the CTA-per-sample kernel with its T tiles stored, whose forward-only instance is the
// plain one
int launch_ffm_score(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    return ffm_launch(c, s, rb, re, c->grad_path != GRAD_FEATURE_MAJOR, false, false, true);
}

}  // namespace lctr
