// lightctr_b200/csrc/ffm_warp.cu -- the FFM training step (train/train_ffm_algo.cpp:51-118), one WARP per sample.
//
// Same factorisation and the same terms as ffm.cu (per-sample field-pair sums T[a][slot] = sum over the sample's entries
// of field a of x * row[slot]; slot = (target field b, 4-float part)), but organised around the instruction count: the
// CTA-per-sample kernel is issue bound (39 of 64 threads own a slot, every entry pays a block-wide index staging, shared-memory read-modify-writes of T,
// thread-0 scalar work and two __syncthreads per chunk).  Here
//   * a warp owns a sample and its own T tile in shared memory: no block barrier anywhere in the sample loop;
//   * lane j reads the (fid, field, x, W[fid]) of entry j of a 32-entry chunk -- the wide sum, the gW REDs and the touched
//     marks are lane-parallel over entries -- and the row loop gets its (fid, field, x) by shuffles;
//   * entries of one field are accumulated in registers and T[a] is written once per field run (first write is a plain
//     store: no zero fill of the tile), fields absent from the sample are zeroed afterwards;
//   * the pair sum walks the Fc(Fc+1)/2 unordered field pairs, flattened over the lanes through a small table;
//   * the gradient phase re-reads the rows (L2 hits: the sample's rows were read microseconds earlier), U entries in
//     flight, and leaves as one red.global.add.v4.f32 per slot -- contiguous per row.
// CTAs are persistent (one per SM, as many warps as T tiles fit into 227 KB: 9 at Fc=39,k=4; 4 at k=8) and stride over
// the samples.  Requirements: k % 4 == 0, Fc <= 64, Fc*k/4 <= 128 slots; everything else stays on ffm.cu.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace lctr {

namespace {

// entries whose row loads are in flight together (registers: KU * PASSES float4 per lane; few warps per SM, so the register
// file is the prefetch buffer)
__host__ __device__ constexpr int group_size(int passes) { return passes <= 2 ? 8 : (passes == 3 ? 8 : 4); }

__device__ __forceinline__ float4 ld4(const float* p) { return ldg_f4(p); }

// The library is compiled with -fmad=false (the exact-order kernels must round like the reference's SSE code); this
// kernel is the order-free path, so it contracts explicitly.
template <bool HAS_VAL>
__device__ __forceinline__ void acc4(float4& acc, const float4& v, float x) {
    if (HAS_VAL) { acc.x = fmaf(v.x, x, acc.x); acc.y = fmaf(v.y, x, acc.y); acc.z = fmaf(v.z, x, acc.z); acc.w = fmaf(v.w, x, acc.w); }
    else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
}

constexpr int max_warps(int passes) { return passes <= 2 ? 10 : 5; }  // 3-4 passes keep kU rows of 3-4 x 16 B per lane: 255 registers

// TRAIN = false: the forward-only instance of lctr_score (phases 1 and 2, the pCTR; no statistics, no gradient)
template <int PASSES, bool HAS_VAL, bool TRAIN>
__global__ void __launch_bounds__(max_warps(PASSES) * 32, 1)
ffm_warp_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid, const uint16_t* __restrict__ field,
                const float* __restrict__ val, const float* __restrict__ label, const float* __restrict__ W,
                const float* __restrict__ V, int Fc, int k, float* __restrict__ pred, float* __restrict__ gW,
                float* __restrict__ gV, uint8_t* __restrict__ touched, float l2, int64_t rb, int64_t rows, int tile_bytes,
                double* partial, unsigned int* done, double* out_slot, int do_stats) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int KU = group_size(PASSES);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    const int PPF = k >> 2;          // 16 B parts per field
    const int A = Fc * PPF;          // slots per row
    const size_t rowlen = (size_t)Fc * k;
    const int npair = Fc * (Fc + 1) / 2 * PPF;
    // pair table (shared by the CTA): a | b << 8 | part << 16, unordered field pairs a <= b
    uint32_t* ptab = reinterpret_cast<uint32_t*>(smem_raw);
    float4* T = reinterpret_cast<float4*>(smem_raw + (((size_t)npair * 4 + 127) & ~(size_t)127) + (size_t)wid * tile_bytes);
    for (int q = threadIdx.x; q < npair; q += blockDim.x) {
        const int pr = q / PPF, part = q - pr * PPF;
        int a = 0, rem = pr;  // row a of the upper triangle holds Fc - a pairs
        while (rem >= Fc - a) { rem -= Fc - a; a++; }
        ptab[q] = (uint32_t)a | ((uint32_t)(a + rem) << 8) | ((uint32_t)part << 16);
    }
    __syncthreads();

    // per-lane slot constants.  Only the last pass can have lanes without a slot; those lanes shadow the last slot (they
    // load and compute on valid data, and are masked where something leaves the lane), which keeps every load and
    // arithmetic instruction of the row loops unpredicated.
    int sb[PASSES], tb[PASSES], so[PASSES];
    const bool own_last = (PASSES - 1) * 32 + lane < A;
#pragma unroll
    for (int p = 0; p < PASSES; p++) {
        const int slot = min(p * 32 + lane, A - 1);
        const int b = slot / PPF;
        sb[p] = (p < PASSES - 1 || own_last) ? b : -1;  // the field this lane's slot belongs to (-1: shadow lane)
        tb[p] = b * A + (slot - b * PPF);               // T[b][. * PPF + my part]
        so[p] = slot * 4;                                // float offset of the slot inside a row
    }

    double loss = 0.0, correct = 0.0;
    const int64_t r_end = rb + rows, r_step = (int64_t)gridDim.x * nwarp;
    int64_t r = rb + (int64_t)blockIdx.x * nwarp + wid;
    int64_t nb0 = 0, ne0 = 0;
    if (r < r_end) { nb0 = row_ptr[r]; ne0 = row_ptr[r + 1]; }
    for (; r < r_end; r += r_step) {
        const int64_t b0 = nb0, e0 = ne0;
        if (r + r_step < r_end) { nb0 = row_ptr[r + r_step]; ne0 = row_ptr[r + r_step + 1]; }  // the next sample's extent: off the chain
        // the sample's (fid, field, x, W[fid]) live in registers, lane j of chunk c holding entry 32 c + j of a 128-entry
        // window: one round trip for the whole sample, and the gradient phase reuses them when the sample fits one window
        uint32_t f_c[4]; int a_c[4]; float x_c[4], w_c[4];
        auto load_window = [&](int64_t s0) {
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int64_t e = s0 + 32 * c + lane;
                const bool ok = e < e0;
                f_c[c] = ok ? __ldg(fid + e) : 0u;
                a_c[c] = ok ? (int)__ldg(field + e) : 0;
                x_c[c] = ok ? (HAS_VAL ? __ldg(val + e) : 1.f) : 0.f;
            }
#pragma unroll
            for (int c = 0; c < 4; c++) w_c[c] = (s0 + 32 * c + lane < e0) ? __ldg(W + f_c[c]) : 0.f;
        };
        const bool one_window = e0 - b0 <= 128;
        // ---- phase 1: gather, T, wide sum, diagonal, per-field counts ---------------------------------------------
        float4 acc[PASSES];
        int cntf[PASSES];
        float wsum = 0.f, dsq = 0.f;
        int cur = -1;
        unsigned long long seen = 0ull;
#pragma unroll
        for (int p = 0; p < PASSES; p++) { acc[p] = make_float4(0.f, 0.f, 0.f, 0.f); cntf[p] = 0; }
        auto flush = [&](int a) {  // warp-uniform a: T[a] (+)= the register sums of a run of entries of field a
            float4* Ta = T + a * A;
            const bool first = !((seen >> a) & 1ull);
#pragma unroll
            for (int p = 0; p < PASSES; p++) {
                if (p < PASSES - 1 || own_last) {
                    float4 t = acc[p];
                    if (!first) {
                        const float4 o = Ta[p * 32 + lane];
                        t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w;
                    }
                    Ta[p * 32 + lane] = t;
                }
                acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            seen |= 1ull << a;
        };
        for (int64_t s0 = b0; s0 < e0; s0 += 128) {
          load_window(s0);
#pragma unroll
          for (int c = 0; c < 4; c++) wsum = fmaf(w_c[c], x_c[c], wsum);  // fm_pred += W[fid] * X  (train_ffm_algo.cpp:60)
#pragma unroll 1
          for (int c = 0; c < 4; c++) {
            const int64_t c0 = s0 + 32 * c;
            if (c0 >= e0) break;
            const int nst = (int)min((int64_t)32, e0 - c0);
            const uint32_t f_l = c == 0 ? f_c[0] : (c == 1 ? f_c[1] : (c == 2 ? f_c[2] : f_c[3]));
            const int a_l = c == 0 ? a_c[0] : (c == 1 ? a_c[1] : (c == 2 ? a_c[2] : a_c[3]));
            const float x_l = c == 0 ? x_c[0] : (c == 1 ? x_c[1] : (c == 2 ? x_c[2] : x_c[3]));
            auto group = [&](auto tag, int i) {
                constexpr int UU = decltype(tag)::value;
                float4 v[UU][PASSES];
                int a[UU]; float x[UU];
#pragma unroll
                for (int u = 0; u < UU; u++) {
                    const uint32_t f = __shfl_sync(0xffffffffu, f_l, i + u);
                    a[u] = __shfl_sync(0xffffffffu, a_l, i + u);
                    x[u] = HAS_VAL ? __shfl_sync(0xffffffffu, x_l, i + u) : 1.f;
                    const float* row = V + (size_t)f * rowlen;
#pragma unroll
                    for (int p = 0; p < PASSES; p++) v[u][p] = ld4(row + so[p]);
                }
#pragma unroll
                for (int u = 0; u < UU; u++) {
                    if (a[u] != cur) {  // warp-uniform
                        if (cur >= 0) flush(cur);
                        cur = a[u];
                    }
#pragma unroll
                    for (int p = 0; p < PASSES; p++) {
                        acc4<HAS_VAL>(acc[p], v[u][p], x[u]);
                        if (sb[p] == a[u]) {  // the slot of the entry's own field: diagonal term and the field's count
                            const float4 t = HAS_VAL ? make_float4(v[u][p].x * x[u], v[u][p].y * x[u], v[u][p].z * x[u], v[u][p].w * x[u]) : v[u][p];
                            dsq = fmaf(t.x, t.x, fmaf(t.y, t.y, fmaf(t.z, t.z, fmaf(t.w, t.w, dsq))));
                            cntf[p]++;
                        }
                    }
                }
            };
            int i = 0;
            for (; i + KU <= nst; i += KU) group(std::integral_constant<int, KU>{}, i);
            for (; i + 4 <= nst; i += 4) group(std::integral_constant<int, 4>{}, i);  // tails in 4 / 2 / 1: each group is one round trip
            for (; i + 2 <= nst; i += 2) group(std::integral_constant<int, 2>{}, i);
            for (; i < nst; i++) group(std::integral_constant<int, 1>{}, i);
          }
        }
        if (cur >= 0) flush(cur);
        {   // fields the sample does not have: their T rows are read by the pair sum and the gradient phase as zeros
            unsigned long long miss = ~seen & (Fc >= 64 ? ~0ull : ((1ull << Fc) - 1ull));
            while (miss) {
                const int a = __ffsll((long long)miss) - 1;
                miss &= miss - 1;
#pragma unroll
                for (int p = 0; p < PASSES; p++)
                    if (p < PASSES - 1 || own_last) T[a * A + p * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        __syncwarp();

        // ---- phase 2: P = sum_{a,b} <T[a][b], T[b][a]> over unordered pairs (off-diagonal pairs count twice) -------
        float P = 0.f;
        for (int q = lane; q < npair; q += 32) {
            const uint32_t e = ptab[q];
            const int a = e & 0xff, b = (e >> 8) & 0xff, part = e >> 16;
            const float4 u1 = T[a * A + b * PPF + part];
            const float4 u2 = T[b * A + a * PPF + part];
            const float d4 = fmaf(u1.x, u2.x, fmaf(u1.y, u2.y, fmaf(u1.z, u2.z, u1.w * u2.w)));
            P = fmaf(a == b ? 1.f : 2.f, d4, P);
        }
        P = warp_sum(P);
        dsq = warp_sum(dsq);
        wsum = warp_sum(wsum);
        const float fm_pred = (float)((double)wsum + 0.5 * ((double)P - (double)dsq));
        const float pr = ref_sigmoid(fm_pred);
        const float y = label[r];
        if (lane == 0) pred[r] = pr;
        if (!TRAIN) continue;
        const float d = pr - y;
        if (d == 0.f) continue;  // train_ffm_algo.cpp:81-83: rows with pred == label contribute nothing at all
        if (lane == 0 && do_stats) {
            double l1, c1;
            loss_terms(pr, y, l1, c1);
            loss += l1; correct += c1;
        }

        // ---- phase 3: gradients -------------------------------------------------------------------------------------
        // g[i][b] = d x_i (T[b][a_i] - [b == a_i] x_i v) + l2 c_ib v,  c_ib = cnt[b] - [b == a_i]; nothing at all when c_ib == 0
        float lc0[PASSES], lc1[PASSES];  // l2 * c_ib for an entry of another field / of the slot's own field
        bool go0[PASSES], go1[PASSES];
#pragma unroll
        for (int p = 0; p < PASSES; p++) {
            lc0[p] = l2 * (float)cntf[p]; lc1[p] = l2 * (float)(cntf[p] - 1);
            go0[p] = sb[p] >= 0 && cntf[p] > 0; go1[p] = sb[p] >= 0 && cntf[p] > 1;
        }
        for (int64_t s0 = b0; s0 < e0; s0 += 128) {
          if (!one_window) load_window(s0);
#pragma unroll
          for (int c = 0; c < 4; c++)
              if (s0 + 32 * c + lane < e0) {
                  red_add_f32(gW + f_c[c], fmaf(l2, w_c[c], d * x_c[c]));  // train_ffm_algo.cpp:98
                  if (touched) touched[f_c[c]] = 1;
              }
#pragma unroll 1
          for (int c = 0; c < 4; c++) {
            const int64_t c0 = s0 + 32 * c;
            if (c0 >= e0) break;
            const int nst = (int)min((int64_t)32, e0 - c0);
            const uint32_t f_l = c == 0 ? f_c[0] : (c == 1 ? f_c[1] : (c == 2 ? f_c[2] : f_c[3]));
            const int a_l = c == 0 ? a_c[0] : (c == 1 ? a_c[1] : (c == 2 ? a_c[2] : a_c[3]));
            const float x_l = c == 0 ? x_c[0] : (c == 1 ? x_c[1] : (c == 2 ? x_c[2] : x_c[3]));
            auto group = [&](auto tag, int i) {
                constexpr int UU = decltype(tag)::value;
                float4 v[UU][PASSES];
                uint32_t f[UU]; int a[UU]; float x[UU];
#pragma unroll
                for (int u = 0; u < UU; u++) {
                    f[u] = __shfl_sync(0xffffffffu, f_l, i + u);
                    a[u] = __shfl_sync(0xffffffffu, a_l, i + u);
                    x[u] = HAS_VAL ? __shfl_sync(0xffffffffu, x_l, i + u) : 1.f;
                    const float* row = V + (size_t)f[u] * rowlen;
#pragma unroll
                    for (int p = 0; p < PASSES; p++) v[u][p] = ld4(row + so[p]);
                }
#pragma unroll
                for (int u = 0; u < UU; u++) {
                    const float sx = d * x[u];
                    float* grow = gV + (size_t)f[u] * rowlen;
                    const int ta = a[u] * PPF;
#pragma unroll
                    for (int p = 0; p < PASSES; p++) {
                        const bool self = sb[p] == a[u];
                        const float4 tt = T[tb[p] + ta];  // T[b][a], my part
                        const float c1 = self ? fmaf(-sx, x[u], lc1[p]) : lc0[p];  // coefficient of v
                        const float4 vv = v[u][p];
                        if (self ? go1[p] : go0[p])
                            red_add_v4(grow + so[p], make_float4(fmaf(sx, tt.x, c1 * vv.x), fmaf(sx, tt.y, c1 * vv.y),
                                                                 fmaf(sx, tt.z, c1 * vv.z), fmaf(sx, tt.w, c1 * vv.w)));
                    }
                }
            };
            int i = 0;
            for (; i + KU <= nst; i += KU) group(std::integral_constant<int, KU>{}, i);
            for (; i + 4 <= nst; i += 4) group(std::integral_constant<int, 4>{}, i);  // tails in 4 / 2 / 1: each group is one round trip
            for (; i + 2 <= nst; i += 2) group(std::integral_constant<int, 2>{}, i);
            for (; i < nst; i++) group(std::integral_constant<int, 1>{}, i);
          }
        }
        __syncwarp();  // T is rewritten by the next sample
    }
    if (TRAIN && do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

}  // namespace

// returns 0 when launched, -1 when the shape is not covered (caller falls back to ffm.cu), 1 on error.  train = false: the
// forward-only instance (stats unused)
template <int PASSES>
static auto warp_kernel(bool hv, bool train) {
    return hv ? (train ? ffm_warp_kernel<PASSES, true, true> : ffm_warp_kernel<PASSES, true, false>)
              : (train ? ffm_warp_kernel<PASSES, false, true> : ffm_warp_kernel<PASSES, false, false>);
}

int launch_ffm_warp(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats, bool train) {
    static const bool off = getenv("LCTR_FFM_WARP") && atoi(getenv("LCTR_FFM_WARP")) == 0;
    const int k = (int)c->cfg.factor_cnt, Fc = (int)c->cfg.field_cnt;
    if (off || k % 4 != 0 || Fc > 64) return -1;
    const int A = Fc * k / 4, passes = (A + 31) / 32;
    if (passes > 4) return -1;
    const int64_t rows = re - rb;
    const size_t tile = ((size_t)Fc * A * 16 + 127) & ~(size_t)127;
    const size_t tab = (((size_t)Fc * (Fc + 1) / 2 * (k / 4)) * 4 + 127) & ~(size_t)127;
    const size_t budget = (size_t)227 * 1024 - 1024;  // static shared memory of publish_stats
    if (tab + tile > budget) return -1;
    int warps = (int)std::min<size_t>((budget - tab) / tile, (size_t)max_warps(passes));
    const size_t smem = tab + (size_t)warps * tile;
    const int sm = c->sm_count;
    const unsigned grid = (unsigned)std::min<int64_t>(sm, (rows + warps - 1) / warps);
    double* out_slot = c->stats + 2 * (c->step % kStatRing);
    ProfScope prof(c, PROF_FFM_FUSED);
    const uint32_t* ids = c->cfg.world > 1 ? s.ent_pslot : s.fid;
    uint8_t* touched = c->cfg.world > 1 ? nullptr : c->touched.get();
    auto kern = passes == 1 ? warp_kernel<1>(s.has_val, train) : passes == 2 ? warp_kernel<2>(s.has_val, train)
              : passes == 3 ? warp_kernel<3>(s.has_val, train) : warp_kernel<4>(s.has_val, train);
    return launch(c, {grid, (unsigned)warps * 32, smem, c->stream}, kern, s.row_ptr, ids, s.field, s.val, s.label, c->cW, c->cV, Fc,
                  k, s.pred, c->cgW, c->cgV, touched, c->cfg.l2_reg, rb, rows, (int)tile, c->stat_partial, c->stat_done, out_slot,
                  stats ? 1 : 0);
}

}  // namespace lctr
