// lightctr_b200/csrc/fm.cu -- FM / NFM embedding gather (forward) and scatter-add (backward), sm_90a.
//
// Reference semantics: Train_FM_Algo::batchGradCompute / accumWVGrad (train/train_fm_algo.cpp:63-118)
// and the wide + bi-interaction / accumWideGrad / accumDeepGrad parts of Train_NFM_Algo
// (train/train_nfm_algo.cpp:78-94,126-159).
//
// Mapping: one warp per sample.  A V row (k floats) is covered by LPR lanes, each holding VEC
// contiguous floats (k = 16 -> 4 lanes x float4: one 64 B row = two 32 B sectors, fully used), so a
// warp gathers G = 32/LPR rows per step.  The CSR columns of the sample are read 32 at a time
// with one coalesced 128 B load and redistributed by shuffle.  All gathers of a 32-entry chunk are
// issued before any is consumed (LPR independent 16 B loads in flight per lane).  Interaction sums
// are reduced with xor-shuffles.  HBM/L2-bound integer+fp32 work: no tensor cores here by design.
#include <stdlib.h>

#include "opt.cuh"

namespace lctr {

template <int VEC>
struct Vec {
    float a[VEC];
};

template <int VEC>
__device__ __forceinline__ Vec<VEC> load_row(const float* p, bool active) {
    Vec<VEC> r;
    if (VEC == 4) {
        float4 t = active ? ldg_f4(p) : make_float4(0.f, 0.f, 0.f, 0.f);
        r.a[0] = t.x; r.a[1 % VEC] = t.y; r.a[2 % VEC] = t.z; r.a[3 % VEC] = t.w;
    } else {
        r.a[0] = active ? __ldg(p) : 0.f;
    }
    return r;
}

// ------------------------------------------------------------------------------------------------
// forward -- arithmetic in the reference's own order
// ------------------------------------------------------------------------------------------------
// avx_dotProduct(t, t, K) (common/avx.h:102-127) on K register-resident values, in the reference's order:
// 8 lane accumulators over the full 8-chunks, the hsum tree, then the scalar tail.
template <int K>
__device__ __forceinline__ float avx_dot_regs(const float (&t)[K]) {
    float result = 0.f;
    constexpr int NFULL = K / 8;
    if (NFULL > 0) {
        float d[8];
#pragma unroll
        for (int l = 0; l < 8; l++) d[l] = t[l] * t[l];
#pragma unroll
        for (int m = 1; m < NFULL; m++)
#pragma unroll
            for (int l = 0; l < 8; l++) d[l] = d[l] + t[8 * m + l] * t[8 * m + l];
        const float a0 = d[4] + d[0], a1 = d[5] + d[1], a2 = d[6] + d[2], a3 = d[7] + d[3];
        const float b0 = a0 + a2, b1 = a1 + a3;
        result = b0 + b1;
    }
#pragma unroll
    for (int i = NFULL * 8; i < K; i++) result = result + t[i] * t[i];
    return result;
}

// Forward, two phases per warp (= one sample):
//   phase 1 (order-free, wide): lane j owns feature j of the current block of NB features: it gathers the whole
//     V row (K floats, K/4 x 16 B loads, all in flight at once), forms t = V*x, its avx-ordered self dot product
//     entirely in registers (no shuffles) and W*x, and parks {t[0..K), dot, w*x} in the warp's shared-memory tile.
//   phase 2 (in-order, light): the tile is read back transposed -- lane c accumulates sumVX[c] (and NFM's z[c])
//     over the features IN ORDER, every lane replays the scalar fm_pred chain -- so the per-sample arithmetic
//     sequence is exactly train_fm_algo.cpp:69-84.  (fm_pred -= 0.5*dot is formed in double there and rounded
//     to float; 0.5*dot is exact and a single double add/sub rounded to float equals the float operation
//     [53 >= 2*24+2 bits: innocuous double rounding], so the chain runs in fp32, bit-identically.)
template <int K, bool HAS_VAL, bool NFM>
__global__ void __launch_bounds__(256)
fm_forward_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                  const float* __restrict__ val, const float* __restrict__ label, const float* __restrict__ W,
                  const float* __restrict__ V, float* __restrict__ pred, float* __restrict__ sumvx,
                  float* __restrict__ z_out, float* __restrict__ wide_out, int64_t rb, int64_t re_arg, double* partial,
                  unsigned int* done, double* out_slot, int do_stats, const int64_t* __restrict__ hdr,
                  const float* __restrict__ quirk_sumvx, int64_t quirk_rows) {
    const int64_t re = hdr ? hdr[0] : re_arg;  // graph launches read the batch size from the slot header
    constexpr int STR = K + 4;     // tile row: t[0..K), dot, w*x, pad (16 B aligned, conflict-free strides)
    constexpr int NB = 64;         // features per pass (two 32-lane gathers in flight)
    extern __shared__ __align__(16) float fwd_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float* tile = fwd_smem + (size_t)wid * NB * STR;
    const int64_t r = rb + (int64_t)blockIdx.x * (blockDim.x >> 5) + wid;
    double loss = 0.0, correct = 0.0;
    if (r < re) {
        const int64_t b = row_ptr[r];
        const int n = (int)(row_ptr[r + 1] - b);
        float s = 0.f, z = 0.f, fm = 0.f;
        for (int base = 0; base < n; base += NB) {
            // ---- phase 1
            float t[2][K], wx[2];
            bool ok[2];
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const int i = base + u * 32 + lane;
                ok[u] = i < n;
                const uint32_t f = ok[u] ? __ldg(fid + b + i) : 0u;
                const float x = HAS_VAL ? (ok[u] ? __ldg(val + b + i) : 0.f) : 1.f;
                const float* row = V + (size_t)f * K;
                if (K % 4 == 0) {
#pragma unroll
                    for (int q = 0; q < K / 4; q++) {
                        const float4 v4 = ldg_f4(row + 4 * q);
                        t[u][4 * q] = v4.x; t[u][4 * q + 1] = v4.y; t[u][4 * q + 2] = v4.z; t[u][4 * q + 3] = v4.w;
                    }
                } else {
#pragma unroll
                    for (int q = 0; q < K; q++) t[u][q] = __ldg(row + q);
                }
                wx[u] = __ldg(W + f) * x;                       // W[fid] * X             train_fm_algo.cpp:74
                if (HAS_VAL) {
#pragma unroll
                    for (int q = 0; q < K; q++) t[u][q] = t[u][q] * x;   // avx_vecScale(V, tmp, X)   :76
                }
            }
#pragma unroll
            for (int u = 0; u < 2; u++) {
                if (!ok[u]) continue;
                float* dst = tile + (size_t)(u * 32 + lane) * STR;
                if (K % 4 == 0) {
#pragma unroll
                    for (int q = 0; q < K / 4; q++)
                        *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(t[u][4 * q], t[u][4 * q + 1], t[u][4 * q + 2], t[u][4 * q + 3]);
                } else {
#pragma unroll
                    for (int q = 0; q < K; q++) dst[q] = t[u][q];
                }
                dst[K] = NFM ? 0.f : avx_dot_regs<K>(t[u]);     // dot(tmp, tmp)          :78
                dst[K + 1] = wx[u];
            }
            __syncwarp();
            // ---- phase 2: features base .. base+cnt in order
            const int cnt = min(NB, n - base);
            const int col = lane < K ? lane : 0;
#pragma unroll 4
            for (int j = 0; j < cnt; j++) {
                const float* src = tile + (size_t)j * STR;
                const float tj = src[col];
                const float dot = src[K], w1 = src[K + 1];
                s = s + tj;                                     // sumVX += tmp           :77
                if (NFM) {
                    z = z + tj * (tj * -0.5f);                  // train_nfm_algo.cpp:87-91
                    fm = fm + w1;                               // wide part              train_nfm_algo.cpp:83
                } else {
                    fm = fm + w1;                               // fm_pred += W[fid] * X  :74
                    fm = fm - 0.5f * dot;                       // fm_pred -= 0.5 * dot   :78
                }
            }
            __syncwarp();
        }
        if (lane < K) sumvx[(size_t)r * K + lane] = s;
        if (NFM) {
            // z = z + sumVX * (sumVX * 0.5)    (train_nfm_algo.cpp:93-94)
            if (lane < K) z_out[(size_t)(r - rb) * K + lane] = z + s * (s * 0.5f);
            if (lane == 0) wide_out[r] = fm;
        } else {
            // avx_dotProduct(sumVX, sumVX, K) across lanes 0..K-1 in the reference's order, via the tile.
            // FM_Predict quirk (predict/fm_predict.cpp:31): the TRAINING sumVX row of the same index instead
            if (lane < K) tile[lane] = quirk_sumvx ? (r < quirk_rows ? quirk_sumvx[(size_t)r * K + lane] : 0.f) : s;
            __syncwarp();
            if (lane == 0) {
                float sv[K];
#pragma unroll
                for (int q = 0; q < K; q++) sv[q] = tile[q];
                const float dot = avx_dot_regs<K>(sv);
                fm = (float)((double)fm + 0.5 * (double)dot);  // :82
                const float pr = ref_sigmoid(fm);              // :84
                pred[r] = pr;
                if (do_stats) loss_terms(pr, label[r], loss, correct);
            }
        }
    }
    if (!NFM && do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

// ------------------------------------------------------------------------------------------------
// backward: scatter-add into the dense update_g (W part, V part) with vector REDs + touched marks
// ------------------------------------------------------------------------------------------------
// RW: the slot's row weights rw scale the head and the per-occurrence L2 terms
template <int LPR, int VEC, bool HAS_VAL, bool NFM, bool RW = false>
__global__ void __launch_bounds__(256)
fm_backward_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                   const float* __restrict__ val, const float* __restrict__ label, const float* __restrict__ W,
                   const float* __restrict__ V, int k, const float* __restrict__ pred,
                   const float* __restrict__ sumvx, const float* __restrict__ dz, float* __restrict__ gW,
                   float* __restrict__ gV, uint8_t* __restrict__ touched, float l2_arg, int64_t rb, int64_t re,
                   const float* __restrict__ rw) {
    constexpr int G = 32 / LPR;
    const int lane = threadIdx.x & 31;
    const int q = lane % LPR, g = lane / LPR;
    const int64_t r = rb + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= re) return;
    const bool qa = q * VEC < k;
    const int64_t b = row_ptr[r], e = row_ptr[r + 1];
    const float d = row_head<RW>(pred[r], label[r], rw, r);  // LogisticGradW: (pred - label) * x  (fm_algo_abst.h:159-161)
    const float l2 = row_l2<RW>(l2_arg, rw, r);
    float s[VEC], dzv[VEC];
#pragma unroll
    for (int c = 0; c < VEC; c++) {
        s[c] = qa ? sumvx[(size_t)r * k + q * VEC + c] : 0.f;
        dzv[c] = (NFM && qa) ? dz[(size_t)(r - rb) * k + q * VEC + c] : 0.f;
    }
    for (int64_t base = b; base < e; base += 32) {
        const int cnt = (int)min((int64_t)32, e - base);
        const uint32_t my_f = lane < cnt ? __ldg(fid + base + lane) : 0u;
        const float my_x = HAS_VAL ? (lane < cnt ? __ldg(val + base + lane) : 0.f) : 1.f;
        Vec<VEC> v[LPR];
        float w[LPR], x[LPR];
        uint32_t ff[LPR];
#pragma unroll
        for (int j = 0; j < LPR; j++) {
            const int idx = j * G + g;
            ff[j] = __shfl_sync(kFull, my_f, idx);
            x[j] = __shfl_sync(kFull, my_x, idx);
            const bool ok = idx < cnt;
            v[j] = load_row<VEC>(V + (size_t)ff[j] * k + q * VEC, ok && qa);
            w[j] = ok ? __ldg(W + ff[j]) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < LPR; j++) {
            const int idx = j * G + g;
            if (idx >= cnt) continue;
            const float gw = d * x[j] + l2 * w[j];  // train_fm_algo.cpp:108 / train_nfm_algo.cpp:135
            float gv[VEC];
#pragma unroll
            for (int c = 0; c < VEC; c++) {
                const float t = s[c] + v[j].a[c] * (-x[j]);  // sumVX - x*V  (:112-113 / nfm :152-153)
                if (NFM) gv[c] = t * (dzv[c] * x[j]) + v[j].a[c] * l2;  // train_nfm_algo.cpp:154-157
                else gv[c] = t * gw + v[j].a[c] * l2;                   // train_fm_algo.cpp:114-115
            }
            if (qa) {
                float* dst = gV + (size_t)ff[j] * k + q * VEC;
                if (VEC == 4) red_add_v4(dst, make_float4(gv[0], gv[1 % VEC], gv[2 % VEC], gv[3 % VEC]));
                else red_add_f32(dst, gv[0]);
            }
            if (q == 0) {
                red_add_f32(gW + ff[j], gw);  // *update_W(fid) += gradW  (:109)
                if (touched) touched[ff[j]] = 1;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
struct Shape { int lpr, vec; };
static bool pick_shape(int k, Shape& sh) {
    if (k % 4 == 0 && k <= 128 && (k / 4 & (k / 4 - 1)) == 0) { sh.vec = 4; sh.lpr = k / 4; return true; }
    if (k <= 32) { int l = 1; while (l < k) l <<= 1; sh.vec = 1; sh.lpr = l; return true; }
    return false;
}

// Coalesced variant for K % 8 == 0: LPR = K/4 lanes cover one V row with float4 loads (a 64 B row is ONE request of two
// fully used sectors instead of four scattered 16 B requests), so a warp gathers G = 32/LPR rows per load instruction.
// The avx-ordered self dot runs across the LPR lanes (chunk sums, then the hsum tree), the shared tile is
// FACTOR-major -- T[c][j], rows K and K+1 hold dot and w*x -- so that the in-order scan of phase 2 reads four
// features per LDS.128.  Same expression sequence as fm_forward_kernel; ~3x fewer LSU wavefronts per sample.
template <int K, bool HAS_VAL, bool NFM>
__global__ void __launch_bounds__(128, (K <= 16 ? 7 : 4))
fm_forward_coalesced_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid,
                            const float* __restrict__ val, const float* __restrict__ label, const float* __restrict__ W,
                            const float* __restrict__ V, float* __restrict__ pred, float* __restrict__ sumvx,
                            float* __restrict__ z_out, float* __restrict__ wide_out, int64_t rb, int64_t re_arg,
                            double* partial, unsigned int* done, double* out_slot, int do_stats,
                            const int64_t* __restrict__ hdr, const float* __restrict__ quirk_sumvx, int64_t quirk_rows) {
    static_assert(K % 8 == 0 && K <= 32, "coalesced forward: K in {8, 16, 24, 32}");
    const int64_t re = hdr ? hdr[0] : re_arg;
    constexpr int LPR = K / 4 > 4 ? 8 : K / 4;  // lanes per row: K/4, or 8 for K=24 (power of two >= K/4)
    constexpr int G = 32 / LPR;         // rows per gather instruction
    constexpr int NB = 64;              // features per pass
    constexpr int NIT = NB / G;         // gather iterations per pass
    constexpr int TS = NB + 4;          // tile row stride in floats (16 B aligned, conflict-free LDS.128)
    constexpr int NFULL = K / 8;
    extern __shared__ __align__(16) float fwd_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float* tile = fwd_smem + (size_t)wid * (K + 2) * TS;
    const int q = lane % LPR, g = lane / LPR;
    const bool qa = 4 * q < K;          // K = 24: lanes q = 6,7 idle
    const int64_t r = rb + (int64_t)blockIdx.x * (blockDim.x >> 5) + wid;
    double loss = 0.0, correct = 0.0;
    if (r < re) {
        const int64_t b = row_ptr[r];
        const int n = (int)(row_ptr[r + 1] - b);
        float s = 0.f, z = 0.f, fm = 0.f;
        for (int base = 0; base < n; base += NB) {
            // ---- phase 1: columns of this pass (2 coalesced loads), then NIT gathers of G rows each
            const int i0 = base + lane, i1 = base + 32 + lane;
            const uint32_t f0 = i0 < n ? __ldg(fid + b + i0) : 0u, f1 = i1 < n ? __ldg(fid + b + i1) : 0u;
            const float x0 = HAS_VAL ? (i0 < n ? __ldg(val + b + i0) : 0.f) : 1.f;
            const float x1 = HAS_VAL ? (i1 < n ? __ldg(val + b + i1) : 0.f) : 1.f;
            float4 v[NIT];
            float wv[NIT], xv[NIT];
#pragma unroll
            for (int it = 0; it < NIT; it++) {
                const int j = it * G + g;  // feature index within the pass
                const uint32_t f = __shfl_sync(kFull, j < 32 ? f0 : f1, j & 31);
                xv[it] = HAS_VAL ? __shfl_sync(kFull, j < 32 ? x0 : x1, j & 31) : 1.f;
                v[it] = qa ? ldg_f4_pinned(V + (size_t)f * K + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);  // f = 0 beyond n: masked
                wv[it] = q == 0 ? ldg_f32_pinned(W + f) : 0.f;
            }
#pragma unroll
            for (int it = 0; it < NIT; it++) {
                const int j = it * G + g;
                const bool ok = base + j < n;
                float t[4] = {v[it].x, v[it].y, v[it].z, v[it].w};
                if (HAS_VAL) {
#pragma unroll
                    for (int c = 0; c < 4; c++) t[c] = t[c] * xv[it];          // avx_vecScale(V, tmp, X)  :76
                }
                if (!ok) { t[0] = t[1] = t[2] = t[3] = 0.f; }
                float dot = 0.f;
                if (!NFM) {
                    // avx_dotProduct(tmp, tmp, K): lane q holds elements 4q..4q+3; chunk m = q/2, position (q%2)*4+c
                    float d[4];
#pragma unroll
                    for (int c = 0; c < 4; c++) d[c] = t[c] * t[c];
                    float p[4] = {d[0], d[1], d[2], d[3]};
#pragma unroll
                    for (int m = 1; m < NFULL; m++)
#pragma unroll
                        for (int c = 0; c < 4; c++) d[c] = d[c] + __shfl_down_sync(kFull, p[c], 2 * m, LPR);
                    float a[4];
#pragma unroll
                    for (int c = 0; c < 4; c++) a[c] = d[c] + __shfl_down_sync(kFull, d[c], 1, LPR);  // d_i + d_{i+4}
                    dot = (a[0] + a[2]) + (a[1] + a[3]);
                }
                if (ok && qa) {
#pragma unroll
                    for (int c = 0; c < 4; c++) tile[(4 * q + c) * TS + j] = t[c];
                }
                if (ok && q == 0) {
                    tile[K * TS + j] = dot;                                  // dot(tmp, tmp)            :78
                    tile[(K + 1) * TS + j] = wv[it] * xv[it];                // W[fid] * X               :74
                }
            }
            __syncwarp();
            // ---- phase 2: features base .. base+cnt in order, four per LDS.128
            const int cnt = min(NB, n - base);
            const int col = lane < K ? lane : 0;
            for (int j0 = 0; j0 < cnt; j0 += 4) {
                const float4 t4 = *reinterpret_cast<const float4*>(tile + col * TS + j0);
                const float4 d4 = *reinterpret_cast<const float4*>(tile + K * TS + j0);
                const float4 w4 = *reinterpret_cast<const float4*>(tile + (K + 1) * TS + j0);
                const float tt[4] = {t4.x, t4.y, t4.z, t4.w}, dd[4] = {d4.x, d4.y, d4.z, d4.w}, ww[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (j0 + u < cnt) {
                        s = s + tt[u];                                      // sumVX += tmp             :77
                        if (NFM) {
                            z = z + tt[u] * (tt[u] * -0.5f);                // train_nfm_algo.cpp:87-91
                            fm = fm + ww[u];
                        } else {
                            fm = fm + ww[u];                                // fm_pred += W[fid] * X    :74
                            fm = fm - 0.5f * dd[u];                         // fm_pred -= 0.5 * dot     :78
                        }
                    }
                }
            }
            __syncwarp();
        }
        if (lane < K) sumvx[(size_t)r * K + lane] = s;
        if (NFM) {
            if (lane < K) z_out[(size_t)(r - rb) * K + lane] = z + s * (s * 0.5f);
            if (lane == 0) wide_out[r] = fm;
        } else {
            if (lane < K) tile[lane] = quirk_sumvx ? (r < quirk_rows ? quirk_sumvx[(size_t)r * K + lane] : 0.f) : s;  // fm_predict.cpp:31
            __syncwarp();
            if (lane == 0) {
                float sv[K];
#pragma unroll
                for (int c = 0; c < K; c++) sv[c] = tile[c];
                const float dot = avx_dot_regs<K>(sv);
                fm = (float)((double)fm + 0.5 * (double)dot);  // :82
                const float pr = ref_sigmoid(fm);              // :84
                pred[r] = pr;
                if (do_stats) loss_terms(pr, label[r], loss, correct);
            }
        }
    }
    if (!NFM && do_stats) publish_stats(loss, correct, partial, done, out_slot, false);
}

template <int K>
static int fwd_go(lctr_ctx* c, Slot& s, bool nfm, int64_t rb, int64_t re, double* out_slot, int stats, const int64_t* hdr) {
    constexpr bool kCoalesced = (K % 8 == 0) && K <= 32;
    static const bool want_coalesced = !(getenv("LCTR_FWD_COALESCED") && atoi(getenv("LCTR_FWD_COALESCED")) == 0);
    const bool co = kCoalesced && want_coalesced;
    // coalesced kernel: 4 warps per CTA (its 8 row gathers per pass are all in flight: ~70 registers per thread, and
    // at batch 4096 / 132 SMs = 31 warps per SM every sample must be resident in ONE wave)
    const int wpb = co ? 4 : 8;
    const unsigned grid = (unsigned)((re - rb + wpb - 1) / wpb);
    const size_t smem = co ? (size_t)wpb * (K + 2) * 68 * sizeof(float) : (size_t)wpb * 64 * (K + 4) * sizeof(float);
    auto kern = by_flags([co](auto hv, auto nf) {
        return co ? fm_forward_coalesced_kernel<kCoalesced ? K : 8, hv, nf> : fm_forward_kernel<K, hv, nf>;
    }, s.has_val, nfm);
    return launch(c, {grid, (unsigned)wpb * 32, smem, c->stream}, kern, s.row_ptr, c->cfg.world > 1 ? s.ent_pslot : s.fid, s.val,
                  s.label, c->cW, c->cV, s.pred, s.sumvx, c->z, s.wide, rb, re, c->stat_partial, c->stat_done, out_slot, stats, hdr,
                  c->fwd_quirk_sumvx, c->fwd_quirk_rows);
}

int launch_fm_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm, bool stats) {
    return launch_fm_forward_ex(c, s, rb, re, nfm, stats, nullptr, nullptr);
}

// hdr != nullptr (graph capture): `re` is the grid-sizing upper bound, the kernel takes the row count from hdr[0]
int launch_fm_forward_ex(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm, bool stats, const int64_t* hdr,
                         double* out_slot_override) {
    const int k = (int)c->cfg.factor_cnt;
    const int64_t rows = re - rb;
    if (rows <= 0) return 0;
    double* out_slot = out_slot_override ? out_slot_override : c->stats + 2 * (c->step % kStatRing);
    const int st = stats ? 1 : 0;
    ProfScope prof(c, PROF_FM_FWD);
    // the factor count is a compile-time constant of the kernel (register-resident rows)
    using FwdK = Built<1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 16, 20, 24, 32>;
    if (!FwdK::has(k)) {
        set_error("factor_cnt=%d is not instantiated (built: 1-8, 10, 12, 16, 20, 24, 32)", k);
        return 1;
    }
    int rc = 0;
    static const int dbg_repeat = getenv("LCTR_DBG_FWD_REPEAT") ? atoi(getenv("LCTR_DBG_FWD_REPEAT")) : 1;
    for (int rep = 0; rep < dbg_repeat && !rc; rep++)
        rc = FwdK::pick(k, [&](auto K) { return fwd_go<K>(c, s, nfm, rb, re, out_slot, st, hdr); });
    return rc;
}

int launch_fm_backward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm) {
    Shape sh;
    const int k = (int)c->cfg.factor_cnt;
    LCTR_CHECK(pick_shape(k, sh), "factor_cnt=%d unsupported", k);
    const int64_t rows = re - rb;
    if (rows <= 0) return 0;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    ProfScope prof(c, PROF_FM_BWD_RED);
    auto kern = by_value<1, 2, 4, 8, 16, 32>(sh.lpr, [&](auto lpr) {
        return by_value<4, 1>(sh.vec, [&](auto vec) {
            return by_flags([&](auto hv, auto nf, auto rw) { return fm_backward_kernel<lpr, vec, hv, nf, rw>; }, s.has_val, nfm, s.has_rw);
        });
    });
    return launch(c, {grid, 256, 0, c->stream}, kern, s.row_ptr, c->cfg.world > 1 ? s.ent_pslot : s.fid, s.val, s.label, c->cW,
                  c->cV, k, s.pred, s.sumvx, c->dz, c->cgW, c->cgV, c->cfg.world > 1 ? nullptr : c->touched.get(), c->cfg.l2_reg, rb,
                  re, row_weights(s));
}


// ------------------------------------------------------------------------------------------------
// deterministic backward + fused updater over the feature-major (CSC) view
// ------------------------------------------------------------------------------------------------
// One group of LR lanes per segment (= one fid of the row block); lane c owns factor c.  The fid's
// entries are visited in ascending row order and accumulated with the reference's exact expression
// sequence (train_fm_algo.cpp:108-115 / train_nfm_algo.cpp:131-157), starting from the zeroed update_g,
// so the summed gradient equals the reference's canonical single-thread result bit for bit (given equal
// inputs).  The updater then runs on the register-resident gradient: no update_g traffic, no atomics,
// no touched map.
// RW: the slot's row weights rw scale each entry's head and L2 terms by its row's weight
template <int LR, bool HAS_VAL, bool NFM, bool RW = false>
__global__ void __launch_bounds__(256)
fm_backward_csc_kernel(const int64_t* __restrict__ seg_ptr, const uint32_t* __restrict__ seg_fid,
                       const uint32_t* __restrict__ ent_row, const float* __restrict__ ent_x, int64_t seg_begin,
                       int64_t seg_end, const float* __restrict__ label, const float* __restrict__ pred,
                       const float* __restrict__ sumvx, const float* __restrict__ dz, int64_t rb, float* __restrict__ W,
                       float* __restrict__ V, float* __restrict__ s1W, float* __restrict__ s1V, float* __restrict__ s2W,
                       float* __restrict__ s2V, int k, float l2, OptParams P, const float* __restrict__ rw) {
    constexpr int SPW = 32 / LR;
    const int lane = threadIdx.x & 31;
    const int c = lane % LR, grp = lane / LR;
    const int64_t seg = seg_begin + ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * SPW + grp;
    const bool sv = seg < seg_end, act = c < k;
    const int64_t eb = sv ? seg_ptr[seg] : 0;
    const int n = sv ? (int)(seg_ptr[seg + 1] - eb) : 0;
    int nmax = n;
#pragma unroll
    for (int o = LR; o < 32; o <<= 1) nmax = max(nmax, __shfl_xor_sync(kFull, nmax, o));
    const uint32_t f = sv ? seg_fid[seg] : 0u;
    const float w = sv ? W[f] : 0.f;
    const float v = (sv && act) ? V[(size_t)f * k + c] : 0.f;
    float u = 0.f, gwsum = 0.f;
    for (int base = 0; base < nmax; base += LR) {
        const int cnt = n - base;
        const uint32_t my_row = c < cnt ? __ldg(ent_row + eb + base + c) : 0u;
        const float my_x = HAS_VAL ? (c < cnt ? __ldg(ent_x + eb + base + c) : 0.f) : 1.f;
        float sv_[LR], d_[LR], dz_[LR], l2_[LR];
#pragma unroll
        for (int j = 0; j < LR; j++) {
            const uint32_t row = __shfl_sync(kFull, my_row, j, LR);
            const bool ok = j < cnt;
            sv_[j] = (ok && act) ? __ldg(sumvx + (size_t)row * k + c) : 0.f;
            d_[j] = ok ? row_head<RW>(__ldg(pred + row), __ldg(label + row), rw, row) : 0.f;  // LogisticGradW  fm_algo_abst.h:159-161
            if (RW) l2_[j] = ok ? row_l2<true>(l2, rw, row) : 0.f;
            dz_[j] = (NFM && ok && act) ? __ldg(dz + (size_t)(row - rb) * k + c) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < LR; j++) {
            if (j >= nmax - base) break;  // warp-uniform
            const float x = __shfl_sync(kFull, my_x, j, LR);
            if (j < cnt) {
                const float l2j = RW ? l2_[j] : l2;
                const float gw = d_[j] * x + l2j * w;        // train_fm_algo.cpp:108 / train_nfm_algo.cpp:135
                gwsum = gwsum + gw;                          // *update_W(fid) += gradW            :109
                const float t = sv_[j] + v * (-x);           // avx_vecScalerAdd(sumVX, V, tmp, -x) :112-113
                if (NFM) u = u + t * (dz_[j] * x);           // train_nfm_algo.cpp:154-156
                else u = u + t * gw;                         // avx_vecScalerAdd(ptr, tmp, ptr, gradW) :114
                u = u + v * l2j;                             // avx_vecScalerAdd(ptr, V, ptr, L2)      :115
            }
        }
    }
    if (!sv) return;
    const bool two = opt_two_states(P.opt);
    if (c == 0) {
        float ww = w, a = s1W[f], b2 = two ? s2W[f] : 0.f;
        update_one(P, P.corrW, ww, gwsum, a, b2);
        W[f] = ww; s1W[f] = a;
        if (two) s2W[f] = b2;
    }
    if (act) {
        const size_t o = (size_t)f * k + c;
        float vv = v, a = s1V[o], b2 = two ? s2V[o] : 0.f;
        update_one(P, P.corrV, vv, u, a, b2);
        V[o] = vv; s1V[o] = a;
        if (two) s2V[o] = b2;
    }
}

int launch_fm_backward_csc(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm) {
    const int k = (int)c->cfg.factor_cnt;
    LCTR_CHECK(k <= 32, "factor_cnt=%d unsupported by the feature-major backward (need k <= 32)", k);
    LCTR_CHECK(s.csc_block > 0 && !s.h_blk_seg_ptr.empty(), "deterministic step on a slot uploaded without the CSC view");
    LCTR_CHECK(rb % s.csc_block == 0 && (re == rb + s.csc_block || re == s.rows) && re - rb <= s.csc_block,
               "deterministic train_step rows [%lld,%lld) do not match the slot's row blocks of %lld",
               (long long)rb, (long long)re, (long long)s.csc_block);
    const int64_t bi = rb / s.csc_block;
    const int64_t sb = s.h_blk_seg_ptr[bi], se = s.h_blk_seg_ptr[bi + 1];
    if (se <= sb) return 0;
    const OptParams P = make_opt_params(c, re - rb);
    int lr = 4;
    while (lr < k) lr <<= 1;
    const int segs_per_cta = 8 * (32 / lr);
    const unsigned grid = (unsigned)((se - sb + segs_per_cta - 1) / segs_per_cta);
    ProfScope prof(c, PROF_FM_BWD_CSC);
    auto kern = by_value<4, 8, 16, 32>(lr, [&](auto LR) {
        return by_flags([&](auto hv, auto nf, auto rw) { return fm_backward_csc_kernel<LR, hv, nf, rw>; }, s.has_val, nfm, s.has_rw);
    });
    return launch(c, {grid, 256, 0, c->stream}, kern, s.seg_ptr, s.seg_fid, s.ent_row, s.ent_x, sb, se, s.label, s.pred, s.sumvx,
                  c->dz, rb, c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V, k, c->cfg.l2_reg, P, row_weights(s));
}

// FM_Predict quirk mode (predict/fm_predict.cpp:20-33): pred = sum w x - 0.5 sum|vx|^2 + 0.5|sumVX_train[rid]|^2, evaluated
// by the in-order forward kernel (same arithmetic sequence as the reference's loop) with the training rows' sumVX
// substituted in the last term.
int launch_predict_quirk(lctr_ctx* c, Slot& s, Slot& train) {
    if (s.rows <= 0) return 0;
    c->fwd_quirk_sumvx = train.sumvx;
    c->fwd_quirk_rows = train.rows;
    const int rc = launch_fm_forward(c, s, 0, s.rows, false, false);
    c->fwd_quirk_sumvx = nullptr;
    c->fwd_quirk_rows = 0;
    return rc;
}

}  // namespace lctr
