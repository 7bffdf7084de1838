// lightctr_b200/csrc/mlp_bf16.cu -- NFM / Wide&Deep dense layers on the tensor cores (mlp_precision = LCTR_MLP_BF16).
//
// Same Fully_Conn_Layer chain as mlp.cu (train/layer/fullyconnLayer.h:80-197), but organised for the machine instead of
// for bit parity: ONE kernel runs forward, loss and backward for a tile of TM samples with every activation resident
// in shared memory, because the whole chain is sample-local except the reduction of dW over samples.
//   * weights (bf16 copies of the fp32 masters, [out][in]) and the tile's activations live in shared memory
//     (C4: 95 KB + 124 KB), rows padded by 16 B so that every ldmatrix phase is bank-conflict free;
//   * warp w owns samples [16w, 16w+16): the forward GEMMs and the dX GEMMs are warp-local (no CTA barrier between
//     layers); delta_{l-1} overwrites a_{l-1} in place;
//   * dW_l = delta_l^T . a_{l-1} (K = the TM samples) is a CTA-level GEMM whose operands are the SAME shared-memory
//     tiles read through ldmatrix.trans; db_l rides along as one extra n-tile against a constant-one B fragment;
//     the fp32 results go to the dense-gradient buffer with vector REDs (fire and forget);
//   * operands bf16, accumulation fp32 (mma.sync.m16n8k16), masters + Adagrad state fp32 (one fused update kernel
//     that also refreshes the bf16 copies).
// The arithmetic differs from the reference's fp32 AVX order by bf16 operand rounding, so this mode is checked
// against a rounding-point-exact emulation in tests/test_mlp_bf16_gpu.py, not against the 1e-5 trajectory bar.
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "mlp_umma.cuh"

namespace lctr {

constexpr int kMaxDense = LCTR_MAX_LAYERS + 1;
constexpr int kPad = 8;  // bf16 elements of padding per shared-memory row (16 B)

struct MlpDev {
    int nl;  // layers including the linear output layer (out == 1)
    int act, has_mask;
    int in[kMaxDense], out[kMaxDense];
    const __nv_bfloat16* w16[kMaxDense];  // hidden layers: bf16 [out][in]
    const float* w32_last;                // output layer weights, fp32 [in]
    const float* bias[kMaxDense];
    const float* mask[kMaxDense];
    float* dw[kMaxDense];
    float* db[kMaxDense];
    int x_off[kMaxDense];  // byte offset of X_l = input of layer l ([TM][in_l + kPad] bf16); X_0 = z
    int w_off[kMaxDense];  // byte offset of W_l ([out_l][in_l + kPad] bf16), hidden layers
    int wl_off, bias_off, mask_off;  // fp32 w_last[in], fp32 bias (hidden, concatenated), bf16 mask (hidden, concatenated)
    int vec_off[kMaxDense];          // element offset of layer l inside the bias / mask arrays
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}
__device__ __forceinline__ float act_fwd(float v, int act) {
    if (act == LCTR_ACT_SIGMOID) return v < -16.f ? 1e-7f : (v > 16.f ? 0.99999988f : __fdividef(1.0f, 1.0f + __expf(-v)));
    const float t1 = __expf(v), t2 = __expf(-v);
    return fabsf(v) > 15.f ? copysignf(1.f, v) : __fdividef(t1 - t2, t1 + t2);
}
__device__ __forceinline__ float act_bwd(float fo, int act) {  // activations.h:85-90,139-143
    return act == LCTR_ACT_SIGMOID ? fo * (1.0f - fo) : 1.0f - fo * fo;
}
__device__ __forceinline__ float clip15(float v) { return fminf(fmaxf(v, -15.f), 15.f); }

// Warp-level C[16 x N] = A[16 x K] . B, A rows in shared memory (k contiguous).  B_KMAJOR: B given as [n][k] rows
// (forward: the weight matrix as stored); otherwise as [k][n] rows (dX: the same weight tile, read transposed).
// N is processed in chunks of NC columns so that the accumulators stay in registers for any layer width.
template <int NC, bool B_KMAJOR, bool MASK_A, class Epi>
__device__ __forceinline__ void warp_gemm(uint32_t a_base, int a_stride, int K, uint32_t b_base, int b_stride, int N,
                                          const __nv_bfloat16* mask16, Epi epi) {
    const int lane = threadIdx.x & 31, mi = lane >> 3, t = lane & 3;
    const uint32_t a_lane = a_base + (lane & 15) * a_stride + (lane >> 4) * 16;
    for (int n0 = 0; n0 < N; n0 += NC) {
        float acc[NC / 8][4];
#pragma unroll
        for (int i = 0; i < NC / 8; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
        for (int k0 = 0; k0 < K; k0 += 16) {
            uint32_t a[4];
            ldsm_x4(a_lane + k0 * 2, a);
            if (MASK_A) {  // dX_i = sum_j W[j,i] mask_j delta_j (fullyconnLayer.h:139-147)
                const uint32_t m_lo = *reinterpret_cast<const uint32_t*>(mask16 + k0 + 2 * t);
                const uint32_t m_hi = *reinterpret_cast<const uint32_t*>(mask16 + k0 + 2 * t + 8);
                auto mul = [](uint32_t x, uint32_t m) {
                    __nv_bfloat162 r = __hmul2(*reinterpret_cast<__nv_bfloat162*>(&x), *reinterpret_cast<__nv_bfloat162*>(&m));
                    return *reinterpret_cast<uint32_t*>(&r);
                };
                a[0] = mul(a[0], m_lo); a[1] = mul(a[1], m_lo); a[2] = mul(a[2], m_hi); a[3] = mul(a[3], m_hi);
            }
#pragma unroll
            for (int j = 0; j < NC / 16; j++) {
                uint32_t b[4];
                if (B_KMAJOR)
                    ldsm_x4(b_base + (n0 + j * 16 + (mi >> 1) * 8 + (lane & 7)) * b_stride + (k0 + (mi & 1) * 8) * 2, b);
                else
                    ldsm_x4_t(b_base + (k0 + (mi & 1) * 8 + (lane & 7)) * b_stride + (n0 + j * 16 + (mi >> 1) * 8) * 2, b);
                mma_bf16(acc[2 * j], a, b[0], b[1]);
                mma_bf16(acc[2 * j + 1], a, b[2], b[3]);
            }
        }
        epi(n0, acc);
    }
}

// dW tile: C[16 x NC] = A^T . B with A = delta[TM][out] (columns j0..j0+16), B = x[TM][in] (columns i0..i0+NC), K = TM.
template <int NC, int TM>
__device__ __forceinline__ void warp_gemm_tn(uint32_t d_base, int d_stride, int j0, uint32_t x_base, int x_stride, int i0,
                                             float (&acc)[NC / 8][4], float (&accb)[4], bool with_bias) {
    const int lane = threadIdx.x & 31, mi = lane >> 3;
#pragma unroll
    for (int i = 0; i < NC / 8; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    accb[0] = accb[1] = accb[2] = accb[3] = 0.f;
#pragma unroll 2
    for (int s0 = 0; s0 < TM; s0 += 16) {
        uint32_t a[4];
        ldsm_x4_t(d_base + (s0 + (mi >> 1) * 8 + (lane & 7)) * d_stride + (j0 + (mi & 1) * 8) * 2, a);
#pragma unroll
        for (int j = 0; j < NC / 16; j++) {
            uint32_t b[4];
            ldsm_x4_t(x_base + (s0 + (mi & 1) * 8 + (lane & 7)) * x_stride + (i0 + j * 16 + (mi >> 1) * 8) * 2, b);
            mma_bf16(acc[2 * j], a, b[0], b[1]);
            mma_bf16(acc[2 * j + 1], a, b[2], b[3]);
        }
        if (with_bias) mma_bf16(accb, a, 0x3F803F80u, 0x3F803F80u);  // B == 1: column sums of delta (biasDelta, :179)
    }
}

// TRAIN = false: the forward-only instance of lctr_score -- the same staging, forward and output layer, then the pCTR
// alone: no labels, loss, statistics, deltas or dW / db (dz, label and the statistics arguments are unused).  RW: the output
// delta is the clip of w (p - y) with the slot's row weights rw
template <int TM, bool TRAIN, bool RW = false>
__global__ void __launch_bounds__(TM * 2, 1)
nfm_mlp_fused_kernel(MlpDev P, const float* __restrict__ z, float* __restrict__ dz, const float* __restrict__ wide,
                     const float* __restrict__ label, float* __restrict__ pred, int64_t rb, int B, double* partial,
                     unsigned int* done, double* out_slot, const float* __restrict__ rw) {
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = lane >> 2, t = lane & 3;
    constexpr int NT = TM * 2, NW = TM / 16;
    const int nl = P.nl, nh = nl - 1;
    const int row0 = blockIdx.x * TM;
    const int valid = min(TM, B - row0);
    float* s_wl = reinterpret_cast<float*>(smem + P.wl_off);
    float* s_bias = reinterpret_cast<float*>(smem + P.bias_off);
    __nv_bfloat16* s_mask = reinterpret_cast<__nv_bfloat16*>(smem + P.mask_off);

    // ---- stage weights (cp.async, 16 B chunks), small vectors and the z tile
    for (int l = 0; l < nh; l++) {
        const int chunks = P.in[l] / 8, stride = (P.in[l] + kPad) * 2;
        const __nv_bfloat16* src = P.w16[l];
        for (int idx = tid; idx < P.out[l] * chunks; idx += NT) {
            const int r = idx / chunks, ch = idx - r * chunks;
            const uint32_t dst = sbase + P.w_off[l] + r * stride + ch * 16;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + (size_t)r * P.in[l] + ch * 8));
        }
        for (int j = tid; j < P.out[l]; j += NT) {
            s_bias[P.vec_off[l] + j] = P.bias[l][j];
            s_mask[P.vec_off[l] + j] = __float2bfloat16(P.mask[l][j]);
        }
    }
    asm volatile("cp.async.commit_group;");
    for (int i = tid; i < P.in[nh]; i += NT) s_wl[i] = P.w32_last[i];
    {
        const int k = P.in[0], q4 = k / 4, stride = (k + kPad) * 2;
        for (int idx = tid; idx < TM * q4; idx += NT) {
            const int r = idx / q4, c4 = idx - r * q4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < valid) v = *reinterpret_cast<const float4*>(z + (size_t)(row0 + r) * k + c4 * 4);
            uint2 u = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
            *reinterpret_cast<uint2*>(smem + P.x_off[0] + r * stride + c4 * 8) = u;
        }
    }
    asm volatile("cp.async.wait_group 0;");
    __syncthreads();

    const int m0 = wid * 16;
    // ---- forward through the hidden layers (fullyconnLayer.h:80-118); warp-local
    for (int l = 0; l < nh; l++) {
        const int K = P.in[l], N = P.out[l];
        const int xs = (K + kPad) * 2, ys = (N + kPad) * 2;
        unsigned char* y = smem + P.x_off[l + 1];
        const float* bias = s_bias + P.vec_off[l];
        const __nv_bfloat16* mk = s_mask + P.vec_off[l];
        auto run = [&](auto nc_tag) {
            constexpr int NC = decltype(nc_tag)::value;
            warp_gemm<NC, true, false>(sbase + P.x_off[l] + m0 * xs, xs, K, sbase + P.w_off[l], xs, N, nullptr,
                [&](int n0, float (&acc)[NC / 8][4]) {
#pragma unroll
                    for (int nt = 0; nt < NC / 8; nt++) {
                        const int col = n0 + nt * 8 + 2 * t;
                        const float b0 = bias[col], b1 = bias[col + 1];
                        float v0 = acc[nt][0] + b0, v1 = acc[nt][1] + b1, v2 = acc[nt][2] + b0, v3 = acc[nt][3] + b1;
                        if (P.has_mask) {  // masked neurons: pre-activation forced to 0, activation still applied (:96-99,110-113)
                            if (__bfloat162float(mk[col]) == 0.f) v0 = v2 = 0.f;
                            if (__bfloat162float(mk[col + 1]) == 0.f) v1 = v3 = 0.f;
                        }
                        *reinterpret_cast<uint32_t*>(y + (m0 + g) * ys + col * 2) = pack_bf16(act_fwd(v0, P.act), act_fwd(v1, P.act));
                        *reinterpret_cast<uint32_t*>(y + (m0 + g + 8) * ys + col * 2) = pack_bf16(act_fwd(v2, P.act), act_fwd(v3, P.act));
                    }
                });
        };
        if (N % 64 == 0) run(std::integral_constant<int, 64>{}); else run(std::integral_constant<int, 16>{});
        __syncwarp();
    }

    // ---- output layer (linear, out = 1), loss, delta_L, its dW/db, and delta of the last hidden layer in place
    double loss = 0.0, correct = 0.0;
    {
        const int K = P.in[nh], xs = (K + kPad) * 2;
        unsigned char* x = smem + P.x_off[nh];
        const float b_last = P.bias[nh][0];
        float dwl[4][2];  // lane owns columns 2*lane + 64*q, q < 4 (in <= 256)
#pragma unroll
        for (int q = 0; q < 4; q++) dwl[q][0] = dwl[q][1] = 0.f;
        float dbl = 0.f;
        for (int r = 0; r < 16; r++) {
            const int row = m0 + r;
            float part = 0.f;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int c = 2 * lane + 64 * q;
                if (c < K) {
                    const float2 a = unpack_bf16(*reinterpret_cast<const uint32_t*>(x + row * xs + c * 2));
                    part += a.x * s_wl[c] + a.y * s_wl[c + 1];
                }
            }
            const float o = warp_sum(part) + b_last;
            float d3 = 0.f;
            if (row < valid) {
                const int64_t gi = rb + row0 + row;
                const float p = ref_sigmoid(wide[gi] + o);  // train_nfm_algo.cpp:101-116
                if (!TRAIN) {
                    if (lane == 0) pred[gi] = p;
                    continue;
                }
                const float yv = label[gi];
                if (lane == 0) {
                    pred[gi] = p;
                    double l1, c1;
                    loss_terms(p, yv, l1, c1);
                    loss += l1; correct += c1;
                }
                d3 = clip15(row_head<RW>(p, yv, rw, gi));
            }
            if (!TRAIN) continue;
            dbl += d3;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int c = 2 * lane + 64 * q;
                if (c < K) {
                    uint32_t* px = reinterpret_cast<uint32_t*>(x + row * xs + c * 2);
                    const float2 a = unpack_bf16(*px);
                    dwl[q][0] += d3 * a.x;  // weightDelta of the output layer (:165-178)
                    dwl[q][1] += d3 * a.y;
                    // no mask on the output layer's dX (:139-147 with has_next false); previous activation' (:153-156)
                    const float e0 = clip15(d3 * s_wl[c] * act_bwd(a.x, P.act));
                    const float e1 = clip15(d3 * s_wl[c + 1] * act_bwd(a.y, P.act));
                    *px = pack_bf16(e0, e1);
                }
            }
        }
        if (TRAIN) {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int c = 2 * lane + 64 * q;
                if (c < K) red_add_v2(P.dw[nh] + c, dwl[q][0], dwl[q][1]);
            }
            if (lane == 0) atomicAdd(P.db[nh], dbl);
        }
    }

    // ---- backward through the hidden layers (fullyconnLayer.h:120-180)
    for (int l = nh - 1; TRAIN && l >= 0; l--) {
        const int K = P.in[l], N = P.out[l];
        const int xs = (K + kPad) * 2, ds = (N + kPad) * 2;
        const uint32_t d_base = sbase + P.x_off[l + 1], x_base = sbase + P.x_off[l];
        __syncthreads();  // every warp's delta_l is in place
        {                 // dW_l += delta_l^T . x_l ; db_l += column sums (unmasked delta, :165-179)
            auto run = [&](auto nc_tag) {
                constexpr int NC = decltype(nc_tag)::value;
                const int nchunks = K / NC, items = (N / 16) * nchunks;
                for (int it = wid; it < items; it += NW) {
                    const int mt = it / nchunks, nc = it - mt * nchunks;
                    float acc[NC / 8][4], accb[4];
                    warp_gemm_tn<NC, TM>(d_base, ds, mt * 16, x_base, xs, nc * NC, acc, accb, nc == 0);
                    float* dw0 = P.dw[l] + (size_t)(mt * 16 + g) * K + nc * NC + 2 * t;
                    float* dw1 = dw0 + (size_t)8 * K;
#pragma unroll
                    for (int nt = 0; nt < NC / 8; nt++) {
                        red_add_v2(dw0 + nt * 8, acc[nt][0], acc[nt][1]);
                        red_add_v2(dw1 + nt * 8, acc[nt][2], acc[nt][3]);
                    }
                    if (nc == 0 && t == 0) {
                        atomicAdd(P.db[l] + mt * 16 + g, accb[0]);
                        atomicAdd(P.db[l] + mt * 16 + g + 8, accb[2]);
                    }
                }
            };
            if (K % 64 == 0) run(std::integral_constant<int, 64>{}); else run(std::integral_constant<int, 16>{});
        }
        __syncthreads();  // x_l is overwritten below
        {                 // dX_l = (mask .* delta_l) . W_l, then the previous activation' (:139-156); warp-local rows
            unsigned char* xl = smem + P.x_off[l];
            const __nv_bfloat16* mk = s_mask + P.vec_off[l];
            auto run = [&](auto nc_tag, auto mask_tag) {
                constexpr int NC = decltype(nc_tag)::value;
                constexpr bool MA = decltype(mask_tag)::value;
                warp_gemm<NC, false, MA>(d_base + m0 * ds, ds, N, sbase + P.w_off[l], xs, K, mk,
                    [&](int n0, float (&acc)[NC / 8][4]) {
#pragma unroll
                        for (int nt = 0; nt < NC / 8; nt++) {
                            const int col = n0 + nt * 8 + 2 * t;
                            if (l > 0) {
                                uint32_t* p0 = reinterpret_cast<uint32_t*>(xl + (m0 + g) * xs + col * 2);
                                uint32_t* p1 = reinterpret_cast<uint32_t*>(xl + (m0 + g + 8) * xs + col * 2);
                                const float2 a0 = unpack_bf16(*p0), a1 = unpack_bf16(*p1);
                                *p0 = pack_bf16(clip15(acc[nt][0] * act_bwd(a0.x, P.act)), clip15(acc[nt][1] * act_bwd(a0.y, P.act)));
                                *p1 = pack_bf16(clip15(acc[nt][2] * act_bwd(a1.x, P.act)), clip15(acc[nt][3] * act_bwd(a1.y, P.act)));
                            } else {
                                if (m0 + g < valid)
                                    *reinterpret_cast<float2*>(dz + (size_t)(row0 + m0 + g) * K + col) = make_float2(acc[nt][0], acc[nt][1]);
                                if (m0 + g + 8 < valid)
                                    *reinterpret_cast<float2*>(dz + (size_t)(row0 + m0 + g + 8) * K + col) = make_float2(acc[nt][2], acc[nt][3]);
                            }
                        }
                    });
            };
            if (K % 64 == 0) {
                if (P.has_mask) run(std::integral_constant<int, 64>{}, std::true_type{});
                else run(std::integral_constant<int, 64>{}, std::false_type{});
            } else {
                if (P.has_mask) run(std::integral_constant<int, 16>{}, std::true_type{});
                else run(std::integral_constant<int, 16>{}, std::false_type{});
            }
        }
    }
    if (TRAIN) publish_stats(loss, correct, partial, done, out_slot, false);
}

// fp32 -> bf16 copy of one weight matrix
__global__ void to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, __nv_bfloat16* __restrict__ dst_tiled,
                               int in, int out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const __nv_bfloat16 v = __float2bfloat16(src[i]);
    dst[i] = v;
    if (dst_tiled) dst_tiled[umma::tiled_index(i, in, out)] = v;
}

// AdagradUpdater_Num::update (gradientUpdater.h:139-150) over every dense segment in ONE launch; the gradient buffer is
// the fused [dW0, db0, dW1, db1, ...] array (fullyconnLayer.h:69-75), so segment s of the buffer maps to (w,acc)[s].
struct DenseSegs {
    int n;
    size_t off[2 * kMaxDense + 1];
    float* w[2 * kMaxDense];
    float* acc[2 * kMaxDense];
    __nv_bfloat16* w16[2 * kMaxDense];
    __nv_bfloat16* w16t[2 * kMaxDense];  // chunk-major copy (mlp_umma.cu), or null
    int in[2 * kMaxDense], out[2 * kMaxDense];
};
__global__ void adagrad_dense_all_kernel(DenseSegs S, float* __restrict__ g, float invB, float lr) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    cudaTriggerProgrammaticLaunchCompletion();  // the NFM embedding backward behind this kernel
    int s = 0;
    if (i < S.off[S.n]) while (i >= S.off[s + 1]) s++;
    cudaGridDependencySynchronize();            // the dense kernel in front has completed: its dW / db sums are final
    if (i >= S.off[S.n]) return;
    const size_t j = i - S.off[s];
    const float g1 = g[i] * invB;
    if (g1 != 0.f) {
        const float a = S.acc[s][j] + g1 * g1;
        S.acc[s][j] = a;
        const float wn = (float)((double)S.w[s][j] - (double)(lr * g1) / sqrt((double)a + 1e-7));
        S.w[s][j] = wn;
        if (S.w16[s]) S.w16[s][j] = __float2bfloat16(wn);
        if (S.w16t[s]) S.w16t[s][umma::tiled_index(j, S.in[s], S.out[s])] = __float2bfloat16(wn);
    }
    g[i] = 0.f;
}

static size_t bf16_layout(lctr_ctx* c, int TM, MlpDev& P) {
    const int nl = c->n_layers, nh = nl - 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 15) & ~(size_t)15; return (int)o; };
    int voff = 0;
    for (int l = 0; l < nl; l++) {
        P.in[l] = c->layers[l].in; P.out[l] = c->layers[l].out;
        P.x_off[l] = take((size_t)TM * (P.in[l] + kPad) * 2);
    }
    for (int l = 0; l < nh; l++) {
        P.w_off[l] = take((size_t)P.out[l] * (P.in[l] + kPad) * 2);
        P.vec_off[l] = voff; voff += P.out[l];
    }
    P.wl_off = take((size_t)P.in[nh] * 4);
    P.bias_off = take((size_t)voff * 4);
    P.mask_off = take((size_t)voff * 2);
    return off;
}

int mlp_bf16_prepare(lctr_ctx* c) {
    const int nl = c->n_layers, nh = nl - 1;
    LCTR_CHECK(nh >= 1 && c->layers[nh].out == 1, "bf16 MLP: expects hidden layers + a 1-wide output layer");
    for (int l = 0; l < nl; l++) {
        LCTR_CHECK(c->layers[l].in % 16 == 0 && c->layers[l].in <= 512,
                   "bf16 MLP: layer %d input width %d must be a multiple of 16 (<= 512)", l, c->layers[l].in);
        if (l < nh && !c->layers[l].w16) {
            if (c->layers[l].w16.alloc((size_t)c->layers[l].out * c->layers[l].in) ||
                c->layers[l].w16t.alloc((size_t)c->layers[l].out * c->layers[l].in))
                return 1;
        }
    }
    c->mlp_umma = mlp_umma_supported(c) ? 1 : 0;
    if (c->mlp_umma && mlp_umma_prepare(c)) return 1;
    LCTR_CHECK(c->layers[nh].in <= 256, "bf16 MLP: last hidden layer wider than 256");
    MlpDev P;
    size_t need = bf16_layout(c, 128, P);
    c->mlp_tm = 128;
    if (need > 227 * 1024 - 1024) { need = bf16_layout(c, 64, P); c->mlp_tm = 64; }
    LCTR_CHECK(need <= 227 * 1024 - 1024, "bf16 MLP: layers need %zu B of shared memory per CTA (max %d)", need, 227 * 1024 - 1024);
    c->mlp_smem = need;
    return 0;
}

int mlp_bf16_refresh(lctr_ctx* c, int layer) {
    MlpLayer& L = c->layers[layer];
    if (!L.w16) return 0;
    const size_t n = (size_t)L.out * L.in;
    return launch(c, {(unsigned)((n + 255) / 256), 256, 0, c->stream}, to_bf16_kernel, L.w, L.w16, L.w16t, L.in, L.out, n);
}

// the dense chain on the B rows staged in c->z (rows [rb, rb + B) of the slot): the wgmma kernel (mlp_umma.cu) or, with a
// dropout mask or a shape it does not take, the mma.sync kernel.  train: forward, loss and backward of a step; otherwise
// the forward-only instances, which write the rows' pred alone.
static int launch_mlp_bf16_kernel(lctr_ctx* c, Slot& s, int64_t rb, int B, bool train) {
    const int nl = c->n_layers, nh = nl - 1;
    double* out_slot = c->stats + 2 * (c->step % kStatRing);
    if (c->mlp_umma && !c->mlp_has_mask) return launch_mlp_umma(c, s, rb, B, out_slot, train);
    MlpDev P;
    bf16_layout(c, c->mlp_tm, P);
    P.nl = nl; P.act = c->cfg.activation; P.has_mask = c->mlp_has_mask;
    for (int l = 0; l < nl; l++) {
        MlpLayer& L = c->layers[l];
        P.w16[l] = L.w16; P.bias[l] = L.b; P.mask[l] = L.mask; P.dw[l] = L.dw; P.db[l] = L.db;
    }
    P.w32_last = c->layers[nh].w;
    const unsigned grid = (unsigned)((B + c->mlp_tm - 1) / c->mlp_tm);
    const bool t128 = c->mlp_tm == 128;
    auto kern = by_flags([](auto t, auto tr, auto rw) { return nfm_mlp_fused_kernel<t ? 128 : 64, tr, tr && rw>; }, t128, train, s.has_rw);
    return launch(c, {grid, t128 ? 256u : 128u, c->mlp_smem, c->stream}, kern, P, c->z, c->dz, s.wide, s.label, s.pred, rb, B,
                  c->stat_partial, c->stat_done, out_slot, row_weights(s));
}

int launch_mlp_bf16_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    if (re - rb <= 0) return 0;
    ProfScope prof(c, PROF_MLP);
    return launch_mlp_bf16_kernel(c, s, rb, (int)(re - rb), false);
}

int launch_nfm_mlp_bf16(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int64_t rows_divisor) {
    const int B = (int)(re - rb);
    const int nl = c->n_layers;
    ProfScope prof(c, PROF_MLP);
    // B == 0 (a rank's empty share on several GPUs): no rows, no gradient; the rank still joins the all-reduce and the
    // replicated updater below
    if (B > 0 && launch_mlp_bf16_kernel(c, s, rb, B, true)) return 1;
    if (mlp_sync_dense_grad(c)) return 1;
    if (!c->mlp_skip_update) {
        DenseSegs S;
        S.n = 2 * nl;
        size_t off = 0;
        for (int l = 0; l < nl; l++) {
            MlpLayer& L = c->layers[l];
            S.off[2 * l] = off; S.w[2 * l] = L.w; S.acc[2 * l] = L.acc_w; S.w16[2 * l] = L.w16;
            S.w16t[2 * l] = L.w16t; S.in[2 * l] = L.in; S.out[2 * l] = L.out;
            S.w16t[2 * l + 1] = nullptr; S.in[2 * l + 1] = 1; S.out[2 * l + 1] = L.out;
            off += (size_t)L.out * L.in;
            S.off[2 * l + 1] = off; S.w[2 * l + 1] = L.b; S.acc[2 * l + 1] = L.acc_b; S.w16[2 * l + 1] = nullptr;
            off += L.out;
        }
        S.off[2 * nl] = off;
        const uint64_t mb = c->cfg.minibatch_size ? c->cfg.minibatch_size : (uint64_t)rows_divisor;
        return launch(c, {(unsigned)((off + 255) / 256), 256, 0, c->stream, c->cfg.world == 1}, adagrad_dense_all_kernel, S,
                      c->dense_grad, (float)(1.0 / (double)mb), c->cfg.learning_rate);
    }
    return 0;
}

}  // namespace lctr
