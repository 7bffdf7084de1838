// lightctr_b200/csrc/mlp_umma.cu -- the NFM dense layers on the Hopper tensor cores (wgmma.mma_async, accumulators in
// registers).  Same Fully_Conn_Layer chain and the same bf16 rounding points as mlp_bf16.cu (train/layer/
// fullyconnLayer.h:80-180; operands bf16, accumulation fp32, masters fp32), different machine mapping:
//
//   * one CTA = 128 samples = two warpgroups of 128 threads; warpgroup g owns samples [64g, 64g + 64) in the forward
//     pass, the loss and dX (the M = 64 of every wgmma), and the 64-row tiles m = g, g + 2, ... of every dW;
//   * every matrix that is ever an MMA operand lives in shared memory as an un-swizzled "chunk-major" tile
//         byte offset of element (r, c) of an R x C matrix = (c / 8) * (R * 16) + r * 16 + (c % 8) * 2
//     (8 x 16 B core matrices; 8-row groups 128 B apart, 8-column chunks R*16 B apart).  The tile is a K-major operand
//     when its columns are the reduction index and an MN-major operand when its rows are, so ONE copy of the activations
//     X_l [sample][feature], of the deltas (written over X_{l+1} in place) and of the weights W_l [out][in] serves all
//     three products of a layer -- only LBO/SBO and the transpose bits of the instruction differ:
//         forward  Y  = X_l . W_l^T          A = X_l     K-major    B = W_l     K-major    K = in_l
//         dX       dX = delta_l . W_l        A = delta_l K-major    B = W_l     MN-major   K = out_l
//         dW       dW = delta_l^T . X_l      A = delta_l MN-major   B = X_l     MN-major   K = 128 samples
//   * weights arrive by bulk-copy (TMA) transfers from chunk-major bf16 copies kept in global memory next to the fp32
//     masters (mlp_bf16.cu maintains them in the dense Adagrad kernel);
//   * the epilogues work on the accumulator fragments (a thread holds rows 16 w + lane / 4 and + 8 of its warp w, column
//     pair 2 (lane % 4) of every 8 columns): bias / activation / activation' / clipping, and the next operand written
//     straight back into its chunk-major tile (128 contiguous bytes per warp store), or dW sent to the dense-gradient
//     buffer with REDs;
//   * the output layer (out = 1) is folded into the last forward epilogue: a sample's dot product is complete inside the
//     four lanes that hold its row;
//   * db_l (column sums of delta_l over the samples) is taken where delta_l is produced, by a 14-shuffle reduce-scatter
//     over the 8 row groups of a warp per 64 columns, not by an extra MMA.
// Shapes outside the support test below (and any dropout mask) run on the mma.sync kernel of mlp_bf16.cu.
#include <cuda_bf16.h>

#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "mlp_umma.cuh"

namespace lctr {
namespace umma {

constexpr int kTM = 128;          // samples per CTA
constexpr int kThreads = 256;     // two warpgroups
constexpr int kChunk = kTM * 16;  // bytes between 8-column chunks of a [128 x C] tile

__device__ __forceinline__ void stamp(const Dev& P, int& n) {
    if (P.trace && blockIdx.x == 0 && threadIdx.x == 0) {
        P.trace[n] = (unsigned long long)clock64();
    }
    n++;
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier of the 128 threads of warpgroup g (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(g + 1) : "memory"); }

__device__ __forceinline__ void bar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// A wait that cannot hang the device: a descriptor or protocol bug traps instead.
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    for (uint32_t spin = 0; !ok; spin++) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// wgmma shared-memory matrix descriptor, no swizzle: start >> 4 at [0,14), LBO >> 4 at [16,30), SBO >> 4 at [32,46),
// layout type 0 at [62,64).  K-major operand: LBO = stride of the 8-column (K) chunks, SBO = stride of the 8-row (M/N)
// groups; MN-major operand: LBO = stride of the 8-row (K) groups, SBO = stride of the 8-column (M/N) chunks.
__device__ __forceinline__ uint64_t sdesc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32);
}
// keeps the compiler from moving accesses to accumulator registers across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x NT] (+)= A[64 x 16] . B[16 x NT], bf16 operands, fp32 accumulators; TA / TB = 1: the operand is MN-major.
// Fragment: d[4j + 2h + b] = (row 16 w + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + b) for warp w of the warpgroup.
template <int NT, int TA, int TB>
struct Wgmma;
template <int TA, int TB>
struct Wgmma<64, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                     "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
                     "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                       "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                       "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                       "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
                     : "memory");
    }
};
template <int TA, int TB>
struct Wgmma<16, TA, TB> {
    static __device__ __forceinline__ void run(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
                     "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
                     : "memory");
    }
};

// A warpgroup's products are taken in passes of at most 128 columns (64 accumulator registers a thread; a whole 256-column
// product would not leave the epilogues enough registers).
template <int NT>
using Acc = float[128 / NT][NT / 2];
// acc[t] = sum over k < ksteps of A(k) . B(t, k), for the NT-column tiles t < nt of one pass.  Every MMA of the pass is in
// flight at once; returns with the results in registers.
template <int NT, int TA, int TB, class DA, class DB>
__device__ __forceinline__ void wg_gemm(Acc<NT>& acc, int nt, int ksteps, DA da, DB db) {
#pragma unroll
    for (int t = 0; t < 128 / NT; t++) fence_regs(acc[t]);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int t = 0; t < 128 / NT; t++)
        if (t < nt)
            for (int k = 0; k < ksteps; k++) Wgmma<NT, TA, TB>::run(acc[t], da(k), db(t, k), k > 0);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int t = 0; t < 128 / NT; t++) fence_regs(acc[t]);
}

__device__ __forceinline__ void red_add(float* p, float a) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory"); }
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack2(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u)); }
// activations.h:71-90,126-143 on the MUFU unit, branch free and without the denormal fix-ups of __expf / __fdividef (the
// epilogues are issue bound: 18 instructions per element with the intrinsics, 6 here).
//   Sigmoid: 1 / (1 + 2^t), t = -log2(e) * (acc + b) clamped to +-16 log2(e); the bias arrives pre-multiplied by -log2(e)
//            so that t is one FFMA.  The reference's clamp values (1e-7, 1 - 1e-7 beyond |x| = 16) become sigmoid(+-16)
//            = 1.1e-7 / 0.9999999: the same bf16 number above, 1.13e-7 instead of 1.0e-7 below.
//   Tanh:    tanh.approx (relative error 2^-11, an eighth of a bf16 ulp); saturates to +-1 by itself.
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_ftz(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
constexpr float kLog2e = 1.4426950408889634f;
template <int ACT>
__device__ __forceinline__ float bias_scale() { return ACT == LCTR_ACT_SIGMOID ? -kLog2e : 1.0f; }
template <int ACT>
__device__ __forceinline__ float fwd_act(float acc, float b_scaled) {
    if (ACT == LCTR_ACT_SIGMOID) {
        const float t = fminf(fmaxf(fmaf(acc, -kLog2e, b_scaled), -16.f * kLog2e), 16.f * kLog2e);
        return rcp_ftz(1.0f + ex2_ftz(t));
    } else {
        float y;
        asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(acc + b_scaled));
        return y;
    }
}
template <int ACT>
__device__ __forceinline__ float bwd_act(float fo) { return ACT == LCTR_ACT_SIGMOID ? fo * (1.0f - fo) : 1.0f - fo * fo; }
__device__ __forceinline__ float clip15(float v) { return fminf(fmaxf(v, -15.f), 15.f); }

// One reduce-scatter step over lane bit `step`: lanes with the bit keep the upper n of their 2n values.
template <int N>
__device__ __forceinline__ void fold(float (&v)[16], int lane, int step) {
    const bool upper = (lane & step) != 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
        const float send = upper ? v[i] : v[i + N];
        const float keep = upper ? v[i + N] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, step);
    }
}
// Column sums of a 64-column fragment tile over the 8 row groups of a warp: v[2j + b] holds the thread's partial sum of
// column 8 j + 2 (lane % 4) + b; on return v[b] holds the warp's sum of column 8 (lane / 4) + 2 (lane % 4) + b.
__device__ __forceinline__ void colsum64(float (&v)[16], int lane) {
    fold<8>(v, lane, 16);
    fold<4>(v, lane, 8);
    fold<2>(v, lane, 4);
}

// Backward of hidden layer l (fullyconnLayer.h:120-180): delta_l is in X_{l+1}'s tile.  dW_l goes to the dense-gradient buffer;
// for l > 0 delta_{l-1} = clip(dX_l * act'(x_l)) replaces X_l and its column sums go to db_{l-1}; for l = 0 dX_0 is the
// fp32 gradient dz handed back to the embedding backward.  NT: column tile of the products whose N is in_l.
template <int ACT, int NT>
__device__ __forceinline__ void backward_layer(const Dev& P, unsigned char* smem, int l, int g, int lane, int rw, int cq,
                                               int row0, int valid, float* __restrict__ dz) {
    constexpr int kPass = 128 / NT;  // column tiles per pass
    const int K = P.in[l], N = P.out[l], r0 = 64 * g + rw;
    const uint32_t sbase = smem_addr(smem);
    const uint32_t xd = sbase + P.x_off[l + 1], xl = sbase + P.x_off[l], wl = sbase + P.w_off[l];
    Acc<NT> acc;
    // dW_l = delta_l^T . X_l -> dense gradient buffer (weightDelta, :165-178); fire-and-forget REDs
    for (int m = g; m < N / 64; m += 2) {
        for (int n0 = 0; n0 < K; n0 += 128) {
            const int t0 = n0 / NT, nt = min(kPass, (K - n0) / NT);
            wg_gemm<NT, 1, 1>(acc, nt, kTM / 16, [&](int k) { return sdesc(xd + m * 8 * kChunk + k * 256, 128, kChunk); },
                              [&](int t, int k) { return sdesc(xl + (t0 + t) * (NT / 8) * kChunk + k * 256, 128, kChunk); });
            float* dw = P.dw[l] + (size_t)(m * 64 + rw) * K + n0 + cq;
#pragma unroll
            for (int t = 0; t < kPass; t++)
                if (t < nt)
#pragma unroll
                    for (int j = 0; j < NT / 8; j++)
#pragma unroll
                        for (int h = 0; h < 2; h++)
                            red_add_v2(dw + (size_t)(8 * h) * K + t * NT + 8 * j, acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1]);
        }
    }
    __syncthreads();  // every dW_l MMA has read X_l before delta_{l-1} replaces it
    // dX_l = delta_l . W_l over this warpgroup's samples; a thread rewrites only the X_l elements of its own fragment
    for (int n0 = 0; n0 < K; n0 += 128) {
        const int t0 = n0 / NT, nt = min(kPass, (K - n0) / NT);
        wg_gemm<NT, 0, 1>(acc, nt, N / 16, [&](int k) { return sdesc(xd + g * 1024 + k * 2 * kChunk, kChunk, 128); },
                          [&](int t, int k) { return sdesc(wl + (t0 + t) * (NT / 8) * N * 16 + k * 256, 128, N * 16); });
        if (l > 0) {
            if constexpr (NT == 64) {  // in_l = out_{l-1}, a multiple of 64
                unsigned char* x = smem + P.x_off[l];
#pragma unroll
                for (int t = 0; t < kPass; t++) {
                    if (t >= nt) break;
                    float sd[16];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int c = n0 + t * 64 + j * 8 + cq;
                        sd[2 * j] = sd[2 * j + 1] = 0.f;
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            uint32_t* px = reinterpret_cast<uint32_t*>(x + (c >> 3) * kChunk + (r0 + 8 * h) * 16 + cq * 2);
                            const float2 a = unpack2(*px);
                            const uint32_t pk = pack2(clip15(acc[t][4 * j + 2 * h] * bwd_act<ACT>(a.x)),
                                                      clip15(acc[t][4 * j + 2 * h + 1] * bwd_act<ACT>(a.y)));
                            *px = pk;
                            const float2 e = unpack2(pk);
                            sd[2 * j] += e.x;
                            sd[2 * j + 1] += e.y;
                        }
                    }
                    colsum64(sd, lane);
                    red_add_v2(P.db[l - 1] + n0 + t * 64 + (lane >> 2) * 8 + cq, sd[0], sd[1]);
                }
            }
        } else {
#pragma unroll
            for (int t = 0; t < kPass; t++)
                if (t < nt)
#pragma unroll
                    for (int j = 0; j < NT / 8; j++)
#pragma unroll
                        for (int h = 0; h < 2; h++)
                            if (r0 + 8 * h < valid)
                                *reinterpret_cast<float2*>(dz + (size_t)(row0 + r0 + 8 * h) * K + n0 + t * NT + 8 * j + cq) =
                                    make_float2(acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1]);
        }
    }
}

// TRAIN = false: the forward-only instance of lctr_score -- the same staging, forward passes and output layer, then the
// pCTR alone: no labels, loss, statistics, deltas or dW / db (dz, label and the statistics arguments are unused).
template <int ACT, bool TRAIN>
__global__ void __launch_bounds__(kThreads, 1)
nfm_mlp_umma_kernel(Dev P, const float* __restrict__ z, float* __restrict__ dz, const float* __restrict__ wide,
                    const float* __restrict__ label, float* __restrict__ pred, int64_t rb, int B, double* partial,
                    unsigned int* done, double* out_slot) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_addr(smem);
    int ns = 0;
    stamp(P, ns);
    // g through a shuffle: the compiler then knows it is warp-uniform, and the wgmmas under branches on it (the dW tile
    // loop) are not serialised one wait per MMA
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = __shfl_sync(0xffffffffu, tid >> 7, 0);
    const int rw = (wid & 3) * 16 + (lane >> 2);  // fragment rows rw and rw + 8 of the warpgroup's 64
    const int r0 = 64 * g + rw;                   // the same as sample rows of the CTA
    const int cq = 2 * (lane & 3);                // fragment column pair in every 8 columns
    const int nh = P.nh;
    const int row0 = blockIdx.x * kTM;
    const int valid = min(kTM, B - row0);
    float* s_wl = reinterpret_cast<float*>(smem + P.wl_off);
    float* s_bias = reinterpret_cast<float*>(smem + P.bias_off);
    const uint32_t bar_w = sbase + P.bar_off;
    const float b_last = P.bias[nh][0];
    cudaTriggerProgrammaticLaunchCompletion();  // the dense updater behind this kernel may be scheduled as our CTAs retire

    if (tid == 0) {
        bar_init(bar_w, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        uint32_t total = 0;
        for (int l = 0; l < nh; l++) total += (uint32_t)P.out[l] * P.in[l] * 2;
        bar_expect_tx(bar_w, total);
        for (int l = 0; l < nh; l++) bulk_g2s(sbase + P.w_off[l], P.w16t[l], (uint32_t)P.out[l] * P.in[l] * 2, bar_w);
    }
    for (int l = 0; l < nh; l++)
        for (int j = tid; j < P.out[l]; j += kThreads) s_bias[P.vec_off[l] + j] = P.bias[l][j] * bias_scale<ACT>();
    for (int i = tid; i < P.in[nh]; i += kThreads) s_wl[i] = P.w32_last[i];
    // Everything above is independent of the kernel in front (the embedding forward that writes z and the wide term): when
    // launched programmatically dependent, the barrier, the weight copies and the bias vectors are under way before that
    // kernel has finished.  (No-op for an ordinary launch.)
    cudaGridDependencySynchronize();
    // the rows' wide terms and labels: requested now, used after the forward pass
    float wide_r[2], label_r[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const bool ok = r0 + 8 * h < valid;
        wide_r[h] = ok ? wide[rb + row0 + r0 + 8 * h] : 0.f;
        label_r[h] = TRAIN && ok ? label[rb + row0 + r0 + 8 * h] : 0.f;
    }
    {   // z tile -> bf16, chunk-major
        const int k = P.in[0], chunks = k / 8;
        for (int idx = tid; idx < kTM * chunks; idx += kThreads) {
            const int r = idx & (kTM - 1), ch = idx >> 7;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
            if (r < valid) {
                const float4* src = reinterpret_cast<const float4*>(z + (size_t)(row0 + r) * k + ch * 8);
                a = src[0]; b = src[1];
            }
            *reinterpret_cast<uint4*>(smem + P.x_off[0] + ch * kChunk + r * 16) =
                make_uint4(pack2(a.x, a.y), pack2(a.z, a.w), pack2(b.x, b.y), pack2(b.z, b.w));
        }
    }
    fence_async_smem();
    __syncthreads();
    bar_wait(bar_w, 0);
    stamp(P, ns);

    // ---- forward through the hidden layers (fullyconnLayer.h:80-118); each warpgroup on its own 64 samples
    Acc<64> acc;
    float part[2] = {0.f, 0.f};  // the output layer's dot products of rows r0, r0 + 8 (this thread's columns)
    for (int l = 0; l < nh; l++) {
        const int K = P.in[l], N = P.out[l];
        const uint32_t xa = sbase + P.x_off[l] + g * 1024, wb = sbase + P.w_off[l];
        const float* bias = s_bias + P.vec_off[l];
        unsigned char* y = smem + P.x_off[l + 1];
        const bool last = l == nh - 1;
        for (int n0 = 0; n0 < N; n0 += 128) {
            const int nt = min(2, (N - n0) / 64);
            wg_gemm<64, 0, 0>(acc, nt, K / 16, [&](int k) { return sdesc(xa + k * 2 * kChunk, kChunk, 128); },
                              [&](int t, int k) { return sdesc(wb + (n0 / 64 + t) * 1024 + k * 2 * N * 16, N * 16, 128); });
#pragma unroll
            for (int t = 0; t < 2; t++) {
                if (t >= nt) break;
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int c = n0 + t * 64 + j * 8 + cq;
                    const float2 b2 = *reinterpret_cast<const float2*>(bias + c);
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const uint32_t pk = pack2(fwd_act<ACT>(acc[t][4 * j + 2 * h], b2.x), fwd_act<ACT>(acc[t][4 * j + 2 * h + 1], b2.y));
                        *reinterpret_cast<uint32_t*>(y + (c >> 3) * kChunk + (r0 + 8 * h) * 16 + cq * 2) = pk;
                        if (last) {  // output layer (linear, out = 1) on the rounded activations, like the other operands
                            const float2 ar = unpack2(pk);
                            const float2 w2 = *reinterpret_cast<const float2*>(s_wl + c);
                            part[h] += ar.x * w2.x + ar.y * w2.y;
                        }
                    }
                }
            }
        }
        if (!last) {  // the next layer reads this warpgroup's rows only
            fence_async_smem();
            wg_sync(g);
        }
        stamp(P, ns);
    }

    // ---- output layer, loss, delta of the last hidden layer in place, dW/db of the output layer, db of the last hidden.
    // A thread reads back only the activations it wrote itself.
    double loss = 0.0, correct = 0.0;
    {
        const int K = P.in[nh];
        float d3[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float o = part[h];
            o += __shfl_xor_sync(0xffffffffu, o, 1);
            o += __shfl_xor_sync(0xffffffffu, o, 2);
            d3[h] = 0.f;
            if (r0 + 8 * h < valid) {
                const int64_t gi = rb + row0 + r0 + 8 * h;
                const float p = ref_sigmoid(wide_r[h] + (o + b_last));  // train_nfm_algo.cpp:101-116
                if ((lane & 3) == 0) {
                    pred[gi] = p;
                    double lt, ct;
                    loss_terms(p, label_r[h], lt, ct);
                    loss += lt;
                    correct += ct;
                }
                d3[h] = clip15(p - label_r[h]);
            }
        }
        if constexpr (!TRAIN) return;
        unsigned char* x = smem + P.x_off[nh];
        for (int t = 0; t < K / 64; t++) {
            float sw[16], sd[16];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int c = t * 64 + j * 8 + cq;
                const float2 w2 = *reinterpret_cast<const float2*>(s_wl + c);
                sw[2 * j] = sw[2 * j + 1] = sd[2 * j] = sd[2 * j + 1] = 0.f;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    uint32_t* px = reinterpret_cast<uint32_t*>(x + (c >> 3) * kChunk + (r0 + 8 * h) * 16 + cq * 2);
                    const float2 a = unpack2(*px);
                    // no mask on the output layer's dX; previous activation' (:139-156)
                    const uint32_t pk = pack2(clip15(d3[h] * w2.x * bwd_act<ACT>(a.x)), clip15(d3[h] * w2.y * bwd_act<ACT>(a.y)));
                    *px = pk;
                    const float2 e = unpack2(pk);
                    sw[2 * j] += d3[h] * a.x;  // weightDelta of the output layer (:165-178)
                    sw[2 * j + 1] += d3[h] * a.y;
                    sd[2 * j] += e.x;
                    sd[2 * j + 1] += e.y;
                }
            }
            colsum64(sw, lane);
            colsum64(sd, lane);
            const int c = t * 64 + (lane >> 2) * 8 + cq;
            red_add_v2(P.dw[nh] + c, sw[0], sw[1]);
            red_add_v2(P.db[nh - 1] + c, sd[0], sd[1]);  // biasDelta of the last hidden layer (:179)
        }
        const float dbl = warp_sum((lane & 3) == 0 ? d3[0] + d3[1] : 0.f);
        if (lane == 0) red_add(P.db[nh], dbl);
        fence_async_smem();
        __syncthreads();
        stamp(P, ns);
    }

    // ---- backward through the hidden layers
    for (int l = nh - 1; l >= 0; l--) {
        if (P.in[l] % 64 == 0)
            backward_layer<ACT, 64>(P, smem, l, g, lane, rw, cq, row0, valid, dz);
        else
            backward_layer<ACT, 16>(P, smem, l, g, lane, rw, cq, row0, valid, dz);
        fence_async_smem();
        __syncthreads();
        stamp(P, ns);
    }
    publish_stats(loss, correct, partial, done, out_slot, false);
    stamp(P, ns);
}

static size_t layout(const lctr_ctx* c, Dev& P) {
    const int nl = c->n_layers, nh = nl - 1;
    size_t off = 0;
    auto take = [&](size_t bytes, size_t align) { off = (off + align - 1) & ~(align - 1); size_t o = off; off += bytes; return (int)o; };
    int voff = 0;
    P.nh = nh;
    for (int l = 0; l < nl; l++) {
        P.in[l] = c->layers[l].in; P.out[l] = c->layers[l].out;
        P.x_off[l] = take((size_t)kTM * P.in[l] * 2, 128);
    }
    for (int l = 0; l < nh; l++) {
        P.w_off[l] = take((size_t)P.out[l] * P.in[l] * 2, 128);
        P.vec_off[l] = voff; voff += P.out[l];
    }
    P.wl_off = take((size_t)P.in[nh] * 4, 16);
    P.bias_off = take((size_t)voff * 4, 16);
    P.bar_off = take(16, 16);
    return off;
}

}  // namespace umma

// Shapes the wgmma kernel takes: every hidden width a multiple of 64 (<= 256), input width a multiple of 16 (<= 256),
// everything in 227 KB of shared memory.
bool mlp_umma_supported(const lctr_ctx* c) {
    const char* e = getenv("LCTR_MLP_UMMA");
    if (e && e[0] == '0') return false;
    const int nl = c->n_layers, nh = nl - 1;
    if (nh < 1 || c->layers[nh].out != 1 || c->layers[nh].in > 256) return false;
    if (c->layers[0].in % 16 != 0 || c->layers[0].in > 256) return false;
    for (int l = 0; l < nh; l++) {
        const int in = c->layers[l].in, out = c->layers[l].out;
        if (out % 64 != 0 || out > 256 || in > 256) return false;
    }
    umma::Dev P;
    return umma::layout(c, P) <= (size_t)227 * 1024;
}

int mlp_umma_prepare(lctr_ctx* c) {
    umma::Dev P;
    const size_t need = umma::layout(c, P);
    c->mlp_umma_smem = need;
    return 0;
}

int launch_mlp_umma(lctr_ctx* c, Slot& s, int64_t rb, int B, double* out_slot, bool train) {
    umma::Dev P;
    umma::layout(c, P);
    const int nl = c->n_layers, nh = nl - 1;
    P.act = c->cfg.activation;
    for (int l = 0; l < nl; l++) {
        MlpLayer& L = c->layers[l];
        P.w16t[l] = L.w16t; P.bias[l] = L.b; P.dw[l] = L.dw; P.db[l] = L.db;
    }
    P.w32_last = c->layers[nh].w;
    P.trace = nullptr;
    const bool trace = getenv("LCTR_MLP_UMMA_TRACE") && getenv("LCTR_MLP_UMMA_TRACE")[0] == '1';
    static unsigned long long* d_trace = nullptr;
    if (trace) {
        if (!d_trace) LCTR_CUDA(cudaMalloc((void**)&d_trace, 64 * sizeof(unsigned long long)));
        LCTR_CUDA(cudaMemsetAsync(d_trace, 0, 64 * sizeof(unsigned long long), c->stream));
        P.trace = d_trace;
    }
    const unsigned grid = (unsigned)((B + umma::kTM - 1) / umma::kTM);
    // one GPU: dependent on the embedding forward in front of it (fm_fused.cu, MODE 2), in a train step and in a score alike
    const bool sig = P.act == LCTR_ACT_SIGMOID;
    auto kern = train ? (sig ? umma::nfm_mlp_umma_kernel<LCTR_ACT_SIGMOID, true> : umma::nfm_mlp_umma_kernel<LCTR_ACT_TANH, true>)
                      : (sig ? umma::nfm_mlp_umma_kernel<LCTR_ACT_SIGMOID, false> : umma::nfm_mlp_umma_kernel<LCTR_ACT_TANH, false>);
    if (launch(c, {grid, (unsigned)umma::kThreads, c->mlp_umma_smem, c->stream, c->cfg.world == 1}, kern, P, c->z, c->dz, s.wide,
               s.label, s.pred, rb, B, c->stat_partial, c->stat_done, out_slot))
        return 1;
    if (trace) {  // phase boundaries of CTA 0: setup | per layer (mma, epilogue) | output | per layer backward | stats
        unsigned long long h[64];
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        LCTR_CUDA(cudaMemcpy(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost));
        fprintf(stderr, "[mlp_umma trace, SM cycles]");
        for (int i = 1; i < 64 && h[i]; i++) fprintf(stderr, " %llu", h[i] - h[i - 1]);
        fprintf(stderr, "  total %llu\n", h[0] ? [&] { int i = 1; while (i < 64 && h[i]) i++; return h[i - 1] - h[0]; }() : 0ull);
    }
    return 0;
}

}  // namespace lctr
