// lightctr_b200/csrc/mlp_umma.cuh -- launch parameters of the wgmma dense-layer kernel (mlp_umma.cu)
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace lctr {
namespace umma {

constexpr int kMaxDense = LCTR_MAX_LAYERS + 1;

struct Dev {
    int nh, act;                            // hidden layers (the output layer, out == 1, is layer nh)
    int in[kMaxDense], out[kMaxDense];
    const __nv_bfloat16* w16t[kMaxDense];   // hidden layers: chunk-major bf16 tiles of W_l [out][in]
    const float* w32_last;                  // output layer weights, fp32 [in]
    const float* bias[kMaxDense];
    float* dw[kMaxDense];
    float* db[kMaxDense];
    int x_off[kMaxDense];                   // byte offset of X_l = input of layer l, [128 x in_l] chunk-major; X_0 = z
    int w_off[kMaxDense];                   // byte offset of W_l, [out_l x in_l] chunk-major
    int vec_off[kMaxDense];                 // element offset of layer l in the concatenated bias vector
    int wl_off, bias_off, bar_off;
    unsigned long long* trace;              // LCTR_MLP_UMMA_TRACE=1: clock64 stamps of CTA 0 per phase, else null
};

// element index of W[o][i] inside the chunk-major tile of an [out x in] matrix
__host__ __device__ __forceinline__ size_t tiled_index(size_t j, int in, int out) {
    const size_t o = j / in, i = j - o * in;
    return ((i >> 3) * out + o) * 8 + (i & 7);
}

}  // namespace umma

bool mlp_umma_supported(const lctr_ctx* c);
int mlp_umma_prepare(lctr_ctx* c);
// train = false: the forward-only instance (pred of rows [rb, rb + B) only; out_slot unused)
int launch_mlp_umma(lctr_ctx* c, Slot& s, int64_t rb, int B, double* out_slot, bool train);

}  // namespace lctr
