// lightctr_b200/csrc/mlp.cu -- the dense part of NFM / Wide&Deep: Fully_Conn_Layer chain, batched.
//
// Reference semantics (train/layer/fullyconnLayer.h, per SAMPLE): forward y_i = <x, W[i,:]> + b_i with
// masked hidden neurons forced to 0 BEFORE the activation (:96-99,110-113; sigmoid(0)=0.5 flows on),
// last layer linear (:116); backward clips delta to +-15 (:129-131), dX_i = sum_j W[j,i] mask_j delta_j
// (:139-147, mask only on hidden layers), previous activation' (:153-156), dW[j,:] += delta_j x
// (:165-178, UNmasked delta), db += delta (:179); Adagrad on bias then weights (:194-197).
// fp32 mode here is the PARITY mode: every dot product is evaluated in the reference's AVX lane order and every
// batch accumulation in sample order (one thread per output element), so that with equal inputs the MLP state
// follows the reference bit for bit.  (Training on the reference's data is chaotic: a 1-ulp difference in one
// activation grows to percent-level loss differences within an epoch, see DESIGN.md.)
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace lctr {

// Fully_Conn_Layer::forward (fullyconnLayer.h:80-118), one thread per (sample, output neuron).
__global__ void fc_forward_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                  const float* __restrict__ mask, float* __restrict__ y, int B, int in, int out,
                                  int has_next, int act) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)B * out) return;
    const int r = (int)(idx / out), j = (int)(idx % out);
    float v;
    if (has_next && mask[j] == 0.f) {
        v = 0.f;  // :96-99
    } else {
        const float* xr = x + (size_t)r * in;
        const float* wj = w + (size_t)j * in;
        v = avx_dot_seq([&](int i) { return xr[i]; }, [&](int i) { return wj[i]; }, in);  // :100
        v = v + bias[j];                                                                    // :101
    }
    if (has_next) {  // activation over ALL outputs, masked ones included (:110-113)
        if (act == LCTR_ACT_SIGMOID) {
            v = v < -16.f ? 1e-7f : (v > 16.f ? 0.99999988f : 1.0f / (1.0f + lctr_ref_expf(-v)));  // activations.h:73-84
        } else {
            const float t1 = ref_exp_any(v), t2 = ref_exp_any(-v);  // activations.h:132-138
            v = (t1 - t2) / (t1 + t2);
        }
    }
    y[idx] = v;
}

// clip(+-15) in place (matrix.h:152-162; fullyconnLayer.h:129-131)
__global__ void clip_kernel(float* __restrict__ d, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = d[i];
    d[i] = v < -15.f ? -15.f : (v > 15.f ? 15.f : v);
}

// input_delta[r][i] = avx_dot(mask .* W[:,i], delta[r][:])  (fullyconnLayer.h:139-147), then the previous layer's
// activation' (:153-156) when prev_act != nullptr.  One thread per (sample, input).
__global__ void fc_input_delta_kernel(const float* __restrict__ delta, const float* __restrict__ w,
                                      const float* __restrict__ mask, const float* __restrict__ prev_act,
                                      float* __restrict__ dx, int B, int in, int out, int has_next, int act) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)B * in) return;
    const int r = (int)(idx / in), i = (int)(idx % in);
    const float* dr = delta + (size_t)r * out;
    float v = avx_dot_seq([&](int j) { const float t = w[(size_t)j * in + i]; return has_next ? t * mask[j] : t; },
                          [&](int j) { return dr[j]; }, out);
    if (prev_act) {
        const float fo = prev_act[idx];
        v = act == LCTR_ACT_SIGMOID ? (v * fo) * (1.0f - fo) : v * (1.0f - fo * fo);  // activations.h:85-90,139-143
    }
    dx[idx] = v;
}

// weightDelta[j][i] += x[r][i] * delta[r][j] for r = 0..B-1 IN ORDER (fullyconnLayer.h:165-178);
// thread (j,i) with i == in accumulates biasDelta[j] += delta[r][j] (:179).
__global__ void fc_weight_grad_kernel(const float* __restrict__ x, const float* __restrict__ delta,
                                      float* __restrict__ dw, float* __restrict__ db, int B, int in, int out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)out * (in + 1)) return;
    const int j = (int)(idx / (in + 1)), i = (int)(idx % (in + 1));
    if (i < in) {
        float acc = dw[(size_t)j * in + i];
        for (int r = 0; r < B; r++) acc = acc + x[(size_t)r * in + i] * delta[(size_t)r * out + j];
        dw[(size_t)j * in + i] = acc;
    } else {
        float acc = db[j];
        for (int r = 0; r < B; r++) acc = acc + delta[(size_t)r * out + j];
        db[j] = acc;
    }
}

// p = sigmoid(wide + mlp_out); loss/acc; delta_L = p - y  (train_nfm_algo.cpp:101-116); RW: delta_L = w (p - y) with the
// slot's row weights rw (the layers' clip then applies to the weighted delta)
template <bool RW = false>
__global__ void nfm_loss_kernel(const float* __restrict__ wide, const float* __restrict__ out,
                                const float* __restrict__ label, float* __restrict__ pred, float* __restrict__ delta,
                                int64_t rb, int64_t n, double* partial, unsigned int* done, double* out_slot,
                                const float* __restrict__ rw) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double loss = 0.0, correct = 0.0;
    if (i < n) {
        const float p = ref_sigmoid(wide[rb + i] + out[i]);
        pred[rb + i] = p;
        const float y = label[rb + i];
        loss_terms(p, y, loss, correct);
        delta[i] = row_head<RW>(p, y, rw, rb + i);
    }
    publish_stats(loss, correct, partial, done, out_slot, false);
}

// AdagradUpdater_Num::update on a dense array (gradientUpdater.h:139-150)
__global__ void adagrad_dense_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ acc, size_t n,
                                     float invB, float lr) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float g1 = g[i] * invB;
    if (g1 != 0.f) {
        const float a = acc[i] + g1 * g1;
        acc[i] = a;
        w[i] = (float)((double)w[i] - (double)(lr * g1) / sqrt((double)a + 1e-7));
    }
    g[i] = 0.f;
}

int mlp_alloc(lctr_ctx* c) {
    const lctr_cfg& cf = c->cfg;
    LCTR_CHECK(cf.n_hidden >= 1 && cf.n_hidden <= LCTR_MAX_LAYERS, "NFM needs 1..%d hidden layers", LCTR_MAX_LAYERS);
    c->n_layers = cf.n_hidden + 1;
    size_t total = 0;
    int in = (int)mlp_in0(cf);
    for (int l = 0; l < c->n_layers; l++) {
        MlpLayer& L = c->layers[l];
        L.in = in;
        L.out = l < cf.n_hidden ? (int)cf.hidden[l] : 1;
        LCTR_CHECK(L.out > 0, "hidden[%d] must be > 0", l);
        total += (size_t)L.out * L.in + L.out;
        in = L.out;
    }
    c->dense_grad_n = total;
    if (c->dense_grad.alloc(total)) return 1;
    LCTR_CUDA(cudaMemsetAsync(c->dense_grad, 0, total * sizeof(float), c->stream));
    size_t off = 0;
    for (int l = 0; l < c->n_layers; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        if (L.w.alloc(nw) || L.b.alloc(L.out) || L.mask.alloc(L.out) || L.acc_w.alloc(nw) || L.acc_b.alloc(L.out)) return 1;
        LCTR_CUDA(cudaMemsetAsync(L.w, 0, nw * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(L.b, 0, L.out * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(L.acc_w, 0, nw * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(L.acc_b, 0, L.out * sizeof(float), c->stream));
        std::vector<float> ones(L.out, 1.f);
        LCTR_CUDA(cudaMemcpyAsync(L.mask, ones.data(), L.out * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        L.dw = c->dense_grad + off; off += nw;   // registerGradient order: weightDelta then biasDelta (fullyconnLayer.h:69-75)
        L.db = c->dense_grad + off; off += L.out;
    }
    const char* sk = getenv("LCTR_MLP_SKIP_UPDATE");
    c->mlp_skip_update = sk && sk[0] == '1';
    if (cf.mlp_precision == LCTR_MLP_BF16) return mlp_bf16_prepare(c);
    return 0;
}

int mlp_reserve(lctr_ctx* c, int64_t rows) {
    if ((size_t)rows <= c->mlp_cap_rows) return 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const size_t cap = (size_t)rows;
    const size_t k = mlp_in0(c->cfg);
    c->mlp_cap_rows = 0;
    if (alloc_group(sized(c->z, cap * k), sized(c->dz, cap * k), sized(c->mlp_out, cap))) return 1;
    for (int l = 0; l < c->n_layers && c->cfg.mlp_precision == LCTR_MLP_FP32; l++) {  // bf16 mode keeps activations on chip
        MlpLayer& L = c->layers[l];
        if (alloc_group(sized(L.act, cap * L.out), sized(L.delta, cap * (size_t)std::max(L.out, L.in)))) {
            for (MlpLayer& M : c->layers) { M.act.reset(); M.delta.reset(); }  // the whole group goes
            c->z.reset(); c->dz.reset(); c->mlp_out.reset();
            return 1;
        }
    }
    c->mlp_cap_rows = cap;
    return 0;
}

// world > 1: the dense gradients of the ranks are summed before the updater (data-parallel dense layers).  Wide&Deep without
// a registered hook keeps the reference's behaviour: every worker trains its OWN dense layers, only the wide weights and the
// tensors are shared through the parameter servers (distributed_algo_abst.h:115-118,279)
int mlp_sync_dense_grad(lctr_ctx* c) {
    if (c->cfg.world <= 1) return 0;
    if (c->cfg.model == LCTR_MODEL_WND && !c->dense_allreduce) return 0;
    LCTR_CHECK(c->dense_allreduce, "NFM with world=%d needs lctr_set_dense_allreduce (dense gradients are all-reduced "
               "between the MLP backward and its updater)", c->cfg.world);
    LCTR_CHECK(c->dense_allreduce(c->dense_allreduce_user, c->dense_grad, c->dense_grad_n, (void*)c->stream) == 0,
               "dense all-reduce callback failed");
    return 0;
}

static inline unsigned mlp_blocks(int64_t n) { return (unsigned)((n + 255) / 256); }

// Fully_Conn_Layer::forward down the chain (fullyconnLayer.h:80-118) on B rows of c->z; layer l's output in layers[l].act
static int mlp_forward_dev(lctr_ctx* c, int B) {
    const int nl = c->n_layers;
    const float* x = c->z;
    for (int l = 0; l < nl; l++) {
        MlpLayer& L = c->layers[l];
        if (launch(c, {mlp_blocks((int64_t)B * L.out), 256, 0, c->stream}, fc_forward_kernel, x, L.w, L.b, L.mask, L.act, B, L.in,
                   L.out, l + 1 < nl ? 1 : 0, c->cfg.activation))
            return 1;
        x = L.act;
    }
    return 0;
}
// Fully_Conn_Layer::backward up the chain (fullyconnLayer.h:120-180) from layers[nl-1].delta: clip, inputDelta into
// c->dz (first layer) / the previous layer's delta, weightDelta / biasDelta accumulated in the fused dense-gradient buffer
static int mlp_backward_dev(lctr_ctx* c, int B) {
    const int nl = c->n_layers;
    for (int l = nl - 1; l >= 0; l--) {
        MlpLayer& L = c->layers[l];
        const bool has_next = l + 1 < nl;
        const float* xin = l == 0 ? c->z : c->layers[l - 1].act;
        float* dx = l == 0 ? c->dz : c->layers[l - 1].delta;
        if (launch(c, {mlp_blocks((int64_t)B * L.out), 256, 0, c->stream}, clip_kernel, L.delta, (int64_t)B * L.out) ||
            launch(c, {mlp_blocks((int64_t)B * L.in), 256, 0, c->stream}, fc_input_delta_kernel, L.delta, L.w, L.mask,
                   l > 0 ? c->layers[l - 1].act.get() : nullptr, dx, B, L.in, L.out, has_next ? 1 : 0, c->cfg.activation) ||
            launch(c, {mlp_blocks((int64_t)L.out * (L.in + 1)), 256, 0, c->stream}, fc_weight_grad_kernel, xin, L.delta, L.dw, L.db,
                   B, L.in, L.out))
            return 1;
    }
    return 0;
}
// Fully_Conn_Layer::applyBatchGradient (fullyconnLayer.h:194-197): Adagrad on bias then weights, per layer; deltas zeroed
static int mlp_apply_dev(lctr_ctx* c, uint64_t mb) {
    const float invB = (float)(1.0 / (double)mb);
    for (int l = 0; l < c->n_layers; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        if (launch(c, {mlp_blocks(L.out), 256, 0, c->stream}, adagrad_dense_kernel, L.b, L.db, L.acc_b, L.out, invB,
                   c->cfg.learning_rate) ||
            launch(c, {mlp_blocks((int64_t)nw), 256, 0, c->stream}, adagrad_dense_kernel, L.w, L.dw, L.acc_w, nw, invB,
                   c->cfg.learning_rate))
            return 1;
    }
    return 0;
}

int launch_dense_score(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    if (re - rb <= 0) return 0;
    if (c->cfg.mlp_precision == LCTR_MLP_BF16) return launch_mlp_bf16_forward(c, s, rb, re);
    ProfScope prof(c, PROF_MLP);
    // wnd_pred_kernel's sigmoid(wide + out) is the expression nfm_loss_kernel writes
    return mlp_forward_dev(c, (int)(re - rb)) || launch_wnd_pred(c, s, c->layers[c->n_layers - 1].act, rb, re);
}

// forward MLP on c->z, loss, backward to c->dz, accumulate dW/db, Adagrad on the MLP (fp32, reference order).
int launch_nfm_mlp(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int64_t rows_divisor) {
    const int B = (int)(re - rb);
    const int nl = c->n_layers;
    if (c->cfg.mlp_precision == LCTR_MLP_BF16) return launch_nfm_mlp_bf16(c, s, rb, re, rows_divisor);
    LCTR_CHECK(c->cfg.mlp_precision == LCTR_MLP_FP32, "mlp_precision=%d unknown", c->cfg.mlp_precision);
    ProfScope prof(c, PROF_MLP);
    // B == 0 (a rank's empty share on several GPUs): no rows, no gradient (the buffer is zero between steps); the rank
    // still joins the all-reduce and the replicated updater, so the collective stays matched and the layers stay equal
    if (B > 0) {
        // forward, loss and delta of the output layer, backward
        double* out_slot = c->stats + 2 * (c->step % kStatRing);
        MlpLayer& last = c->layers[nl - 1];
        if (mlp_forward_dev(c, B) ||
            launch(c, {mlp_blocks(B), 256, 0, c->stream}, s.has_rw ? nfm_loss_kernel<true> : nfm_loss_kernel<false>, s.wide,
                   last.act, s.label, s.pred, last.delta, rb, B, c->stat_partial, c->stat_done, out_slot, row_weights(s)) ||
            mlp_backward_dev(c, B))
            return 1;
    }
    if (mlp_sync_dense_grad(c)) return 1;
    return c->mlp_skip_update ? 0 : mlp_apply_dev(c, c->cfg.minibatch_size ? c->cfg.minibatch_size : (uint64_t)rows_divisor);
}

}  // namespace lctr

using namespace lctr;
extern "C" {
// ---- the Fully_Conn_Layer chain as a stand-alone operator (fp32 reference-order mode) ---------------------------------
int lctr_mlp_forward(lctr_ctx* c, int64_t rows, const float* x, float* out) {
    LCTR_CHECK(c && x && rows > 0, "lctr_mlp_forward: null / empty input");
    LCTR_CHECK(c->n_layers > 0, "lctr_mlp_forward: the context has no dense layers (model NFM / WND with hidden[])");
    LCTR_CHECK(c->cfg.mlp_precision == LCTR_MLP_FP32, "lctr_mlp_forward/backward/apply run the fp32 reference-order layers");
    if (mlp_reserve(c, rows)) return 1;
    const size_t in0 = mlp_in0(c->cfg);
    LCTR_CUDA(cudaMemcpyAsync(c->z, x, (size_t)rows * in0 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    if (mlp_forward_dev(c, (int)rows)) return 1;
    c->mlp_fwd_rows = rows;
    if (out) {
        MlpLayer& last = c->layers[c->n_layers - 1];
        LCTR_CUDA(cudaMemcpyAsync(out, last.act, (size_t)rows * last.out * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    return 0;
}
int lctr_mlp_backward(lctr_ctx* c, int64_t rows, const float* dout, float* dx) {
    LCTR_CHECK(c && dout, "lctr_mlp_backward: null input");
    LCTR_CHECK(c->n_layers > 0 && rows > 0 && rows == c->mlp_fwd_rows, "lctr_mlp_backward: %lld rows, but the last lctr_mlp_forward "
               "ran %lld", (long long)rows, (long long)c->mlp_fwd_rows);
    MlpLayer& last = c->layers[c->n_layers - 1];
    LCTR_CUDA(cudaMemcpyAsync(last.delta, dout, (size_t)rows * last.out * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    if (mlp_backward_dev(c, (int)rows)) return 1;
    if (dx) {
        LCTR_CUDA(cudaMemcpyAsync(dx, c->dz, (size_t)rows * mlp_in0(c->cfg) * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    return 0;
}
int lctr_mlp_apply(lctr_ctx* c, uint64_t minibatch) {
    LCTR_CHECK(c && c->n_layers > 0, "lctr_mlp_apply: the context has no dense layers");
    LCTR_CHECK(minibatch > 0, "lctr_mlp_apply: minibatch divisor must be > 0");
    if (mlp_sync_dense_grad(c)) return 1;
    return mlp_apply_dev(c, minibatch);
}
int lctr_mlp_upload(lctr_ctx* c, int layer, const float* weight, const float* bias) {
    LCTR_CHECK(c && layer >= 0 && layer < c->n_layers, "mlp layer %d out of range", layer);
    MlpLayer& L = c->layers[layer];
    if (weight) LCTR_CUDA(cudaMemcpyAsync(L.w, weight, (size_t)L.out * L.in * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    if (bias) LCTR_CUDA(cudaMemcpyAsync(L.b, bias, (size_t)L.out * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    if (weight && mlp_bf16_refresh(c, layer)) return 1;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_set_dense_allreduce(lctr_ctx* c, lctr_allreduce_fn fn, void* user) {
    LCTR_CHECK(c, "null ctx");
    c->dense_allreduce = fn;
    c->dense_allreduce_user = user;
    return 0;
}
int lctr_mlp_download_grad(lctr_ctx* c, int layer, float* dweight, float* dbias) {
    LCTR_CHECK(c && layer >= 0 && layer < c->n_layers, "mlp layer %d out of range", layer);
    MlpLayer& L = c->layers[layer];
    if (dweight) LCTR_CUDA(cudaMemcpyAsync(dweight, L.dw, (size_t)L.out * L.in * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    if (dbias) LCTR_CUDA(cudaMemcpyAsync(dbias, L.db, (size_t)L.out * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_mlp_download(lctr_ctx* c, int layer, float* weight, float* bias) {
    LCTR_CHECK(c && layer >= 0 && layer < c->n_layers, "mlp layer %d out of range", layer);
    MlpLayer& L = c->layers[layer];
    if (weight) LCTR_CUDA(cudaMemcpyAsync(weight, L.w, (size_t)L.out * L.in * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    if (bias) LCTR_CUDA(cudaMemcpyAsync(bias, L.b, (size_t)L.out * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_mlp_set_mask(lctr_ctx* c, int layer, const float* mask) {
    LCTR_CHECK(c && mask && layer >= 0 && layer < c->n_layers, "mlp layer %d out of range", layer);
    MlpLayer& L = c->layers[layer];
    LCTR_CUDA(cudaMemcpyAsync(L.mask, mask, (size_t)L.out * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    for (int j = 0; j < L.out; j++) if (mask[j] == 0.f) c->mlp_has_mask = 1;  // sticky: the masked code path stays on
    return 0;
}
}
