// lightctr_b200/csrc/wnd.cu -- Wide&Deep with the per-field concat input of Distributed_Algo_Abst::batchGradCompute
// (distributed_algo_abst.h:176-280; SURVEY.md 8a-19), one synchronous process per GPU.
//   wide   pred += w[fid] * X over the row's entries, in entry order                                   (:205-211)
//   deep   input[field*d .. +d) = the d-float tensor of the FIRST entry of each field, 0 for absent fields
//          (:213-216 builds tensor_map from the first entry per field, :224-229 copies the tensors)
//   then the Fully_Conn_Layer chain (mlp.cu / mlp_bf16.cu) on the Fc*d input, pCTR = sigmoid(pred + fc)  (:236)
//   backward: gradW = loss * X + L2 * w per entry (:256); the chain's inputDelta is the gradient of the
//          first-entry tensors (:274-276, no L2 on tensors)
// Both gathers are HBM-bound row reads; the scatter uses the same RED + touched-map + sparse-apply path as FM.
// The reference runs this against asynchronous parameter servers; the synchronous restatement it is checked against
// is oracle/lightctr_oracle.c:orc_wnd_epoch (synchronous schedule of the worker pinned in tests/test_oracle_wnd_pin_cpu.py).
#include "common.cuh"

namespace lctr {

constexpr int kWndMaxFields = 2048;  // bitmap of seen fields: 64 words per warp

// warp = row.  z row zeroed, entries walked 32 at a time: the wide chain is replayed in entry order by every lane,
// first-of-field entries are found with __match_any_sync + a per-warp bitmap and copy their tensor into the row.
__global__ void __launch_bounds__(256)
wnd_forward_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid, const uint16_t* __restrict__ field,
                   const float* __restrict__ val, const float* __restrict__ W, const float* __restrict__ E, int Fc, int d,
                   float* __restrict__ z, uint32_t* __restrict__ zsrc, float* __restrict__ wide_out, int64_t rb, int64_t re) {
    __shared__ unsigned int seen_all[8][kWndMaxFields / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned int* seen = seen_all[wid];
    const int64_t r = rb + (int64_t)blockIdx.x * (blockDim.x >> 5) + wid;
    if (r >= re) return;
    const int in0 = Fc * d;
    float* zr = z + (size_t)(r - rb) * in0;
    uint32_t* sr = zsrc + (size_t)(r - rb) * Fc;
    for (int i = lane; i < in0; i += 32) zr[i] = 0.f;
    for (int i = lane; i < Fc; i += 32) sr[i] = 0xffffffffu;
    for (int i = lane; i < (Fc + 31) / 32; i += 32) seen[i] = 0u;
    __syncwarp();
    const int64_t b = row_ptr[r];
    const int n = (int)(row_ptr[r + 1] - b);
    float wide = 0.f;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool valid = i < n;
        const uint32_t f = valid ? __ldg(fid + b + i) : 0u;
        const unsigned a = valid ? (unsigned)__ldg(field + b + i) : 0u;
        const float x = valid ? (val ? __ldg(val + b + i) : 1.f) : 0.f;
        const float wx = valid ? __ldg(W + f) * x : 0.f;
        const int cnt = min(32, n - base);
        for (int j = 0; j < cnt; j++) wide = wide + __shfl_sync(kFull, wx, j);  // pred += w * X in entry order (:210)
        const unsigned m = __ballot_sync(kFull, valid);
        bool first = false;
        if (valid) {
            const unsigned same = __match_any_sync(m, a);
            first = (__ffs(same) - 1 == lane) && !((seen[a >> 5] >> (a & 31)) & 1u);
        }
        __syncwarp();
        if (first) {
            atomicOr(&seen[a >> 5], 1u << (a & 31));
            sr[a] = f;
            const float* src = E + (size_t)f * d;
            float* dst = zr + (size_t)a * d;
            for (int c = 0; c < d; c++) dst[c] = __ldg(src + c);
        }
        __syncwarp();
    }
    if (lane == 0) wide_out[r] = wide;
}

// warp = row: wide gradients of every entry, tensor gradients of the first-of-field entries.  RW: the slot's row weights rw
// scale the wide head and its L2 term (the tensor gradients arrive weighted in dz)
template <bool RW = false>
__global__ void __launch_bounds__(256)
wnd_backward_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid, const float* __restrict__ val,
                    const float* __restrict__ label, const float* __restrict__ pred, const float* __restrict__ W,
                    const uint32_t* __restrict__ zsrc, const float* __restrict__ dz, int Fc, int d, float* __restrict__ gW,
                    float* __restrict__ gE, uint8_t* __restrict__ touched, float l2_arg, int64_t rb, int64_t re,
                    const float* __restrict__ rw) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t r = rb + (int64_t)blockIdx.x * (blockDim.x >> 5) + wid;
    if (r >= re) return;
    const float lossv = row_head<RW>(pred[r], label[r], rw, r);  // :248
    const float l2 = row_l2<RW>(l2_arg, rw, r);
    const int64_t b = row_ptr[r], e = row_ptr[r + 1];
    for (int64_t i = b + lane; i < e; i += 32) {
        const uint32_t f = __ldg(fid + i);
        const float x = val ? __ldg(val + i) : 1.f;
        red_add_f32(gW + f, lossv * x + l2 * __ldg(W + f));  // gradW = loss * X + L2Reg_ratio * w (:256)
        if (touched) touched[f] = 1;
    }
    const uint32_t* sr = zsrc + (size_t)(r - rb) * Fc;
    const float* dr = dz + (size_t)(r - rb) * Fc * d;
    for (int a = lane; a < Fc; a += 32) {
        const uint32_t f = sr[a];
        if (f == 0xffffffffu) continue;
        for (int c = 0; c < d; c++) red_add_f32(gE + (size_t)f * d + c, dr[(size_t)a * d + c]);  // :274-276
        if (touched) touched[f] = 1;
    }
}

int wnd_reserve(lctr_ctx* c, int64_t rows) {
    if ((size_t)rows <= c->wnd_cap_rows) return 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    c->wnd_cap_rows = 0;
    if (alloc_group(sized(c->wnd_src, (size_t)rows * c->cfg.field_cnt))) return 1;
    c->wnd_cap_rows = (size_t)rows;
    return 0;
}

int launch_wnd_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    const int64_t rows = re - rb;
    if (rows <= 0) return 0;
    LCTR_CHECK(s.has_field, "Wide&Deep batch uploaded without the field array");
    ProfScope prof(c, PROF_FM_FWD);
    return launch(c, {(unsigned)((rows + 7) / 8), 256, 0, c->stream}, wnd_forward_kernel, s.row_ptr,
                  c->cfg.world > 1 ? s.ent_pslot : s.fid, s.field, s.has_val ? s.val.get() : nullptr, c->cW, c->cV, (int)c->cfg.field_cnt,
                  (int)c->cfg.factor_cnt, c->z, c->wnd_src, s.wide, rb, re);
}

// Distributed_Algo_Abst::Predict (distributed_algo_abst.h:163-174): pCTR = sigmoid(wide + chain output), no gradients
__global__ void wnd_pred_kernel(const float* __restrict__ wide, const float* __restrict__ out, float* __restrict__ pred, int64_t rb, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pred[rb + i] = ref_sigmoid(wide[rb + i] + out[i]);  // :236
}
int launch_wnd_pred(lctr_ctx* c, Slot& s, const float* mlp_out, int64_t rb, int64_t re) {
    if (re - rb <= 0) return 0;
    return launch(c, {(unsigned)((re - rb + 255) / 256), 256, 0, c->stream}, wnd_pred_kernel, s.wide, mlp_out, s.pred, rb, re - rb);
}

int launch_wnd_backward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    const int64_t rows = re - rb;
    if (rows <= 0) return 0;
    ProfScope prof(c, PROF_FM_BWD_RED);
    return launch(c, {(unsigned)((rows + 7) / 8), 256, 0, c->stream}, s.has_rw ? wnd_backward_kernel<true> : wnd_backward_kernel<false>, s.row_ptr,
                  c->cfg.world > 1 ? s.ent_pslot : s.fid, s.has_val ? s.val.get() : nullptr, s.label, s.pred, c->cW, c->wnd_src, c->dz,
                  (int)c->cfg.field_cnt, (int)c->cfg.factor_cnt, c->cgW, c->cgV, c->cfg.world > 1 ? nullptr : c->touched.get(),
                  c->cfg.l2_reg, rb, re, row_weights(s));
}

}  // namespace lctr
