// lightctr_b200/csrc/metrics.cu -- test-set metrics on the device (SURVEY.md 8f-1): the summed logloss / accuracy of
// FM_Predict::Predict (predict/fm_predict.cpp:63-72) and AucEvaluator (util/evaluator.h:51-104) computed from the pCTR
// and label arrays a predict pass left in the slot, so that only three numbers cross PCIe.
//
// AucEvaluator buckets p into (size_t)(p * (2^24 - 1)) (two 2^24-entry int histograms), then walks the buckets from the
// top accumulating trapezoids in fp32.  Empty buckets add exactly 0 and leave the running totals unchanged, so the walk
// over the <= n NON-EMPTY buckets in the same order gives the same bits.  Here:
//   hist    : integer atomics into the two histograms, indexed by (2^24 - 1 - bucket) so that ascending = the walk order
//   compact : non-empty buckets -> dense (pos, neg) list in walk order (tile counts, one-block scan, ordered write;
//             the touched histogram entries are re-zeroed on the way: no 128 MB memset per call)
//   chain   : ONE warp replays the two sequential fp32 chains (trapezoids; logloss in row order) -- they are
//             order-dependent by definition, every lane computes the same chain from shuffled operands.
// Integer work is bit-exact; AUC is bit-identical to the reference for the same pCTR array (tests/test_parity_gpu.py);
// the logloss differs from glibc only through logf/log (<= 1 ulp per term).
//
// Weighted metrics (lctr_eval_weighted / lctr_eval_pred_weighted) keep the shape: one max-weight reduction, then the same
// bucket index into two u64 histograms of fixed-point weights q = rint(w 2^(32-E)) (2^(E-1) <= max w < 2^E), the same
// compaction over them, and a chain that walks fl32 of the u64 sums and weights the row-order logloss and correct count.
// Integer sums make the buckets independent of arrival order; the walk runs in units of 2^(E-32), a power-of-two scale
// that every fp32 operation of the walk commutes with and the final auc / totPos / totNeg divides out.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace lctr {

constexpr uint32_t kHashLen = (1u << 24) - 1;
constexpr int kAucTile = 512;
constexpr uint32_t kAucTiles = (kHashLen + 1) / kAucTile;  // 32768

__global__ void auc_hist_kernel(const float* __restrict__ pred, const float* __restrict__ label, int64_t n,
                                unsigned int* __restrict__ pos, unsigned int* __restrict__ neg) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t idx = (uint32_t)(pred[i] * (float)kHashLen);  // evaluator.h:64-65 (float * size_t -> float, truncation)
    const uint32_t rev = kHashLen - min(idx, kHashLen);
    if (label[i] == 1.f) atomicAdd(&pos[rev], 1u); else atomicAdd(&neg[rev], 1u);
}

// weighted: max over the row weights as float bits (weights are >= 0, so the bit order is the value order; -0 counts as 0)
__global__ void auc_wmax_kernel(const float* __restrict__ w, int64_t n, unsigned int* __restrict__ wmax) {
    unsigned m = 0u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        m = max(m, w[i] > 0.f ? __float_as_uint(w[i]) : 0u);
    m = __reduce_max_sync(kFull, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(wmax, m);
}

// weighted: q = rint(w 2^(32-E)) in [0, 2^32] added to the row's bucket; exact in u64 for n < 2^31
__global__ void auc_hist_w_kernel(const float* __restrict__ pred, const float* __restrict__ label, const float* __restrict__ w,
                                  int64_t n, const unsigned int* __restrict__ wmax, unsigned long long* __restrict__ pos,
                                  unsigned long long* __restrict__ neg) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || *wmax == 0u) return;
    int E;
    frexp((double)__uint_as_float(*wmax), &E);  // 2^(E-1) <= max w < 2^E
    const unsigned long long q = (unsigned long long)rint(ldexp((double)w[i], 32 - E));  // exact scale, one rounding
    if (q == 0ull) return;
    const uint32_t idx = (uint32_t)(pred[i] * (float)kHashLen);  // the bucket of auc_hist_kernel
    const uint32_t rev = kHashLen - min(idx, kHashLen);
    if (label[i] == 1.f) atomicAdd(&pos[rev], q); else atomicAdd(&neg[rev], q);
}

template <class H>
__global__ void __launch_bounds__(256)
auc_tile_count_kernel(const H* __restrict__ pos, const H* __restrict__ neg, unsigned int* __restrict__ tile_cnt) {
    const int lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= kAucTiles) return;
    unsigned c = 0;
    for (int j = lane; j < kAucTile; j += 32) {
        const uint32_t b = tile * kAucTile + j;
        c += (pos[b] | neg[b]) != (H)0;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(kFull, c, o);
    if (lane == 0) tile_cnt[tile] = c;
}

// exclusive scan of the 32768 tile counts by one block of 1024 threads (32 consecutive tiles per thread)
__global__ void __launch_bounds__(1024)
auc_tile_scan_kernel(const unsigned int* __restrict__ tile_cnt, unsigned int* __restrict__ tile_off, unsigned int* __restrict__ total) {
    __shared__ unsigned int sh[1024];
    const int t = threadIdx.x;
    unsigned v[32], s = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) { v[i] = tile_cnt[t * 32 + i]; s += v[i]; }
    sh[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        unsigned a = t >= o ? sh[t - o] : 0u;
        __syncthreads();
        sh[t] += a;
        __syncthreads();
    }
    unsigned run = sh[t] - s;
#pragma unroll
    for (int i = 0; i < 32; i++) { tile_off[t * 32 + i] = run; run += v[i]; }
    if (t == 1023) *total = sh[t];
}

template <class H, class L>
__global__ void __launch_bounds__(256)
auc_tile_write_kernel(H* __restrict__ pos, H* __restrict__ neg, const unsigned int* __restrict__ tile_cnt,
                      const unsigned int* __restrict__ tile_off, L* __restrict__ list) {
    const int lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= kAucTiles || tile_cnt[tile] == 0u) return;
    unsigned base = tile_off[tile];
    for (int j0 = 0; j0 < kAucTile; j0 += 32) {
        const uint32_t b = tile * kAucTile + j0 + lane;
        const H p = pos[b], q = neg[b];
        const bool on = (p | q) != (H)0;
        const unsigned m = __ballot_sync(kFull, on);
        if (on) {
            list[base + __popc(m & ((1u << lane) - 1u))] = L{p, q};
            pos[b] = (H)0;  // ready for the next evaluation
            neg[b] = (H)0;
        }
        base += __popc(m);
    }
}

// evaluator.h:74-93, the trapezoid walk over the m compacted buckets (fl32 of each count), by every lane of one warp
template <class L>
__device__ __forceinline__ float auc_walk(const L* __restrict__ list, unsigned m) {
    const int lane = threadIdx.x & 31;
    float totPos = 0.f, totNeg = 0.f, auc = 0.f;
    for (unsigned b0 = 0; b0 < m; b0 += 32) {
        const L mine = b0 + lane < m ? list[b0 + lane] : L{0, 0};
        const int cnt = (int)min(32u, m - b0);
        for (int j = 0; j < cnt; j++) {
            const auto p = __shfl_sync(kFull, mine.x, j), q = __shfl_sync(kFull, mine.y, j);
            const float totPosPrev = totPos, totNegPrev = totNeg;
            totPos = totPos + (float)p;
            totNeg = totNeg + (float)q;
            const float dx = totNeg > totNegPrev ? (totNeg - totNegPrev) : (totNegPrev - totNeg);
            const float area = (float)((double)(dx * (totPos + totPosPrev)) / 2.0);  // trapezoidArea, :95-104
            auc = auc + area;
        }
    }
    return (totPos > 0.f && totNeg > 0.f) ? auc / totPos / totNeg : 0.f;
}

// the two order-dependent fp32 chains, replayed by one warp
__global__ void auc_chain_kernel(const uint2* __restrict__ list, const unsigned int* __restrict__ n_list,
                                 const float* __restrict__ pred, const float* __restrict__ label, int64_t n,
                                 float* __restrict__ out /* [0]=loss [1]=correct [2]=auc */) {
    const int lane = threadIdx.x & 31;
    const float auc_out = auc_walk(list, *n_list);
    // ---- fm_predict.cpp:63-72: loss = (float)(loss + term) in row order; correct is a count
    float loss = 0.f;
    unsigned correct = 0;
    for (int64_t r0 = 0; r0 < n; r0 += 32) {
        const bool has = r0 + lane < n;
        const float p = has ? pred[r0 + lane] : 0.5f;
        const float y = has ? label[r0 + lane] : 0.f;
        const double term = !has ? 0.0 : (y == 1.f ? (double)(-logf(p)) : -log(1.0 - (double)p));
        const bool ok = has && ((p > 0.5f && y == 1.f) || (p < 0.5f && y == 0.f));
        correct += __popc(__ballot_sync(kFull, ok));
        const int cnt = (int)min((int64_t)32, n - r0);
        for (int j = 0; j < cnt; j++) {
            const double tj = __shfl_sync(kFull, term, j);
            loss = (float)((double)loss + tj);
        }
    }
    if (lane == 0) { out[0] = loss; out[1] = (float)correct; out[2] = auc_out; }
}

// the weighted chains: the walk over fl32 of the u64 bucket sums; loss = (float)(loss + (double)w term) in row order over
// the rows with w != 0 (no 0 * inf at p in {0, 1}); correct = sum w [correct] in double, in row order
__global__ void auc_chain_w_kernel(const ulonglong2* __restrict__ list, const unsigned int* __restrict__ n_list,
                                   const float* __restrict__ pred, const float* __restrict__ label, const float* __restrict__ w,
                                   int64_t n, double* __restrict__ out /* [0]=loss [1]=correct [2]=auc */) {
    const int lane = threadIdx.x & 31;
    const float auc_out = auc_walk(list, *n_list);
    float loss = 0.f;
    double correct = 0.0;
    for (int64_t r0 = 0; r0 < n; r0 += 32) {
        const bool has = r0 + lane < n;
        const float p = has ? pred[r0 + lane] : 0.5f;
        const float y = has ? label[r0 + lane] : 0.f;
        const float wi = has ? w[r0 + lane] : 0.f;
        const double term = wi == 0.f ? 0.0 : (double)wi * (y == 1.f ? (double)(-logf(p)) : -log(1.0 - (double)p));
        const double ok = ((p > 0.5f && y == 1.f) || (p < 0.5f && y == 0.f)) ? (double)wi : 0.0;
        const unsigned live = __ballot_sync(kFull, wi != 0.f);
        const int cnt = (int)min((int64_t)32, n - r0);
        for (int j = 0; j < cnt; j++) {
            const double tj = __shfl_sync(kFull, term, j), cj = __shfl_sync(kFull, ok, j);
            if ((live >> j) & 1u) loss = (float)((double)loss + tj);
            correct = correct + cj;
        }
    }
    if (lane == 0) { out[0] = (double)loss; out[1] = correct; out[2] = (double)auc_out; }
}

struct AucScratch {
    Buf<unsigned int> pos, neg, tile_cnt, tile_off, total;
    Buf<uint2> list;
    size_t list_cap = 0;
    Buf<float> out;
    Buf<float> in_pred, in_label;  // lctr_eval_pred: the caller's arrays on the device
    size_t in_cap = 0;
    // weighted evaluation, allocated by the first one: u64 histograms (2 x 128 MB), their list, the max weight's bits, the
    // results, and lctr_eval_pred_weighted's weights on the device
    Buf<unsigned long long> wpos, wneg;
    Buf<ulonglong2> wlist;
    size_t wlist_cap = 0;
    Buf<unsigned int> wmax;
    Buf<double> wout;
    Buf<float> in_weight;
    size_t in_w_cap = 0;
};
void drop(AucScratch* p) { delete p; }

static int auc_scratch(lctr_ctx* c, AucScratch** out) {
    if (!c->auc_scratch) {
        Owned<AucScratch> a(new AucScratch());  // the context's only once complete
        const size_t hn = (size_t)(kHashLen + 1);
        if (a->pos.alloc(hn) || a->neg.alloc(hn) || a->tile_cnt.alloc(kAucTiles) || a->tile_off.alloc(kAucTiles) ||
            a->total.alloc(1) || a->out.alloc(4))
            return 1;
        LCTR_CUDA(cudaMemsetAsync(a->pos, 0, hn * sizeof(unsigned int), c->stream));
        LCTR_CUDA(cudaMemsetAsync(a->neg, 0, hn * sizeof(unsigned int), c->stream));
        c->auc_scratch = std::move(a);
    }
    *out = c->auc_scratch.get();
    return 0;
}

// the three metrics of n device-resident (pCTR, label) pairs, in row order: histogram, compaction of the non-empty buckets,
// and the two fp32 chains
static int eval_device(lctr_ctx* c, AucScratch* a, const float* pred, const float* label, int64_t n, float* loss_sum,
                       int64_t* correct, float* auc) {
    if ((size_t)n > a->list_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        a->list_cap = 0;
        if (alloc_group(sized(a->list, (size_t)(n + 32)))) return 1;
        a->list_cap = (size_t)n;
    }
    if (launch(c, {(unsigned)((n + 255) / 256), 256, 0, c->stream}, auc_hist_kernel, pred, label, n, a->pos, a->neg) ||
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_count_kernel<unsigned int>, a->pos, a->neg, a->tile_cnt) ||
        launch(c, {1, 1024, 0, c->stream}, auc_tile_scan_kernel, a->tile_cnt, a->tile_off, a->total) ||
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_write_kernel<unsigned int, uint2>, a->pos, a->neg, a->tile_cnt,
               a->tile_off, a->list) ||
        launch(c, {1, 32, 0, c->stream}, auc_chain_kernel, a->list, a->total, pred, label, n, a->out))
        return 1;
    float h[3];
    LCTR_CUDA(cudaMemcpyAsync(h, a->out, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (loss_sum) *loss_sum = h[0];
    if (correct) *correct = (int64_t)h[1];
    if (auc) *auc = h[2];
    return 0;
}

// the weighted scratch, on the first weighted evaluation (the u64 histograms start zeroed; compaction re-zeroes them)
static int auc_scratch_w(lctr_ctx* c, AucScratch** out) {
    if (auc_scratch(c, out)) return 1;
    AucScratch* a = *out;
    if (!a->wout) {
        const size_t hn = (size_t)(kHashLen + 1);
        if (alloc_group(sized(a->wpos, hn), sized(a->wneg, hn), sized(a->wmax, 1), sized(a->wout, 3))) return 1;
        LCTR_CUDA(cudaMemsetAsync(a->wpos, 0, hn * sizeof(unsigned long long), c->stream));
        LCTR_CUDA(cudaMemsetAsync(a->wneg, 0, hn * sizeof(unsigned long long), c->stream));
    }
    return 0;
}

// eval_device over n device-resident (pCTR, label, weight) triples: max weight, u64 histograms, the same compaction, and
// the weighted chains
static int eval_device_w(lctr_ctx* c, AucScratch* a, const float* pred, const float* label, const float* w, int64_t n,
                         float* loss_sum, double* correct, float* auc) {
    if ((size_t)n > a->wlist_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        a->wlist_cap = 0;
        if (alloc_group(sized(a->wlist, (size_t)(n + 32)))) return 1;
        a->wlist_cap = (size_t)n;
    }
    LCTR_CUDA(cudaMemsetAsync(a->wmax, 0, sizeof(unsigned int), c->stream));
    const unsigned rgrid = (unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)c->sm_count * 4);
    if (launch(c, {rgrid, 256, 0, c->stream}, auc_wmax_kernel, w, n, a->wmax) ||
        launch(c, {(unsigned)((n + 255) / 256), 256, 0, c->stream}, auc_hist_w_kernel, pred, label, w, n, a->wmax, a->wpos, a->wneg) ||
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_count_kernel<unsigned long long>, a->wpos, a->wneg, a->tile_cnt) ||
        launch(c, {1, 1024, 0, c->stream}, auc_tile_scan_kernel, a->tile_cnt, a->tile_off, a->total) ||
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_write_kernel<unsigned long long, ulonglong2>, a->wpos, a->wneg,
               a->tile_cnt, a->tile_off, a->wlist) ||
        launch(c, {1, 32, 0, c->stream}, auc_chain_w_kernel, a->wlist, a->total, pred, label, w, n, a->wout))
        return 1;
    double h[3];
    LCTR_CUDA(cudaMemcpyAsync(h, a->wout, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (loss_sum) *loss_sum = (float)h[0];
    if (correct) *correct = h[1];
    if (auc) *auc = (float)h[2];
    return 0;
}

}  // namespace lctr

using namespace lctr;

extern "C" {

int lctr_eval(lctr_ctx* c, int slot, float* loss_sum, int64_t* correct, float* auc) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    LCTR_CHECK(s.rows > 0, "lctr_eval: slot %d is empty", slot);
    AucScratch* a = nullptr;
    if (auc_scratch(c, &a)) return 1;
    return eval_device(c, a, s.pred, s.label, s.rows, loss_sum, correct, auc);
}

// lctr_eval's metrics over host arrays (a whole test set gathered from the ranks of a sharded trainer, for one)
int lctr_eval_pred(lctr_ctx* c, int64_t n, const float* pctr, const int32_t* label, float* loss_sum, int64_t* correct,
                   float* auc) {
    LCTR_CHECK(c && pctr && label, "null argument");
    LCTR_CHECK(n > 0, "lctr_eval_pred: no rows (n = %lld)", (long long)n);
    AucScratch* a = nullptr;
    if (auc_scratch(c, &a)) return 1;
    if ((size_t)n > a->in_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        a->in_cap = 0;
        if (alloc_group(sized(a->in_pred, (size_t)n), sized(a->in_label, (size_t)n))) return 1;
        a->in_cap = (size_t)n;
    }
    std::vector<float> y((size_t)n);  // as upload_batch widens them: (float) of the int32 label
    for (int64_t i = 0; i < n; i++) y[(size_t)i] = (float)label[i];
    LCTR_CUDA(cudaMemcpyAsync(a->in_pred, pctr, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(a->in_label, y.data(), (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    return eval_device(c, a, a->in_pred, a->in_label, n, loss_sum, correct, auc);  // (synchronises before y goes)
}

int lctr_eval_weighted(lctr_ctx* c, int slot, float* loss_sum, double* correct, float* auc) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    LCTR_CHECK(s.rows > 0, "lctr_eval_weighted: slot %d is empty", slot);
    LCTR_CHECK(s.has_rw, "lctr_eval_weighted: slot %d has no row weights (lctr_set_row_weights)", slot);
    AucScratch* a = nullptr;
    if (auc_scratch_w(c, &a)) return 1;
    return eval_device_w(c, a, s.pred, s.label, s.rw, s.rows, loss_sum, correct, auc);
}

int lctr_eval_pred_weighted(lctr_ctx* c, int64_t n, const float* pctr, const int32_t* label, const float* weight,
                            float* loss_sum, double* correct, float* auc) {
    LCTR_CHECK(c && pctr && label && weight, "null argument");
    LCTR_CHECK(n > 0, "lctr_eval_pred_weighted: no rows (n = %lld)", (long long)n);
    for (int64_t r = 0; r < n; r++)
        LCTR_CHECK(std::isfinite(weight[r]) && weight[r] >= 0.f, "lctr_eval_pred_weighted: weight %g of row %lld is not a "
                   "finite value >= 0", (double)weight[r], (long long)r);
    AucScratch* a = nullptr;
    if (auc_scratch_w(c, &a)) return 1;
    if ((size_t)n > a->in_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        a->in_cap = 0;
        if (alloc_group(sized(a->in_pred, (size_t)n), sized(a->in_label, (size_t)n))) return 1;
        a->in_cap = (size_t)n;
    }
    if ((size_t)n > a->in_w_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        a->in_w_cap = 0;
        if (alloc_group(sized(a->in_weight, (size_t)n))) return 1;
        a->in_w_cap = (size_t)n;
    }
    std::vector<float> y((size_t)n);
    for (int64_t i = 0; i < n; i++) y[(size_t)i] = (float)label[i];
    LCTR_CUDA(cudaMemcpyAsync(a->in_pred, pctr, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(a->in_label, y.data(), (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(a->in_weight, weight, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    return eval_device_w(c, a, a->in_pred, a->in_label, a->in_weight, n, loss_sum, correct, auc);
}

// test hook: overwrite the slot's pCTR array (lctr_eval then evaluates exactly these values)
int lctr_upload_pred(lctr_ctx* c, int slot, const float* pctr) {
    LCTR_CHECK(c && pctr, "null argument");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    LCTR_CUDA(cudaMemcpyAsync(s.pred, pctr, (size_t)s.rows * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

}  // extern "C"
