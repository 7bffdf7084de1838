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
#include <algorithm>
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

__global__ void __launch_bounds__(256)
auc_tile_count_kernel(const unsigned int* __restrict__ pos, const unsigned int* __restrict__ neg, unsigned int* __restrict__ tile_cnt) {
    const int lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= kAucTiles) return;
    unsigned c = 0;
    for (int j = lane; j < kAucTile; j += 32) {
        const uint32_t b = tile * kAucTile + j;
        c += (pos[b] | neg[b]) != 0u;
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

__global__ void __launch_bounds__(256)
auc_tile_write_kernel(unsigned int* __restrict__ pos, unsigned int* __restrict__ neg, const unsigned int* __restrict__ tile_cnt,
                      const unsigned int* __restrict__ tile_off, uint2* __restrict__ list) {
    const int lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= kAucTiles || tile_cnt[tile] == 0u) return;
    unsigned base = tile_off[tile];
    for (int j0 = 0; j0 < kAucTile; j0 += 32) {
        const uint32_t b = tile * kAucTile + j0 + lane;
        const unsigned p = pos[b], q = neg[b];
        const bool on = (p | q) != 0u;
        const unsigned m = __ballot_sync(kFull, on);
        if (on) {
            list[base + __popc(m & ((1u << lane) - 1u))] = make_uint2(p, q);
            pos[b] = 0u;  // ready for the next evaluation
            neg[b] = 0u;
        }
        base += __popc(m);
    }
}

// the two order-dependent fp32 chains, replayed by one warp
__global__ void auc_chain_kernel(const uint2* __restrict__ list, const unsigned int* __restrict__ n_list,
                                 const float* __restrict__ pred, const float* __restrict__ label, int64_t n,
                                 float* __restrict__ out /* [0]=loss [1]=correct [2]=auc */) {
    const int lane = threadIdx.x & 31;
    // ---- evaluator.h:74-93
    const unsigned m = *n_list;
    float totPos = 0.f, totNeg = 0.f, auc = 0.f;
    for (unsigned b0 = 0; b0 < m; b0 += 32) {
        const uint2 mine = b0 + lane < m ? list[b0 + lane] : make_uint2(0u, 0u);
        const int cnt = (int)min(32u, m - b0);
        for (int j = 0; j < cnt; j++) {
            const unsigned p = __shfl_sync(kFull, mine.x, j), q = __shfl_sync(kFull, mine.y, j);
            const float totPosPrev = totPos, totNegPrev = totNeg;
            totPos = totPos + (float)p;
            totNeg = totNeg + (float)q;
            const float dx = totNeg > totNegPrev ? (totNeg - totNegPrev) : (totNegPrev - totNeg);
            const float area = (float)((double)(dx * (totPos + totPosPrev)) / 2.0);  // trapezoidArea, :95-104
            auc = auc + area;
        }
    }
    const float auc_out = (totPos > 0.f && totNeg > 0.f) ? auc / totPos / totNeg : 0.f;
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

struct AucScratch {
    Buf<unsigned int> pos, neg, tile_cnt, tile_off, total;
    Buf<uint2> list;
    size_t list_cap = 0;
    Buf<float> out;
    Buf<float> in_pred, in_label;  // lctr_eval_pred: the caller's arrays on the device
    size_t in_cap = 0;
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
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_count_kernel, a->pos, a->neg, a->tile_cnt) ||
        launch(c, {1, 1024, 0, c->stream}, auc_tile_scan_kernel, a->tile_cnt, a->tile_off, a->total) ||
        launch(c, {kAucTiles / 8, 256, 0, c->stream}, auc_tile_write_kernel, a->pos, a->neg, a->tile_cnt, a->tile_off, a->list) ||
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
