// lightctr_b200/csrc/common.cuh -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/lightctr_b200.h"
#include "ref_expf.h"

namespace lctr {

void set_error(const char* fmt, ...);

#define LCTR_CUDA(call)                                                                         \
    do {                                                                                        \
        cudaError_t _e = (call);                                                                \
        if (_e != cudaSuccess) {                                                                \
            ::lctr::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return 1;                                                                           \
        }                                                                                       \
    } while (0)

#define LCTR_CHECK(cond, ...)                  \
    do {                                       \
        if (!(cond)) {                         \
            ::lctr::set_error(__VA_ARGS__);    \
            return 1;                          \
        }                                      \
    } while (0)

// what a Buf holds: device memory, pinned host memory, or pinned host memory mapped into the device's address space
enum class Mem { Device, Pinned, Mapped };

// The owner of every allocation of the library: an array of T, released when the Buf is destroyed, reassigned or
// allocated again.  It converts to T*, so kernel arguments and pointer arithmetic read as they would with the raw pointer;
// being move-only, it cannot be passed to a kernel by value.
template <typename T, Mem M = Mem::Device>
class Buf {
  public:
    Buf() = default;
    Buf(Buf&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    Buf& operator=(Buf&& o) noexcept {
        if (this != &o) {
            reset();
            std::swap(p_, o.p_);
        }
        return *this;
    }
    ~Buf() { reset(); }
    // releases what the buffer holds, then allocates n elements (n == 0: none).  On failure the buffer stays empty and
    // set_error names the bytes requested.
    int alloc(size_t n) {
        reset();
        if (n == 0) return 0;
        const size_t bytes = n * sizeof(T);
        void* p = nullptr;
        const cudaError_t e = M == Mem::Device   ? cudaMalloc(&p, bytes)
                              : M == Mem::Pinned ? cudaMallocHost(&p, bytes)
                                                 : cudaHostAlloc(&p, bytes, cudaHostAllocMapped);
        if (e != cudaSuccess) {
            cudaGetLastError();  // the error is reported here; later calls must not see it again
            set_error("cannot allocate %zu bytes of %s memory: %s", bytes, M == Mem::Device ? "device" : "pinned host",
                      cudaGetErrorString(e));
            return 1;
        }
        p_ = static_cast<T*>(p);
        return 0;
    }
    void reset() {
        if (p_) {
            if (M == Mem::Device) cudaFree(p_);
            else cudaFreeHost(p_);
        }
        p_ = nullptr;
    }
    T* get() const { return p_; }
    operator T*() const { return p_; }

  private:
    T* p_ = nullptr;
};
template <typename T>
using HostBuf = Buf<T, Mem::Pinned>;
template <typename T>
using MappedBuf = Buf<T, Mem::Mapped>;

// The regrowth rule of every reserve: its group of buffers is released, then each is allocated with its new count, in
// order.  If one allocation fails the group is released again, so it holds either every buffer at its new size or
// nothing; the caller records the group's capacity only after this returns 0.
template <typename T, Mem M>
struct Sized {
    Buf<T, M>& b;
    size_t n;
};
template <typename T, Mem M>
inline Sized<T, M> sized(Buf<T, M>& b, size_t n) { return {b, n}; }
template <typename... S>
inline int alloc_group(S... s) {
    (s.b.reset(), ...);
    if ((... || s.b.alloc(s.n))) {
        (s.b.reset(), ...);
        return 1;
    }
    return 0;
}

// module states whose type only one .cu defines: that file defines their drop(), which deletes one
struct DistState;
struct KeyTable;
struct CscScratch;
struct AucScratch;
struct TextState;
void drop(DistState* p);
void drop(KeyTable* p);
void drop(CscScratch* p);
void drop(AucScratch* p);
void drop(TextState* p);
struct Drop {
    template <typename T>
    void operator()(T* p) const { drop(p); }
};
template <typename T>
using Owned = std::unique_ptr<T, Drop>;

constexpr int kNumSlots = 8;
constexpr int kPipe = LCTR_PIPE_DEPTH;  // streamed pipeline: batches in flight (the last kPipe slots are its buffers)
constexpr int kNumProf = 18;  // per-kernel timing buckets
enum { PROF_FM_FWD = 0, PROF_FM_BWD_RED = 1, PROF_APPLY = 2, PROF_FFM_FUSED = 3, PROF_FM_BWD_CSC = 4, PROF_MLP = 5, PROF_DIST_MARK = 6, PROF_DIST_COMPACT = 7, PROF_DIST_PULL = 8, PROF_DIST_PUSH = 9, PROF_DIST_BAR0 = 10, PROF_DIST_MERGE = 11, PROF_DIST_BAR1 = 12, PROF_CSC_BUILD = 13, PROF_FM_FUSED = 14, PROF_APPLY_COMPACT = 15, PROF_KEYS = 16, PROF_TEXT = 17 };
constexpr int kStatRing = 64;
constexpr int kHotRep = 32;      // fm_fused: replica rows per hot slot of the batch-compact gradient buffer
constexpr int kHotMax = 2048;    // hot slots per batch (ids beyond the cap stay ordinary slots)
constexpr uint32_t kHotBit = 0x80000000u;  // gradient index of an entry of a hot slot: kHotBit | replica block
constexpr unsigned kFull = 0xffffffffu;

// One resident CSR batch / dataset (FM_Algo_Abst::dataSet + label, fm_algo_abst.h:156,170).
struct Slot {
    int64_t rows = 0, nnz = 0, cap_rows = 0, cap_nnz = 0;
    Buf<int64_t> row_ptr;  // rows+1
    Buf<uint32_t> fid;     // nnz
    Buf<uint16_t> field;   // nnz (FFM)
    Buf<float> val;        // nnz, or unused when !has_val (all 1.0f)
    Buf<float> label;      // rows, as float (the reference compares `float target`)
    Buf<float> pred;       // rows: sigmoid(pred) of the last forward
    Buf<float> sumvx;      // rows*k: FM_Algo_Abst::sumVX (fm_algo_abst.h:145)
    Buf<float> wide;       // rows (NFM: wide part)
    bool has_val = false, has_field = false;
    // feature-major view (built on the host at upload when cfg.deterministic): per row block, the segments
    // (one per distinct fid of the block) list that fid's entries in ascending row order
    int64_t csc_block = 0;          // rows per block (0: none built)
    int64_t n_blocks = 0, n_segs = 0;
    Buf<int64_t> blk_seg_ptr;       // n_blocks+1 (host copy in h_blk_seg_ptr)
    Buf<int64_t> seg_ptr;           // n_segs+1 offsets into ent_*
    Buf<uint32_t> seg_fid;          // n_segs
    Buf<uint32_t> ent_row;          // nnz: row index of the entry
    Buf<float> ent_x;               // nnz (only when has_val)
    Buf<uint16_t> ent_field;        // nnz (FFM, device-built view only)
    std::vector<int64_t> h_blk_seg_ptr;
    int64_t cap_segs = 0, cap_blocks = 0, cap_ent = 0;
    // device-built feature-major view (cfg.deterministic == 2): work lists of short / long segments and
    // totals[4] = {nnz, n_segs, n_short, n_long} (device)
    bool dev_csc = false;
    Buf<uint32_t> short_list;
    Buf<uint2> long_list;                 // {segment, first entry} tasks
    int64_t cap_long = 0;
    Buf<double> csc_acc;                  // meeting point of multi-task segments
    Buf<unsigned int> csc_arrived;
    Buf<unsigned int> csc_totals;
    // multi-GPU: unique fids of the whole slot (the pull/push key set), built once at upload on the upload stream
    Buf<uint32_t> uniq;
    Buf<unsigned int> n_uniq;
    int64_t cap_uniq = 0;
    // order-free fused FM step (fm_fused.cu): per-entry slot of the gradient row (or kHotBit | replica block), the hot
    // slots' replica-block index per slot and their list; `uniq` / `n_uniq` above hold the key set
    Buf<uint32_t> ent_slot;
    Buf<uint32_t> ent_pslot;  // multi-GPU: plain slot per entry = row of the batch-compact parameter cache
    int64_t cap_ent_slot = 0;
    Buf<uint32_t> hot_of, hot_slot;
    Buf<unsigned int> n_hot;
    bool fused_valid = false;
    // keyed mode (keys.cu): SLOT_KEYS_LOOKUP = uploaded with insert = 0 (predict only); SLOT_KEYS_INVALID = the last
    // keyed upload failed, nothing may run on the slot until it is uploaded again; SLOT_KEYS_STALE = lctr_evict_keys
    // renumbered rows after the upload, so the slot's row ids are out of date until it is uploaded again
    int key_state = 0;
    // per-row weights of the resident batch (lctr_set_row_weights): rw[r] scales row r's loss head, its per-occurrence L2
    // terms and its statistics.  Every upload into the slot clears has_rw; rw keeps its storage (cap_rw rows)
    Buf<float> rw;
    int64_t cap_rw = 0;
    bool has_rw = false;
};
// the weights a train step over the slot applies, or null when the slot has none (kernels take their unweighted instance)
inline const float* row_weights(const Slot& s) { return s.has_rw ? s.rw.get() : nullptr; }
enum { SLOT_KEYS_OK = 0, SLOT_KEYS_LOOKUP = 1, SLOT_KEYS_INVALID = 2, SLOT_KEYS_STALE = 3 };

struct OptParams;
// captured graphs of one slot of the streamed pipeline (capi.cu)
struct PipeGraph {
    cudaGraphExec_t build = nullptr, step = nullptr;
    int64_t cap_rows = 0, cap_nnz = 0;
    bool has_val = false;
    Buf<int64_t> d_hdr;       // {rows, nnz} of the batch in the slot
    HostBuf<int64_t> h_hdr;
    Buf<OptParams> d_opt;     // updater parameters of the step
    HostBuf<OptParams> h_opt;
    Buf<double> d_stat;       // (loss, correct)
    HostBuf<double> h_stat;
    uint64_t ticket = ~0ull;
    int build_kernels = 0, step_kernels = 0;  // kernel nodes of each graph: the launches its replay counts
    const uint8_t* tracked = nullptr;         // the change map the step graph ends by marking (lctr_track_changes)
    bool weighted = false;                    // captured with the weighted instances and statistics over rw
    const float* rw = nullptr;                // the slot's weight array the weighted graph reads
};

struct MlpLayer {
    int in = 0, out = 0;
    Buf<float> w, b, mask;                // [out][in], [out], [out]
    float *dw = nullptr, *db = nullptr;   // views into the fused dense-grad buffer
    Buf<float> acc_w, acc_b;              // Adagrad state
    Buf<float> act;                       // [B][out] activations (post-activation for hidden layers)
    Buf<float> delta;                     // [B][out] dL/d(pre-activation)
    Buf<__nv_bfloat16> w16;               // bf16 copy of w (tensor-core mode, hidden layers)
    Buf<__nv_bfloat16> w16t;              // the same, as the chunk-major tile mlp_umma.cu stages by bulk copy
};

}  // namespace lctr

namespace lctr {
// slot map scratch + batch-compact gradient buffers of the order-free fused FM step (fm_fused.cu); the slot map part is
// also what the multi-GPU exchange is keyed by (dist.cu)
struct FusedState {
    Buf<uint8_t> mark;            // 128 * T permuted byte marks
    size_t T = 0;
    Buf<uint32_t> slot_of;        // F: fid -> slot of the batch being built
    Buf<unsigned int> cnt;        // sampled multiplicities (zero between builds)
    size_t cnt_cap = 0;
    Buf<float> G;                 // [G_rows][GS] compact gradient rows (zero between steps)
    size_t G_rows = 0;
    Buf<float> Ghot;              // [kHotMax][kHotRep][GS] replica rows of the hot slots (zero between steps)
    Buf<OptParams> d_opt;         // updater parameters in device memory (graph launches)
    int GS = 0;                   // row stride of G / Ghot (GRAD_COMPACT only; the other paths use the slot map alone)
};
// Where a train step's sparse gradient goes; one value per context, fixed from cfg by lctr_create (grad_path_of).  What a
// context allocates follows it: update_g (gW / gV) for GRAD_DENSE and the grouped FFM backward, the touched map and the
// sparse apply's list for GRAD_DENSE only.
enum GradPath {
    // FM / NFM, deterministic = 0, k in {4, 8, 16, 32}, any world: fm_fused kernels -> batch-compact G / Ghot ->
    // apply_compact (one GPU) or push + merge_apply (several)
    GRAD_COMPACT = 0,
    // FFM with deterministic 0 or 1, Wide&Deep, FM / NFM with deterministic = 0 and any other k, NFM with deterministic = 2:
    // REDs into update_g + touched map -> launch_apply (opt.cu); several GPUs: rows cgW / cgV -> push -> merge_kernel ->
    // launch_apply
    GRAD_DENSE = 1,
    // FM / NFM deterministic = 1 (host-built view), FM / FFM deterministic = 2 (device grouping): the updater runs inside
    // the backward; grouped FFM still meets split segments in update_g
    GRAD_FEATURE_MAJOR = 2,
};
}  // namespace lctr
struct lctr_ctx {
    lctr_cfg cfg;
    cudaStream_t stream = nullptr;
    size_t F = 0, rowlen = 0;  // rowlen = k (FM/NFM) or Fc*k (FFM)
    size_t Fl = 0;             // rows of this rank's table shard (== F when world == 1)
    lctr::GradPath grad_path = lctr::GRAD_DENSE;
    // parameters, gradient accumulators (update_g layout: W part, V part; null unless the path uses them), optimizer state
    lctr::Buf<float> W, V, gW, gV;
    lctr::Buf<float> s1W, s1V, s2W, s2V;
    lctr::Buf<uint8_t> touched;  // Fl bytes: 1 = fid (shard-local index) received gradient this step (GRAD_DENSE)
    // change tracking (lctr_track_changes, delta.cu): Fl bytes, 1 = the row changed since the parent save; null when off.
    // The parent is the last file saved or loaded while tracking was on, named by its hash (checkpoint.cu)
    lctr::Buf<uint8_t> changed;
    int parent_state = 0;        // lctr::PARENT_*
    uint64_t parent_hash = 0;
    // compute view used by the forward/backward kernels: aliases of the arrays above when world == 1; in multi-GPU mode the
    // batch-compact parameter cache and (GRAD_DENSE) gradient rows, indexed by exchange row
    float *cW = nullptr, *cV = nullptr, *cgW = nullptr, *cgV = nullptr;
    lctr::Owned<lctr::DistState> dist;
    std::unique_ptr<lctr::FusedState> fused;  // order-free fused FM step (fm_fused.cu)
    lctr::Owned<lctr::KeyTable> keys;         // keyed mode (keys.cu): key -> row table; F = capacity + 1 (the null row)
    size_t dist_rows = 0;               // world > 1: rows of the exchange index space (gradient / cache rows are indexed by it)
    lctr::Buf<uint32_t> touch_list;      // compacted fids of the step (stage A of the sparse apply)
    lctr::Buf<unsigned int> n_touch;     // list length (device)
    lctr::Buf<unsigned int> apply_done;  // block-completion counter of stage B
    // per-step statistics ring: [kStatRing][2] doubles (loss sum, correct count) + scratch
    lctr::Buf<double> stats;
    lctr::Buf<double> stat_partial;      // [2] running accumulation of the current step
    lctr::Buf<unsigned int> stat_done;   // block-completion counter
    lctr::HostBuf<double> h_stats;       // pinned host mirror [2]
    uint64_t step = 0;
    size_t adam_iter = 0;
    lctr::Slot slots[lctr::kNumSlots];
    // MLP
    int n_layers = 0;
    lctr::MlpLayer layers[LCTR_MAX_LAYERS + 1];
    lctr::Buf<float> dense_grad;  // fused [dW0, db0, dW1, db1, ...]
    size_t dense_grad_n = 0;
    lctr::Buf<float> z, dz;       // [B][k] NFM bi-interaction output and its gradient
    lctr::Buf<float> mlp_out;     // [B]
    size_t mlp_cap_rows = 0;
    int64_t mlp_fwd_rows = 0;      // rows of the last lctr_mlp_forward (lctr_mlp_backward must match)
    lctr::Buf<uint32_t> wnd_src;   // Wide&Deep: fid of the first entry of each field, [rows][Fc]
    size_t wnd_cap_rows = 0;
    lctr::Owned<lctr::AucScratch> auc_scratch;  // metrics.cu: histograms + lists of lctr_eval
    int csc_in_step = 0;        // LCTR_CSC_IN_STEP=1: rebuild the feature-major view inside every train step (bench)
    lctr::Buf<float> ffm_T;     // FFM grouped step: per-sample field-pair tiles [rows][Fc][Fc][k]
    lctr::Buf<uint16_t> ffm_cnt; // [rows][Fc] features per field
    size_t ffm_T_rows = 0;
    lctr_allreduce_fn dense_allreduce = nullptr;  // world > 1: sums dense_grad over the ranks on c->stream
    void* dense_allreduce_user = nullptr;
    int mlp_tm = 0;             // bf16 mode: samples per CTA tile (128 or 64)
    size_t mlp_smem = 0;        // bf16 mode: dynamic shared memory per CTA
    int mlp_umma = 0;           // bf16 mode: the wgmma kernel (mlp_umma.cu) takes this chain
    size_t mlp_umma_smem = 0;
    int mlp_has_mask = 0;       // any dropout mask entry == 0
    int mlp_skip_update = 0;    // LCTR_MLP_SKIP_UPDATE=1: leave the dense gradients in place (tests read them)
    int sm_count = 132;
    int64_t launches = 0;
    const float* fwd_quirk_sumvx = nullptr;  // FM_Predict quirk: training sumVX rows used by the next forward launch
    int64_t fwd_quirk_rows = 0;
    lctr::Owned<lctr::CscScratch> csc_scratch;  // csc.cu: dense count / offset arrays of the device-side grouping
    lctr::Owned<lctr::TextState> text;          // text.cu: staging and parser state of lctr_upload_libffm
    // optional per-kernel timing (lctr_profile): events bracket every launch on the ctx stream
    int profiling = 0;
    std::vector<cudaEvent_t> prof_ev;   // flat list of (start, stop) pairs
    std::vector<int> prof_id;
    double prof_ms[lctr::kNumProf] = {0};
    int64_t prof_cnt[lctr::kNumProf] = {0};
    // streamed training pipeline (lctr_train_batch_async): copy stream, per-slot events, pinned result ring
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copied[lctr::kPipe] = {}, ev_computed[lctr::kPipe] = {};
    cudaStream_t build_stream = nullptr;                  // graph pipeline: the slot-map kernels of batch t run here while the copy
    cudaEvent_t ev_h2d[lctr::kPipe] = {};                   // engine already moves batch t+1 on copy_stream
    cudaEvent_t ev_stat[lctr::kStatRing] = {nullptr};
    lctr::HostBuf<double> h_stat_ring;
    uint64_t pipe_issued = 0, pipe_waited = 0;
    lctr::PipeGraph pipe_graph[lctr::kPipe];
};

namespace lctr {

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}
// vectorised no-return atomic add: one 16-byte RED per 4 floats (sm_90+: red.global.add.v4.f32)
__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float4 ldg_f4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
// Gather loads whose ISSUE ORDER matters: as volatile asm they stay where the source puts them (all gathers of a pass
// back to back), where plain __ldg loads were sunk next to their uses -- one dependent round trip per row instead of
// one per pass (visible in the SASS of the forward kernel).
__device__ __forceinline__ float4 ldg_f4_pinned(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float ldg_f32_pinned(const float* p) {
    float v;
    asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// avx_dotProduct(x, y, n) (common/avx.h:102-127) with strided operands, evaluated by ONE thread in the
// reference's order: 8 lane accumulators over the full 8-chunks, the hsum tree, then the scalar tail.
template <typename FX, typename FY>
__device__ __forceinline__ float avx_dot_seq(FX x, FY y, int n) {
    float result = 0.f;
    int i = 0;
    if (n > 7) {
        float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (; i + 8 <= n; i += 8) {
#pragma unroll
            for (int l = 0; l < 8; l++) d[l] = d[l] + x(i + l) * y(i + l);
        }
        const float a0 = d[4] + d[0], a1 = d[5] + d[1], a2 = d[6] + d[2], a3 = d[7] + d[3];
        const float b0 = a0 + a2, b1 = a1 + a3;
        result = result + (b0 + b1);
    }
    for (; i < n; i++) result = result + x(i) * y(i);
    return result;
}

// Sigmoid::forward, util/activations.h:65-72 (clamps at +-16; accurate expf, no fast-math)
__device__ __forceinline__ float ref_sigmoid(float x) {
    if (x < -16.f) return 1e-7f;
    if (x > 16.f) return 0.99999988f;  // (float)(1.0 - 1e-7)
    return 1.0f / (1.0f + lctr_ref_expf(-x));
}
// std::exp(float) of the reference (glibc expf) for unbounded arguments (Tanh, activations.h:134)
__device__ __forceinline__ float ref_exp_any(float x) { return fabsf(x) < 87.f ? lctr_ref_expf(x) : expf(x); }
// loss term + accuracy, train_fm_algo.cpp:93-98: y==1 ? -logf(p) : -log(1.0 - p) (double)
__device__ __forceinline__ void loss_terms(float p, float y, double& loss, double& correct) {
    loss = (y == 1.f) ? (double)(-logf(p)) : -log(1.0 - (double)p);
    correct = ((p > 0.5f && y == 1.f) || (p < 0.5f && y == 0.f)) ? 1.0 : 0.0;
}
// the head of a weighted row: fl(w (p - y)); the unweighted instances (RW = false) form p - y alone
template <bool RW>
__device__ __forceinline__ float row_head(float p, float y, const float* __restrict__ rw, int64_t r) {
    return RW ? __ldg(rw + r) * (p - y) : p - y;
}
// the per-occurrence L2 coefficient of a weighted row: fl(w l2)
template <bool RW>
__device__ __forceinline__ float row_l2(float l2, const float* __restrict__ rw, int64_t r) {
    return RW ? __ldg(rw + r) * l2 : l2;
}

// Block-level accumulation of (loss, correct) into ctx statistics; the last block to finish publishes
// the step totals into the ring slot and re-arms the accumulators (no memset launches between steps).
__device__ __forceinline__ void publish_stats(double loss, double correct, double* partial, unsigned int* done,
                                               double* out_slot, bool accumulate_out) {
    __shared__ double sh[2][32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    loss = warp_sum_d(loss);
    correct = warp_sum_d(correct);
    if (lane == 0) { sh[0][wid] = loss; sh[1][wid] = correct; }
    __syncthreads();
    if (wid == 0) {
        double a = lane < nw ? sh[0][lane] : 0.0, b = lane < nw ? sh[1][lane] : 0.0;
        a = warp_sum_d(a);
        b = warp_sum_d(b);
        if (lane == 0) {
            atomicAdd(&partial[0], a);
            atomicAdd(&partial[1], b);
            __threadfence();
            unsigned int prev = atomicAdd(done, 1u);
            if (prev == gridDim.x - 1) {
                __threadfence();
                double l = atomicAdd(&partial[0], 0.0), c = atomicAdd(&partial[1], 0.0);
                if (accumulate_out) { out_slot[0] += l; out_slot[1] += c; }
                else { out_slot[0] = l; out_slot[1] = c; }
                partial[0] = 0.0; partial[1] = 0.0;
                *done = 0u;
                __threadfence();
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// kernel launchers (defined in the .cu files)
// ---------------------------------------------------------------------------------------------
// RAII bracket: records a (start, stop) event pair around one launch when profiling is on
struct ProfScope {
    lctr_ctx* c; int id; cudaEvent_t a = nullptr, b = nullptr;
    ProfScope(lctr_ctx* c_, int id_) : c(c_), id(id_) {
        if (!c->profiling) return;
        cudaEventCreate(&a); cudaEventCreate(&b);
        cudaEventRecord(a, c->stream);
    }
    ~ProfScope() {
        if (!a) return;
        cudaEventRecord(b, c->stream);
        c->prof_ev.push_back(a); c->prof_ev.push_back(b); c->prof_id.push_back(id);
    }
};
int launch_fm_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm, bool stats);
int launch_fm_backward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm);
int launch_ffm_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_apply(lctr_ctx* c, int64_t rows_in_step);
int launch_fm_backward_csc(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm);
// csc.cu: feature-major view built on the device at upload + atomic-free backward with fused updater
int csc_reserve(lctr_ctx* c, Slot& s, int64_t max_nnz);
int csc_build_device(lctr_ctx* c, Slot& s, cudaStream_t st, const int32_t* label_i32, const int64_t* hdr,
                     int64_t rows_cap, int64_t nnz_cap);
int launch_fm_backward_devcsc(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
struct OptParams;
int launch_fm_backward_devcsc_ex(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, const OptParams* P_host, const void* dP);
void csc_opt_params(lctr_ctx* c, int64_t rows, void* out);
int launch_fm_forward_ex(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool nfm, bool stats, const int64_t* hdr,
                         double* out_slot_override);
bool csc_device_supported(const lctr_ctx* c);
int launch_predict_quirk(lctr_ctx* c, Slot& s, Slot& train);
// fm_fused.cu: order-free FM / NFM step over a batch-compact gradient buffer (GRAD_COMPACT); the slot map also keys the
// multi-GPU exchange of every path
int fused_reserve(lctr_ctx* c, Slot& s, int64_t nnz);
int fused_build_slot(lctr_ctx* c, Slot& s, cudaStream_t st, const int64_t* hdr, int64_t rows_cap, int64_t nnz_cap);
void dist_wait_info(lctr_ctx* c, const unsigned long long** flags, int* n, unsigned long long* epoch);
int launch_fm_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats, const int64_t* hdr, double* out_slot_override);
int launch_fm_forward_tree(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats);
int launch_nfm_forward_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_nfm_backward_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_apply_compact(lctr_ctx* c, Slot& s, int64_t rows_in_step, const OptParams* P_host, const OptParams* dP);
void fused_opt_params(lctr_ctx* c, int64_t rows, void* out);
void* fused_dev_opt(lctr_ctx* c);
int launch_ffm_predict_inorder(lctr_ctx* c, Slot& s);
// multi-GPU (dist.cu)
int dist_alloc(lctr_ctx* c);
void dist_close_peers(lctr_ctx* c);  // unmaps the peers' arenas (lctr_destroy)
int dist_send_keys(lctr_ctx* c, Slot& s, int slot, cudaStream_t st);               // at upload: key lists -> the owners' inboxes
int dist_send_empty(lctr_ctx* c, int slot, cudaStream_t st);                      // at upload of an empty share: empty lists
int dist_pre_step(lctr_ctx* c, Slot& s, int slot, bool in_kernel_wait, bool train = true);  // owner-driven pull of the step's rows
int dist_release(lctr_ctx* c);                                                     // end of a pull-only round (train = false)
int dist_post_step(lctr_ctx* c, Slot& s, int slot, int64_t rows_divisor);         // push gradients, owner-side merge + update
int dist_check_overflow(lctr_ctx* c);
// keyed contexts (collective upload): begin, requester dedupe into s.fid, refusal in place of the lists, owner translation
int dist_keys_begin(lctr_ctx* c);
int dist_keys_dedupe(lctr_ctx* c, Slot& s, const uint64_t* h_keys, int64_t nnz);
int dist_keys_refuse(lctr_ctx* c, int slot);
int dist_keys_translate(lctr_ctx* c, int slot);
size_t dist_bytes(const lctr_ctx* c);
int mlp_alloc(lctr_ctx* c);
int mlp_reserve(lctr_ctx* c, int64_t rows);
bool ffm_grouped_supported(const lctr_ctx* c);
int ffm_grouped_reserve(lctr_ctx* c, int64_t rows);
int launch_ffm_forward_tiles(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_ffm_score(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool as_step);
int launch_ffm_backward_grouped(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int wnd_reserve(lctr_ctx* c, int64_t rows);
int launch_wnd_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_wnd_backward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_wnd_pred(lctr_ctx* c, Slot& s, const float* mlp_out, int64_t rb, int64_t re);
// width of the dense chain's input: k (NFM bi-interaction) or Fc * d (Wide&Deep concat)
inline size_t mlp_in0(const lctr_cfg& cf) {
    return cf.model == LCTR_MODEL_WND ? (size_t)cf.field_cnt * cf.factor_cnt : (size_t)cf.factor_cnt;
}
int mlp_sync_dense_grad(lctr_ctx* c);
// scan + clear of a permuted byte map (fm_fused.cuh): appends the ids of the set positions to uniq, counts in *n_uniq
int launch_slotmap_compact(lctr_ctx* c, uint8_t* mark, size_t T, uint32_t* uniq, unsigned int* n_uniq, cudaStream_t st);
int launch_ffm_warp(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats, bool train);  // 0 launched, -1 shape not covered, 1 error
int mlp_bf16_prepare(lctr_ctx* c);
int mlp_bf16_refresh(lctr_ctx* c, int layer);
int launch_nfm_mlp_bf16(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int64_t rows_divisor);
int launch_nfm_mlp(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int64_t rows_divisor);
// lctr_score's dense chain on the rows staged in c->z (rows [rb, re) of the slot): pred = sigmoid(wide + out) by the step's
// kernels without loss, backward or update (fp32: the reference-order layers; bf16: the forward-only tensor-core instances)
int launch_mlp_bf16_forward(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int launch_dense_score(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
// keyed mode (keys.cu)
int keys_alloc(lctr_ctx* c);
size_t keys_bytes(const lctr_ctx* c);
int keys_translate(lctr_ctx* c, const uint64_t* h_keys, int64_t n, bool insert, uint32_t* fid);
// the translate's key scratch, room for n keys (valid until the next keyed call), and the translation of its first n keys
int keys_scratch(lctr_ctx* c, size_t n, uint64_t** d_keys);
int keys_translate_scratch(lctr_ctx* c, int64_t n, bool insert, uint32_t* fid);
// fails naming `who` when one of the n keys is ~0, the empty marker of the key table
int check_keys_reserved(const uint64_t* keys, int64_t n, const char* who);
int keys_restore(lctr_ctx* c, const uint64_t* row_key, uint64_t n);
int keys_download(lctr_ctx* c, std::vector<uint64_t>& out);
// key_evict = 1: the upload clock and the stamps of rows [0, n) (checkpoints)
bool keys_tracked(const lctr_ctx* c);
int keys_download_stamps(lctr_ctx* c, uint64_t n, std::vector<uint64_t>& stamps, uint64_t* clock);
int keys_restore_stamps(lctr_ctx* c, const uint64_t* stamps, uint64_t n, uint64_t clock);
// cfg.key_host_rows > 0: the host tier's arrays (pinned host memory, rows [0, n) live), p[] in the order of the row
// sections (W, V, s1W, s1V, s2W, s2V); false without a tier.  keys_tier_restore: the arrays hold n rows, rebuild the index
struct TierRows {
    unsigned long long *key, *stamp;
    float* p[6];
    size_t n, cap;
};
bool keys_tier(const lctr_ctx* c, TierRows* out);
int keys_tier_restore(lctr_ctx* c, uint64_t n);
// frequency admission (lctr_set_key_admission): the compaction of the slot after an insert-upload that dropped entries
// (*nnz in: the entries uploaded, out: those kept); the settings (false when off) and the sketch for checkpoints
int keys_admission_compact(lctr_ctx* c, Slot& s, cudaStream_t st, int64_t rows, int64_t* nnz);
bool keys_admission(const lctr_ctx* c, uint32_t* min_count, uint32_t* log2_width);
int keys_admission_download(lctr_ctx* c, std::vector<uint32_t>& sketch);
int keys_admission_restore(lctr_ctx* c, const uint32_t* sketch);
// rows of the row-indexed parameter / optimizer-state transfers: F, or the capacity in keyed mode (the null row stays out)
inline size_t api_rows(const lctr_ctx* c) { return c->keys ? c->F - 1 : c->F; }
// global rows < rows that rank holds when global row g lives on rank g % world (at local row g / world); rank < world
inline size_t owned_rows(size_t rows, size_t world, size_t rank) { return (rows + world - 1 - rank) / world; }
// the s1 value lctr_create gives every row: the PS Adagrad / DCASGDA rules start data_accum at 1e-7 (paramserver.h:323)
inline float initial_s1(const lctr_cfg& cf) {
    return cf.optimizer == LCTR_OPT_PS_ADAGRAD || cf.optimizer == LCTR_OPT_PS_DCASGDA ? 1e-7f : 0.f;
}
// W, V, s1 and s2 of this rank's shard back to the state lctr_create gives (capi.cu)
int reset_table_rows(lctr_ctx* c);
// change tracking (delta.cu): no parent yet, a parent file, or none because the last load resharded another world's save
enum { PARENT_NONE = 0, PARENT_FILE = 1, PARENT_RESHARDED = 2 };
// every call below returns 0 without launching while tracking is off.  Marks: the rows the entries of slot rows
// [rb, re) name (hdr non-null: re = hdr[0], the graph pipeline's device header), on stream st; the rows of a device list
// of at most max_n rows whose length is *dev_n (null: max_n); every row
int track_mark_entries(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, const int64_t* hdr, cudaStream_t st);
int track_mark_rows(lctr_ctx* c, const uint32_t* rows, const unsigned int* dev_n, size_t max_n);
int track_mark_rows64(lctr_ctx* c, const int64_t* rows, size_t n);
int track_mark_all(lctr_ctx* c);
// the change map cleared and `hash` made the parent (after a save or in-place load while tracking)
int track_set_parent(lctr_ctx* c, uint64_t hash);
// the changed rows as an ascending device list (*m of them; list holds Fl entries) by the eviction's count / scan / index
// kernels (keys.cu)
int flags_to_list(lctr_ctx* c, const uint8_t* flags, size_t n, uint32_t* list, size_t* m);
// rows [lo, hi) of a keyed table back to the state lctr_create gives, key and stamp included (keys.cu)
int keys_reset_rows(lctr_ctx* c, size_t lo, size_t hi);
// single-slot uploads (capi.cu): room in the slot for rows x nnz, and the common end once the batch sits in the slot
int slot_fit(lctr_ctx* c, Slot& s, int64_t rows, int64_t nnz);
// weighted slots (capi.cu): the statistics of rows [rb, re) as sum w loss and sum w [correct], from the step's predictions,
// written over what the step's kernels published
int launch_weighted_stats(lctr_ctx* c, Slot& s, int64_t rb, int64_t re);
int upload_tail(lctr_ctx* c, cudaStream_t st, int slot, int64_t rows, int64_t nnz, bool keyed, const int64_t* h_row_ptr,
                const uint32_t* h_fid, const float* h_val);

}  // namespace lctr

#include "launch.cuh"  // launch(): every kernel launch of the library
