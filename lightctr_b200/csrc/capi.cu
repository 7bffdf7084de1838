// lightctr_b200/csrc/capi.cu -- the C ABI declared in include/lightctr_b200.h.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "opt.cuh"

namespace lctr {
static thread_local std::string g_err;
void set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
}

static int slot_reserve(lctr_ctx* c, Slot& s, int64_t rows, int64_t nnz) {
    const size_t k = c->cfg.factor_cnt;
    if (rows > s.cap_rows) {
        const int64_t cap = std::max<int64_t>(rows, s.cap_rows + s.cap_rows / 2);
        const size_t n = (size_t)cap, nk = c->cfg.model != LCTR_MODEL_FFM ? n * k : 0;
        s.rows = 0; s.cap_rows = 0;
        if (alloc_group(sized(s.row_ptr, n + 1), sized(s.label, n), sized(s.pred, n), sized(s.wide, n), sized(s.sumvx, nk)))
            return 1;
        if (nk) LCTR_CUDA(cudaMemsetAsync(s.sumvx, 0, nk * sizeof(float), c->stream));
        s.cap_rows = cap;
    }
    if (nnz > s.cap_nnz) {
        const int64_t cap = std::max<int64_t>(nnz, s.cap_nnz + s.cap_nnz / 2);
        const size_t n = (size_t)cap + 32;
        s.nnz = 0; s.cap_nnz = 0;
        if (alloc_group(sized(s.fid, n), sized(s.field, n), sized(s.val, n))) return 1;
        s.cap_nnz = cap;
    }
    return 0;
}

__global__ void fill_value_kernel(float* p, size_t n, float v) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

int reset_table_rows(lctr_ctx* c) {
    const size_t nv = c->Fl * c->rowlen;
    const float s1 = initial_s1(c->cfg);
    LCTR_CUDA(cudaMemsetAsync(c->W, 0, c->Fl * sizeof(float), c->stream));
    LCTR_CUDA(cudaMemsetAsync(c->V, 0, nv * sizeof(float), c->stream));
    if (s1 == 0.f) {
        LCTR_CUDA(cudaMemsetAsync(c->s1W, 0, c->Fl * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->s1V, 0, nv * sizeof(float), c->stream));
    } else {
        const Launch l{(unsigned)c->sm_count * 4, 256, 0, c->stream};
        if (launch(c, l, fill_value_kernel, c->s1W, c->Fl, s1) || launch(c, l, fill_value_kernel, c->s1V, nv, s1)) return 1;
    }
    if (c->s2W) {
        LCTR_CUDA(cudaMemsetAsync(c->s2W, 0, c->Fl * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->s2V, 0, nv * sizeof(float), c->stream));
    }
    return 0;
}

__global__ void label_to_float_kernel(const int32_t* in, float* out, int64_t n_arg, const int64_t* hdr) {
    const int64_t n = hdr ? hdr[0] : n_arg;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

// Statistics of a weighted step: sum w loss and sum w [correct] over rows [rb, re), from the predictions the step left in
// the slot and the same loss_terms as the unweighted kernels, written over the ring slot those kernels published to.
// A zero-weight row is absent; FFM (skip_zero_head) also leaves out every row whose weighted head fl(w (p - y)) is zero,
// as its kernels do
__device__ __forceinline__ void weighted_stats_rows(const float* __restrict__ pred, const float* __restrict__ label,
                                                    const float* __restrict__ rw, int64_t rb, int64_t re, int skip_zero_head,
                                                    double* partial, unsigned int* done, double* out_slot) {
    double loss = 0.0, correct = 0.0;
    for (int64_t r = rb + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < re; r += (int64_t)gridDim.x * blockDim.x) {
        const float w = rw[r];
        if (w == 0.f || (skip_zero_head && w * (pred[r] - label[r]) == 0.f)) continue;
        double l1, c1;
        loss_terms(pred[r], label[r], l1, c1);
        loss += (double)w * l1;
        correct += (double)w * c1;
    }
    publish_stats(loss, correct, partial, done, out_slot, false);
}
__global__ void weighted_stats_kernel(const float* __restrict__ pred, const float* __restrict__ label, const float* __restrict__ rw,
                                      int64_t rb, int64_t re, int skip_zero_head, double* partial, unsigned int* done,
                                      double* out_slot) {
    weighted_stats_rows(pred, label, rw, rb, re, skip_zero_head, partial, done, out_slot);
}
// the streamed step graph's instance: rows [0, hdr[0]) of the batch in the pipeline slot, read from its device header
__global__ void weighted_stats_hdr_kernel(const float* __restrict__ pred, const float* __restrict__ label,
                                          const float* __restrict__ rw, const int64_t* __restrict__ hdr, int skip_zero_head,
                                          double* partial, unsigned int* done, double* out_slot) {
    weighted_stats_rows(pred, label, rw, 0, hdr[0], skip_zero_head, partial, done, out_slot);
}

int launch_weighted_stats(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    if (re <= rb) return 0;
    const unsigned grid = (unsigned)std::min<int64_t>((re - rb + 255) / 256, (int64_t)c->sm_count * 4);
    return launch(c, {grid, 256, 0, c->stream}, weighted_stats_kernel, s.pred, s.label, s.rw, rb, re,
                  c->cfg.model == LCTR_MODEL_FFM ? 1 : 0, c->stat_partial, c->stat_done, c->stats + 2 * (c->step % kStatRing));
}

// synthetic initialisation on the device (bench only): W = 0, V[f][j] = scale * N(0,1) from a counter-based hash of
// the GLOBAL element index, so the values do not depend on how the table is sharded
__global__ void fill_params_kernel(float* __restrict__ W, float* __restrict__ V, size_t Fl, size_t rowlen, int rank,
                                   int world, unsigned long long seed, float scale) {
    const size_t n = Fl * rowlen;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t l = i / rowlen, j = i % rowlen;
        const unsigned long long g = ((unsigned long long)(l * world + rank)) * rowlen + j;
        unsigned long long h = g * 0x9E3779B97F4A7C15ull + seed;
        h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
        const float u1 = ((unsigned)(h & 0xffffffu) + 1u) * (1.0f / 16777217.0f);
        const float u2 = (unsigned)((h >> 24) & 0xffffffu) * (1.0f / 16777216.0f);
        V[i] = scale * sqrtf(-2.0f * logf(u1)) * cosf(6.2831853f * u2);
        if (j == 0) W[l] = 0.f;
    }
}

// Feature-major view of a slot, built on the host from the caller's CSR arrays (one counting sort per row
// block; stable, so each fid's entries stay in ascending row order -- the accumulation order of the
// reference's canonical single-thread run, train_fm_algo.cpp:101-116).
static int build_csc(lctr_ctx* c, Slot& s, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                     const float* val) {
    const int64_t block = c->cfg.csc_row_block ? (int64_t)c->cfg.csc_row_block : std::max<int64_t>(rows, 1);
    const int64_t nblocks = (rows + block - 1) / block;
    std::vector<int64_t> blk_seg_ptr(nblocks + 1, 0), seg_ptr;
    std::vector<uint32_t> seg_fid, ent_row((size_t)nnz);
    std::vector<float> ent_x(val ? (size_t)nnz : 0);
    seg_ptr.reserve((size_t)nnz / 4 + 16);
    seg_fid.reserve((size_t)nnz / 4 + 16);
    std::vector<uint32_t> cnt(c->F + 1, 0);
    std::vector<uint32_t> touched_list;
    int64_t out = 0;
    for (int64_t bi = 0; bi < nblocks; bi++) {
        const int64_t rb = bi * block, re = std::min(rows, rb + block);
        const int64_t eb = row_ptr[rb], ee = row_ptr[re];
        touched_list.clear();
        for (int64_t e = eb; e < ee; e++) {
            const uint32_t f = fid[e];
            if (f >= c->F) { set_error("upload_batch: fid %u >= feature_cnt %zu", f, c->F); return 1; }
            if (cnt[f]++ == 0) touched_list.push_back(f);
        }
        std::sort(touched_list.begin(), touched_list.end());
        // segment offsets for this block; cnt[f] becomes the write cursor
        for (uint32_t f : touched_list) {
            seg_fid.push_back(f);
            seg_ptr.push_back(out);
            const uint32_t n = cnt[f];
            cnt[f] = (uint32_t)(out - eb);  // cursor relative to the block (fits u32: block nnz < 2^32)
            out += n;
        }
        for (int64_t r = rb; r < re; r++)
            for (int64_t e = row_ptr[r]; e < row_ptr[r + 1]; e++) {
                const uint32_t f = fid[e];
                const int64_t pos = eb + cnt[f]++;
                ent_row[(size_t)pos] = (uint32_t)r;
                if (val) ent_x[(size_t)pos] = val[e];
            }
        for (uint32_t f : touched_list) cnt[f] = 0;
        blk_seg_ptr[bi + 1] = (int64_t)seg_fid.size();
    }
    seg_ptr.push_back(out);
    const int64_t nseg = (int64_t)seg_fid.size();
    if (nseg > s.cap_segs) {
        s.cap_segs = 0;
        if (alloc_group(sized(s.seg_ptr, (size_t)nseg + 1), sized(s.seg_fid, (size_t)nseg + 1))) return 1;
        s.cap_segs = nseg;
    }
    if (nblocks > s.cap_blocks) {
        s.cap_blocks = 0;
        if (alloc_group(sized(s.blk_seg_ptr, (size_t)nblocks + 1))) return 1;
        s.cap_blocks = nblocks;
    }
    if (nnz > s.cap_ent) {
        s.cap_ent = 0;
        if (alloc_group(sized(s.ent_row, (size_t)nnz + 32), sized(s.ent_x, (size_t)nnz + 32))) return 1;
        s.cap_ent = nnz;
    }
    LCTR_CUDA(cudaMemcpyAsync(s.seg_ptr, seg_ptr.data(), (size_t)(nseg + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (nseg) LCTR_CUDA(cudaMemcpyAsync(s.seg_fid, seg_fid.data(), (size_t)nseg * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(s.blk_seg_ptr, blk_seg_ptr.data(), (size_t)(nblocks + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (nnz) {
        LCTR_CUDA(cudaMemcpyAsync(s.ent_row, ent_row.data(), (size_t)nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        if (val) LCTR_CUDA(cudaMemcpyAsync(s.ent_x, ent_x.data(), (size_t)nnz * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the staging vectors die with this frame
    s.h_blk_seg_ptr = blk_seg_ptr;
    s.csc_block = block; s.n_blocks = nblocks; s.n_segs = nseg;
    return 0;
}
// the one place that says where a context's sparse gradient goes (GradPath, common.cuh)
static GradPath grad_path_of(const lctr_cfg& cf) {
    const int k = (int)cf.factor_cnt;
    const bool fm = cf.model == LCTR_MODEL_FM, nfm = cf.model == LCTR_MODEL_NFM;
    if ((fm || nfm) && cf.deterministic == 0 && (k == 4 || k == 8 || k == 16 || k == 32)) return GRAD_COMPACT;
    if ((fm && cf.deterministic != 0) || (nfm && cf.deterministic == 1) || (cf.model == LCTR_MODEL_FFM && cf.deterministic == 2))
        return GRAD_FEATURE_MAJOR;
    return GRAD_DENSE;
}

// room in the slot for a batch of rows x nnz; buffers are only reallocated once the stream has let go of them
int slot_fit(lctr_ctx* c, Slot& s, int64_t rows, int64_t nnz) {
    if (rows > s.cap_rows || nnz > s.cap_nnz || !s.row_ptr) {  // (!row_ptr: an empty first upload still has row_ptr[0])
        LCTR_CUDA(cudaStreamSynchronize(c->stream));  // buffers about to be reallocated may still be in use
        if (slot_reserve(c, s, std::max<int64_t>(rows, 1), nnz)) return 1;
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

// The end of every single-slot upload, once the batch sits in the slot (row_ptr, field, val; fid, or for `keyed` the rows
// the translate wrote there; s.has_val / s.has_field set) and its int32 labels in s.pred: key admission's compaction, the
// labels widened, the slot map, the grouping.  h_row_ptr / h_fid / h_val: the batch on the host, which only the host-built
// view of deterministic = 1 reads.
int upload_tail(lctr_ctx* c, cudaStream_t st, int slot, int64_t rows, int64_t nnz, bool keyed, const int64_t* h_row_ptr,
                const uint32_t* h_fid, const float* h_val) {
    Slot& s = c->slots[slot];
    s.has_rw = false;  // weights belong to the batch they were set for (key admission drops entries, never rows)
    if (keyed && c->keys) {  // key admission dropped entries: the slot holds the kept ones, before the slot map
        if (keys_admission_compact(c, s, st, rows, &nnz)) return 1;
        s.nnz = nnz;
    }
    const bool grouped = c->cfg.deterministic == 2 && rows > 0 && nnz > 0 && c->cfg.world == 1;
    int32_t* tmp = reinterpret_cast<int32_t*>(s.pred.get());  // pred is overwritten by the next forward anyway
    // labels travel as int32 and are widened on device (the reference compares a `float target`)
    if (rows && !grouped && launch(c, {(unsigned)((rows + 255) / 256), 256, 0, st}, label_to_float_kernel, tmp, s.label, rows, nullptr))
        return 1;
    s.fused_valid = false;
    s.key_state = SLOT_KEYS_OK;
    if (c->grad_path == GRAD_COMPACT || c->cfg.world > 1) {
        // slot map of the batch: the gradient rows of the compact path; on several GPUs also the key set of the pull / push
        // exchange, whose per-owner lists go out right away (posted stores, overlapping the previous step).  An empty batch
        // (0 rows or 0 entries) gets an empty map, and the compact gradient buffers are reserved all the same (a train step
        // reads them).  On several GPUs it still posts its (empty) key lists: the peers' serve waits for every rank's lists
        const bool empty = rows == 0 || nnz == 0;
        if (fused_reserve(c, s, nnz) || fused_build_slot(c, s, st, nullptr, rows, nnz)) return 1;
        if (c->cfg.world > 1 && (empty ? dist_send_empty(c, slot, st) : dist_send_keys(c, s, slot, st))) return 1;
    }
    s.csc_block = 0;
    s.dev_csc = false;
    if (grouped) {
        LCTR_CHECK(csc_device_supported(c), "cfg.deterministic=2 (device-grouped backward) needs FM with k in {4,8,16,32} "
                                            "or FFM with k %% 4 == 0 and field_cnt * k <= 512");
        if (csc_build_device(c, s, st, tmp, nullptr, rows, nnz)) return 1;  // widens the labels in its first kernel
    } else if (c->cfg.deterministic == 1 && c->cfg.model != LCTR_MODEL_FFM && rows > 0) {
        LCTR_CUDA(cudaStreamSynchronize(st));
        if (build_csc(c, s, rows, nnz, h_row_ptr, h_fid, h_val)) return 1;
    }
    return 0;
}
}  // namespace lctr

using namespace lctr;

extern "C" {

const char* lctr_last_error(void) { return g_err.c_str(); }
int lctr_abi_version(void) { return LCTR_ABI_VERSION; }

int lctr_create(const lctr_cfg* cfg, lctr_ctx** out) {
    LCTR_CHECK(cfg && out, "lctr_create: null argument");
    LCTR_CHECK(cfg->abi_version == LCTR_ABI_VERSION, "lctr_create: abi_version %u != %u", cfg->abi_version,
               LCTR_ABI_VERSION);
    LCTR_CHECK(cfg->model >= LCTR_MODEL_FM && cfg->model <= LCTR_MODEL_WND, "lctr_create: bad model %d", cfg->model);
    LCTR_CHECK(cfg->optimizer >= LCTR_OPT_ADAGRAD && cfg->optimizer <= LCTR_OPT_PS_DCASGDA, "lctr_create: bad optimizer %d",
               cfg->optimizer);
    LCTR_CHECK(cfg->key_mode == LCTR_KEYS_DENSE || cfg->key_mode == LCTR_KEYS_HASHED, "lctr_create: bad key_mode %d", cfg->key_mode);
    LCTR_CHECK(cfg->key_host_rows == 0 || (cfg->key_mode == LCTR_KEYS_HASHED && cfg->key_evict == 1 && cfg->world <= 1),
               "lctr_create: key_host_rows = %u (a host tier) needs key_mode = LCTR_KEYS_HASHED, key_evict = 1 and world = 1 "
               "(got key_mode %d, key_evict %d, world %d)", cfg->key_host_rows, cfg->key_mode, cfg->key_evict, cfg->world);
    if (cfg->key_mode == LCTR_KEYS_HASHED) {
        // exact-order modes build their feature-major view on the host from host ids, which a keyed upload does not have;
        // on several GPUs an eviction would renumber rows across the shards, which needs a collective of its own
        LCTR_CHECK(cfg->world <= 1 || cfg->max_nnz > 0,
                   "lctr_create: keyed mode on several GPUs (world %d) needs cfg.max_nnz > 0, which sizes the per-batch key "
                   "tables; without it keyed mode is single-GPU", cfg->world);
        LCTR_CHECK(cfg->world <= 1 || cfg->key_evict == 0,
                   "lctr_create: key_evict = 1 is single-GPU (world %d): evicting from a sharded keyed table is not supported", cfg->world);
        LCTR_CHECK(cfg->world <= 1 || cfg->feature_cnt >= (uint64_t)cfg->world,
                   "lctr_create: keyed capacity (feature_cnt %llu) below world %d", (unsigned long long)cfg->feature_cnt, cfg->world);
        LCTR_CHECK(cfg->deterministic == 0, "lctr_create: keyed mode needs deterministic = 0 (got %d)", cfg->deterministic);
        LCTR_CHECK(cfg->feature_cnt > 0 && cfg->feature_cnt < (1ull << 32) - 1, "lctr_create: keyed capacity (feature_cnt) out of range");
    }
    LCTR_CHECK(cfg->key_evict == 0 || cfg->key_evict == 1, "lctr_create: bad key_evict %d", cfg->key_evict);
    LCTR_CHECK(cfg->key_evict == 0 || cfg->key_mode == LCTR_KEYS_HASHED,
               "lctr_create: key_evict = 1 needs key_mode = LCTR_KEYS_HASHED (a dense table has no rows to free)");
    LCTR_CHECK(cfg->feature_cnt > 0 && cfg->feature_cnt < (1ull << 32), "lctr_create: feature_cnt out of range");
    LCTR_CHECK(cfg->factor_cnt > 0, "lctr_create: factor_cnt must be > 0");
    LCTR_CHECK(cfg->model != LCTR_MODEL_FFM || cfg->field_cnt > 0, "lctr_create: FFM needs field_cnt > 0");
    if (cfg->model == LCTR_MODEL_WND) {
        LCTR_CHECK(cfg->field_cnt > 0 && cfg->field_cnt <= 2048, "lctr_create: Wide&Deep needs 0 < field_cnt <= 2048");
        LCTR_CHECK(cfg->deterministic == 0, "lctr_create: Wide&Deep uses the RED scatter (deterministic = 0)");
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        set_error("lctr_create: no CUDA device available (%s); this library has no CPU fallback",
                  cudaGetErrorString(e));
        return 2;
    }
    LCTR_CHECK(cfg->device >= 0 && cfg->device < ndev, "lctr_create: device %d of %d", cfg->device, ndev);
    LCTR_CUDA(cudaSetDevice(cfg->device));
    std::unique_ptr<lctr_ctx, decltype(&lctr_destroy)> own(new lctr_ctx(), lctr_destroy);  // released by every failure below
    lctr_ctx* c = own.get();
    c->cfg = *cfg;
    if (c->cfg.ftrl_alpha == 0.f) {  // gradientUpdater.h:275
        c->cfg.ftrl_alpha = 0.15f; c->cfg.ftrl_lambda1 = 1.0f; c->cfg.ftrl_beta = 1.0f; c->cfg.ftrl_lambda2 = 1.0f;
    }
    if (c->cfg.world <= 0) { c->cfg.world = 1; c->cfg.rank = 0; }
    c->F = cfg->feature_cnt + (cfg->key_mode == LCTR_KEYS_HASHED ? 1 : 0);  // keyed: + the null row of unseen keys
    c->Fl = (c->F + (size_t)c->cfg.world - 1) / (size_t)c->cfg.world;
    LCTR_CHECK(c->cfg.world == 1 || !cfg->deterministic, "lctr_create: deterministic modes are single-GPU only");
    LCTR_CHECK(cfg->deterministic >= 0 && cfg->deterministic <= 2, "lctr_create: deterministic must be 0, 1 or 2");
    c->rowlen = cfg->model == LCTR_MODEL_FFM ? (size_t)cfg->field_cnt * cfg->factor_cnt : cfg->factor_cnt;
    c->grad_path = grad_path_of(c->cfg);
    const bool dense = c->grad_path == GRAD_DENSE;
    const bool update_g = dense || (cfg->model == LCTR_MODEL_FFM && c->grad_path == GRAD_FEATURE_MAJOR);
    cudaDeviceProp prop;
    LCTR_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
    c->sm_count = prop.multiProcessorCount;
    LCTR_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    const size_t FL = c->Fl;
    const size_t nv = FL * c->rowlen;
    const bool two = cfg->optimizer == LCTR_OPT_FTRL || cfg->optimizer == LCTR_OPT_ADAM || cfg->optimizer == LCTR_OPT_ADADELTA ||
                     cfg->optimizer == LCTR_OPT_PS_DCASGD || cfg->optimizer == LCTR_OPT_PS_DCASGDA;
    if (c->W.alloc(FL) || c->V.alloc(nv) || (update_g && (c->gW.alloc(FL) || c->gV.alloc(nv))) || c->s1W.alloc(FL) ||
        c->s1V.alloc(nv) || (two && (c->s2W.alloc(FL) || c->s2V.alloc(nv))))
        return 1;
    // the sparse apply of opt.cu: touched map, its compacted list and counters
    if (dense && (c->touched.alloc(FL + 512) || c->touch_list.alloc(FL + 32) || c->n_touch.alloc(1) || c->apply_done.alloc(1)))
        return 1;
    if (c->stats.alloc((size_t)2 * kStatRing) || c->stat_partial.alloc(2) || c->stat_done.alloc(1) || c->h_stats.alloc(2)) return 1;
    if (reset_table_rows(c)) return 1;
    if (update_g) {
        LCTR_CUDA(cudaMemsetAsync(c->gW, 0, FL * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->gV, 0, nv * sizeof(float), c->stream));
    }
    if (dense) {
        LCTR_CUDA(cudaMemsetAsync(c->touched, 0, FL + 512, c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->n_touch, 0, sizeof(unsigned int), c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->apply_done, 0, sizeof(unsigned int), c->stream));
    }
    if (c->cfg.world > 1) {
        if (dist_alloc(c)) return 1;
    } else {
        c->cW = c->W; c->cV = c->V; c->cgW = c->gW; c->cgV = c->gV;
    }
    LCTR_CUDA(cudaMemsetAsync(c->stats, 0, sizeof(double) * 2 * kStatRing, c->stream));
    LCTR_CUDA(cudaMemsetAsync(c->stat_partial, 0, sizeof(double) * 2, c->stream));
    LCTR_CUDA(cudaMemsetAsync(c->stat_done, 0, sizeof(unsigned int), c->stream));
    if (cfg->model == LCTR_MODEL_NFM || cfg->model == LCTR_MODEL_WND) {
        if (mlp_alloc(c)) return 1;
    }
    if (cfg->key_mode == LCTR_KEYS_HASHED && keys_alloc(c)) return 1;
    { const char* e = getenv("LCTR_CSC_IN_STEP"); c->csc_in_step = e && e[0] == '1'; }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    *out = own.release();
    return 0;
}

int lctr_destroy(lctr_ctx* c) {
    if (!c) return 0;
    cudaSetDevice(c->cfg.device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    if (c->build_stream) cudaStreamSynchronize(c->build_stream);
    if (c->dist) dist_close_peers(c);
    for (PipeGraph& g : c->pipe_graph) {
        if (g.build) cudaGraphExecDestroy(g.build);
        if (g.step) cudaGraphExecDestroy(g.step);
    }
    if (c->copy_stream) {
        for (int i = 0; i < kPipe; i++) { cudaEventDestroy(c->ev_copied[i]); cudaEventDestroy(c->ev_computed[i]); cudaEventDestroy(c->ev_h2d[i]); }
        if (c->build_stream) cudaStreamDestroy(c->build_stream);
        for (int i = 0; i < kStatRing; i++) cudaEventDestroy(c->ev_stat[i]);
        cudaStreamDestroy(c->copy_stream);
    }
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;  // its buffers release themselves
    return 0;
}

int lctr_sync(lctr_ctx* c) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

// world > 1: W / V are the FULL (global) arrays; each rank keeps / returns only the rows it owns (fid % world == rank)
int lctr_upload_params(lctr_ctx* c, const float* W, const float* V) {
    LCTR_CHECK(c, "null ctx");
    const int R = c->cfg.world, me = c->cfg.rank;
    if (R == 1) {
        if (W) LCTR_CUDA(cudaMemcpyAsync(c->W, W, api_rows(c) * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if (V) LCTR_CUDA(cudaMemcpyAsync(c->V, V, api_rows(c) * c->rowlen * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if ((W || V) && track_mark_all(c)) return 1;
    } else {
        std::vector<float> w, v;
        if (W) {
            w.assign(c->Fl, 0.f);
            for (size_t f = (size_t)me, l = 0; f < api_rows(c); f += R, l++) w[l] = W[f];
            LCTR_CUDA(cudaMemcpyAsync(c->W, w.data(), c->Fl * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        }
        if (V) {
            v.assign(c->Fl * c->rowlen, 0.f);
            for (size_t f = (size_t)me, l = 0; f < api_rows(c); f += R, l++)
                memcpy(&v[l * c->rowlen], V + f * c->rowlen, c->rowlen * sizeof(float));
            LCTR_CUDA(cudaMemcpyAsync(c->V, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        }
        if ((W || V) && track_mark_all(c)) return 1;
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        return 0;
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_download_params(lctr_ctx* c, float* W, float* V) {
    LCTR_CHECK(c, "null ctx");
    const int R = c->cfg.world, me = c->cfg.rank;
    if (R == 1) {
        if (W) LCTR_CUDA(cudaMemcpyAsync(W, c->W, api_rows(c) * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (V) LCTR_CUDA(cudaMemcpyAsync(V, c->V, api_rows(c) * c->rowlen * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        return 0;
    }
    std::vector<float> w(c->Fl), v(c->Fl * c->rowlen);
    LCTR_CUDA(cudaMemcpyAsync(w.data(), c->W, w.size() * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(v.data(), c->V, v.size() * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    for (size_t f = (size_t)me, l = 0; f < api_rows(c); f += R, l++) {
        if (W) W[f] = w[l];
        if (V) memcpy(V + f * c->rowlen, &v[l * c->rowlen], c->rowlen * sizeof(float));
    }
    return 0;
}
int lctr_fill_params(lctr_ctx* c, uint64_t seed, float scale) {
    LCTR_CHECK(c, "null ctx");
    if (launch(c, {(unsigned)c->sm_count * 8, 256, 0, c->stream}, fill_params_kernel, c->W, c->V, c->Fl, c->rowlen, c->cfg.rank,
               c->cfg.world, (unsigned long long)seed, scale) || track_mark_all(c))
        return 1;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
// world > 1: the rows a rank owns are the prefix [0, n) of its shard (local row l = global row l * world + rank); the
// opt-state transfers move that prefix between the shard and the full global arrays [W part | V part]
static int shard_to_global(lctr_ctx* c, float* out, const float* dW, const float* dV) {
    const size_t F = api_rows(c), R = (size_t)c->cfg.world, n = owned_rows(F, R, c->cfg.rank), k = c->rowlen;
    std::vector<float> w(n), v(n * k);
    if (n) {
        LCTR_CUDA(cudaMemcpyAsync(w.data(), dW, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(v.data(), dV, n * k * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    for (size_t l = 0, f = (size_t)c->cfg.rank; l < n; l++, f += R) {
        out[f] = w[l];
        memcpy(out + F + f * k, &v[l * k], k * sizeof(float));
    }
    return 0;
}
static int global_to_shard(lctr_ctx* c, const float* in, float* dW, float* dV) {
    const size_t F = api_rows(c), R = (size_t)c->cfg.world, n = owned_rows(F, R, c->cfg.rank), k = c->rowlen;
    std::vector<float> w(n), v(n * k);
    for (size_t l = 0, f = (size_t)c->cfg.rank; l < n; l++, f += R) {
        w[l] = in[f];
        memcpy(&v[l * k], in + F + f * k, k * sizeof(float));
    }
    if (n) {
        LCTR_CUDA(cudaMemcpyAsync(dW, w.data(), n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(dV, v.data(), n * k * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_download_opt_state(lctr_ctx* c, float* s1, float* s2) {
    LCTR_CHECK(c, "null ctx");
    if (c->cfg.world > 1) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        if (s1 && shard_to_global(c, s1, c->s1W, c->s1V)) return 1;
        if (s2 && c->s2W && shard_to_global(c, s2, c->s2W, c->s2V)) return 1;
        return 0;
    }
    const size_t F = api_rows(c), nv = F * c->rowlen;
    if (s1) {
        LCTR_CUDA(cudaMemcpyAsync(s1, c->s1W, F * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(s1 + F, c->s1V, nv * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    if (s2 && c->s2W) {
        LCTR_CUDA(cudaMemcpyAsync(s2, c->s2W, F * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(s2 + F, c->s2V, nv * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_upload_opt_state(lctr_ctx* c, const float* s1, const float* s2) {
    LCTR_CHECK(c, "null ctx");
    if (c->cfg.world > 1) {
        if (s1 && global_to_shard(c, s1, c->s1W, c->s1V)) return 1;
        if (s2 && c->s2W && global_to_shard(c, s2, c->s2W, c->s2V)) return 1;
        if ((s1 || (s2 && c->s2W)) && (track_mark_all(c) || cudaStreamSynchronize(c->stream) != cudaSuccess)) return 1;
        return 0;
    }
    const size_t F = api_rows(c), nv = F * c->rowlen;
    if (s1) {
        LCTR_CUDA(cudaMemcpyAsync(c->s1W, s1, F * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(c->s1V, s1 + F, nv * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    }
    if (s2 && c->s2W) {
        LCTR_CUDA(cudaMemcpyAsync(c->s2W, s2, F * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(c->s2V, s2 + F, nv * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    }
    if ((s1 || (s2 && c->s2W)) && track_mark_all(c)) return 1;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

// fid_resident: the slot's fid array already holds the batch (keyed uploads translate into it before this runs)
static int upload_batch_on(lctr_ctx* c, cudaStream_t st, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr,
                           const uint32_t* fid, const uint16_t* field, const float* val, const int32_t* label,
                           bool fid_resident = false) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    LCTR_CHECK(rows >= 0 && nnz >= 0 && row_ptr && (nnz == 0 || fid || fid_resident) && (rows == 0 || label), "upload_batch: null input");
    LCTR_CHECK((c->cfg.model != LCTR_MODEL_FFM && c->cfg.model != LCTR_MODEL_WND) || field || nnz == 0,
               "upload_batch: FFM / Wide&Deep need the field array");
    Slot& s = c->slots[slot];
    s.has_rw = false;
    if (slot_fit(c, s, rows, nnz)) return 1;
    s.rows = rows; s.nnz = nnz;
    s.has_val = val != nullptr;
    s.has_field = field != nullptr;
    LCTR_CUDA(cudaMemcpyAsync(s.row_ptr, row_ptr, (size_t)(rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    if (nnz) {
        if (!fid_resident) LCTR_CUDA(cudaMemcpyAsync(s.fid, fid, (size_t)nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        if (field) LCTR_CUDA(cudaMemcpyAsync(s.field, field, (size_t)nnz * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
        if (val) LCTR_CUDA(cudaMemcpyAsync(s.val, val, (size_t)nnz * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    if (rows) LCTR_CUDA(cudaMemcpyAsync(s.pred, label, (size_t)rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return upload_tail(c, st, slot, rows, nnz, fid_resident, row_ptr, fid, val);
}

// the CSR structure of an upload (`who` prefixes the messages): row_ptr from 0 to nnz, never decreasing, and the fields
// below field_cnt where the model reads them
static int check_csr(const lctr_ctx* c, const char* who, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint16_t* field) {
    LCTR_CHECK(row_ptr[0] == 0 && row_ptr[rows] == nnz, "%s: row_ptr must run from 0 to nnz (%lld .. %lld, nnz %lld)", who,
               (long long)row_ptr[0], (long long)row_ptr[rows], (long long)nnz);
    for (int64_t r = 0; r < rows; r++)
        LCTR_CHECK(row_ptr[r] <= row_ptr[r + 1], "%s: row_ptr decreases at row %lld", who, (long long)r);
    if ((c->cfg.model == LCTR_MODEL_FFM || c->cfg.model == LCTR_MODEL_WND) && field)
        for (int64_t i = 0; i < nnz; i++)
            LCTR_CHECK(field[i] < c->cfg.field_cnt, "%s: field %u at entry %lld >= field_cnt %u", who, (unsigned)field[i],
                       (long long)i, c->cfg.field_cnt);
    return 0;
}

int lctr_upload_batch(lctr_ctx* c, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                      const uint16_t* field, const float* val, const int32_t* label) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(!c->keys, "lctr_upload_batch: keyed context (key_mode = LCTR_KEYS_HASHED): use lctr_upload_batch_keys");
    // Resident datasets are validated once, on the host: an out-of-range id would otherwise surface as an illegal
    // address inside a gather (the reference indexes W / V unchecked too, fm_algo_abst.h:146-151, but there feature_cnt
    // is derived from the same file).  The streamed entry points (lctr_train_batch[_async]) trust their caller.
    LCTR_CHECK(rows >= 0 && nnz >= 0 && row_ptr && (nnz == 0 || fid), "upload_batch: null input");
    if (check_csr(c, "upload_batch", rows, nnz, row_ptr, field)) return 1;
    for (int64_t i = 0; i < nnz; i++)
        LCTR_CHECK(fid[i] < c->F, "upload_batch: fid %u at entry %lld >= feature_cnt %zu", fid[i], (long long)i, c->F);
    return upload_batch_on(c, c->stream, slot, rows, nnz, row_ptr, fid, field, val, label);
}

// the arguments of a keyed upload, checked on the host before anything is sent
static int check_batch_keys(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint64_t* key,
                            const uint16_t* field, const int32_t* label) {
    LCTR_CHECK(rows >= 0 && nnz >= 0 && row_ptr && (nnz == 0 || key) && (rows == 0 || label), "upload_batch_keys: null input");
    if (check_csr(c, "upload_batch_keys", rows, nnz, row_ptr, field)) return 1;
    if (check_keys_reserved(key, nnz, "upload_batch_keys")) return 1;
    LCTR_CHECK((c->cfg.model != LCTR_MODEL_FFM && c->cfg.model != LCTR_MODEL_WND) || field || nnz == 0,
               "upload_batch_keys: FFM / Wide&Deep need the field array");
    return 0;
}

// world > 1: a collective call (every rank, same slot, same order).  Requester: dedupe, slot map, keyed lists to the owners;
// owner: translation of what it received (dist.cu).  A rank whose own part fails still takes part with a refusal, so every
// rank returns: its own error, or the first failing owner's status, which every rank reports alike.
static int upload_batch_keys_dist(lctr_ctx* c, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint64_t* key,
                                  const uint16_t* field, const float* val, const int32_t* label, int insert) {
    if (dist_keys_begin(c)) return 1;
    Slot& s = c->slots[slot];
    s.key_state = SLOT_KEYS_INVALID;  // until every owner has translated the batch
    s.fused_valid = false;
    int rc = check_batch_keys(c, rows, nnz, row_ptr, key, field, label);
    if (!rc && !insert) {
        set_error("lctr_upload_batch_keys: insert = 0 is single-GPU (a sharded context predicts on slots uploaded with "
                  "insert = 1; unseen keys of a test set need a world-1 load)");
        rc = 1;
    }
    if (!rc && std::min<int64_t>(nnz, (int64_t)c->F) > (int64_t)std::min<uint64_t>(c->cfg.max_nnz ? c->cfg.max_nnz : c->F, c->F)) {
        set_error("lctr_upload_batch_keys: batch of %lld entries exceeds the key capacity of the multi-GPU context (cfg.max_nnz)",
                  (long long)nnz);
        rc = 1;
    }
    if (!rc && (rows > s.cap_rows || nnz > s.cap_nnz)) {
        rc = cudaStreamSynchronize(c->stream) != cudaSuccess || slot_reserve(c, s, rows, nnz) ||
             cudaStreamSynchronize(c->stream) != cudaSuccess;
        if (rc && g_err.empty()) set_error("lctr_upload_batch_keys: slot buffers could not be reserved");
    }
    if (!rc && nnz > 0) rc = dist_keys_dedupe(c, s, key, nnz);  // an empty share posts empty lists (upload_batch_on)
    if (!rc) rc = upload_batch_on(c, c->stream, slot, rows, nnz, row_ptr, nullptr, field, val, label, true);
    std::string own;
    if (rc) {
        own = g_err;
        s.key_state = SLOT_KEYS_INVALID;
        if (dist_keys_refuse(c, slot)) return 1;
    }
    const int xrc = dist_keys_translate(c, slot);
    if (rc) {
        g_err = own;
        return 1;
    }
    if (xrc) {
        s.key_state = SLOT_KEYS_INVALID;
        return 1;
    }
    s.key_state = SLOT_KEYS_OK;
    return 0;
}

int lctr_upload_batch_keys(lctr_ctx* c, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint64_t* key,
                           const uint16_t* field, const float* val, const int32_t* label, int insert) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_upload_batch_keys: the context was not created with key_mode = LCTR_KEYS_HASHED");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    if (c->cfg.world > 1) return upload_batch_keys_dist(c, slot, rows, nnz, row_ptr, key, field, val, label, insert);
    if (check_batch_keys(c, rows, nnz, row_ptr, key, field, label)) return 1;
    Slot& s = c->slots[slot];
    if (rows > s.cap_rows || nnz > s.cap_nnz) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));  // buffers about to be reallocated may still be in use
        if (slot_reserve(c, s, rows, nnz)) return 1;
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    s.key_state = SLOT_KEYS_INVALID;  // until the whole upload has succeeded
    s.fused_valid = false;
    if (keys_translate(c, key, nnz, insert != 0, s.fid)) return 1;
    if (upload_batch_on(c, c->stream, slot, rows, nnz, row_ptr, nullptr, field, val, label, true)) {
        s.key_state = SLOT_KEYS_INVALID;
        return 1;
    }
    s.key_state = insert ? SLOT_KEYS_OK : SLOT_KEYS_LOOKUP;
    return 0;
}

int lctr_set_row_weights(lctr_ctx* c, int slot, int64_t rows, const float* weight) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "lctr_set_row_weights: slot %d out of range", slot);
    Slot& s = c->slots[slot];
    if (!weight) {
        s.has_rw = false;
        return 0;
    }
    LCTR_CHECK(s.rows > 0, "lctr_set_row_weights: slot %d holds no rows", slot);
    LCTR_CHECK(rows == s.rows, "lctr_set_row_weights: %lld weights for the %lld rows of slot %d", (long long)rows, (long long)s.rows,
               slot);
    for (int64_t r = 0; r < rows; r++)
        LCTR_CHECK(std::isfinite(weight[r]) && weight[r] >= 0.f, "lctr_set_row_weights: weight %g of row %lld is not a finite "
                   "value >= 0", (double)weight[r], (long long)r);
    s.has_rw = false;  // until the new weights are in place
    if (rows > s.cap_rw) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));  // a step may still read the old array
        s.cap_rw = 0;
        if (alloc_group(sized(s.rw, (size_t)s.cap_rows))) return 1;
        s.cap_rw = s.cap_rows;
    }
    LCTR_CUDA(cudaMemcpyAsync(s.rw, weight, (size_t)rows * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the caller's buffer may be reused on return
    s.has_rw = true;
    return 0;
}

static int read_stats(lctr_ctx* c, uint64_t step, float* loss_sum, float* acc_cnt) {
    if (!loss_sum && !acc_cnt) return 0;
    if (c->cfg.world > 1 && dist_check_overflow(c)) return 1;
    LCTR_CUDA(cudaMemcpyAsync(c->h_stats, c->stats + 2 * (step % kStatRing), 2 * sizeof(double), cudaMemcpyDeviceToHost,
                              c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (loss_sum) *loss_sum = (float)c->h_stats[0];
    if (acc_cnt) *acc_cnt = (float)c->h_stats[1];
    return 0;
}

// the slot of a forward entry point (`who` prefixes the messages): in range, holding a usable batch that has rows [rb, re).
// A keyed slot uploaded with insert = 0 is refused for training only
static int check_slot(lctr_ctx* c, const char* who, int slot, int64_t rb, int64_t re, bool train) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    const Slot& s = c->slots[slot];
    LCTR_CHECK(s.key_state != SLOT_KEYS_INVALID, "%s: slot %d holds no usable batch (its last keyed upload failed)", who, slot);
    LCTR_CHECK(!train || s.key_state != SLOT_KEYS_LOOKUP, "%s: slot %d was uploaded with insert = 0 (lookup only: unseen "
                                                          "keys sit on the null row, which is never trained)", who, slot);
    LCTR_CHECK(s.key_state != SLOT_KEYS_STALE, "%s: slot %d is stale: lctr_evict_keys or a keyed checkpoint load renumbered "
                                               "rows after it was uploaded; upload it again", who, slot);
    LCTR_CHECK(rb >= 0 && re <= s.rows && rb <= re, "%s: rows [%lld,%lld) outside slot (%lld rows)", who, (long long)rb,
               (long long)re, (long long)s.rows);
    return 0;
}

// one train step over rows [rb, re) of the slot, statistics into the ring slot of the step; a weighted slot launches its
// weighted statistics when weighted_stats is set (the caller reads them)
static int train_step_on(lctr_ctx* c, int slot, int64_t rb, int64_t re, bool weighted_stats) {
    if (check_slot(c, "train_step", slot, rb, re, true)) return 1;
    Slot& s = c->slots[slot];
    LCTR_CHECK(c->cfg.world == 1 || c->cfg.minibatch_size > 0,
               "train_step: multi-GPU contexts need cfg.minibatch_size = the GLOBAL batch (the updater's divisor)");
    const uint64_t step = c->step;
    const bool multi = c->cfg.world > 1;
    const int64_t rows = re - rb;
    int rc = 0;
    if (rows == 0)  // no forward publishes this step's statistics
        LCTR_CUDA(cudaMemsetAsync(c->stats + 2 * (step % kStatRing), 0, 2 * sizeof(double), c->stream));
    if (c->csc_in_step && c->cfg.deterministic == 2 && c->cfg.world == 1 && rb == 0 && re == s.rows && s.nnz > 0) {
        // bench mode: the grouping of the batch (count / scan / fill) is part of the timed step instead of the upload
        ProfScope prof(c, PROF_CSC_BUILD);
        if (csc_build_device(c, s, c->stream, nullptr, nullptr, s.rows, s.nnz)) return 1;
    }
    // Several GPUs: the rows come from the owners' shards into the batch-compact cache (dist_pre_step) and the gradient rows
    // go back to their owners, who merge and update (dist_post_step).  NFM / Wide&Deep: dense layers replicated, their
    // gradients all-reduced (launch_nfm_mlp).
    const bool fm = c->cfg.model == LCTR_MODEL_FM;
    switch (c->grad_path) {
        case GRAD_COMPACT:  // FM / NFM: one gather, RED scatter into the batch-compact buffer (fm_fused.cu), compact updater
            if (!multi && rows == 0) break;  // nothing to update; on several GPUs the rank still joins the exchange
            rc = (multi && dist_pre_step(c, s, slot, true)) ||
                 (fm ? launch_fm_fused(c, s, rb, re, true, nullptr, nullptr)
                     : mlp_reserve(c, rows) || launch_nfm_forward_fused(c, s, rb, re) || launch_nfm_mlp(c, s, rb, re, rows) ||
                           launch_nfm_backward_fused(c, s, rb, re)) ||
                 (multi ? dist_post_step(c, s, slot, rows) : launch_apply_compact(c, s, rows, nullptr, nullptr));
            break;
        case GRAD_FEATURE_MAJOR:  // one GPU: the updater runs inside the backward
            if (c->cfg.model == LCTR_MODEL_FFM)
                rc = ffm_grouped_reserve(c, s.rows) || launch_ffm_forward_tiles(c, s, rb, re) || launch_ffm_backward_grouped(c, s, rb, re);
            else if (fm)
                rc = launch_fm_forward(c, s, rb, re, false, true) ||
                     (c->cfg.deterministic == 2 ? launch_fm_backward_devcsc(c, s, rb, re) : launch_fm_backward_csc(c, s, rb, re, false));
            else
                rc = mlp_reserve(c, rows) || launch_fm_forward(c, s, rb, re, true, false) || launch_nfm_mlp(c, s, rb, re, rows) ||
                     launch_fm_backward_csc(c, s, rb, re, true);
            break;
        case GRAD_DENSE:  // REDs into update_g (one GPU) or the exchange's gradient rows (several), then the sparse apply
            if (multi && dist_pre_step(c, s, slot, false)) return 1;
            switch (c->cfg.model) {
                case LCTR_MODEL_FM: rc = launch_fm_forward(c, s, rb, re, false, true) || launch_fm_backward(c, s, rb, re, false); break;
                case LCTR_MODEL_FFM: rc = launch_ffm_forward(c, s, rb, re); break;
                case LCTR_MODEL_WND:
                    rc = mlp_reserve(c, rows) || wnd_reserve(c, rows) || launch_wnd_forward(c, s, rb, re) ||
                         launch_nfm_mlp(c, s, rb, re, rows) || launch_wnd_backward(c, s, rb, re);
                    break;
                case LCTR_MODEL_NFM:
                    rc = mlp_reserve(c, rows) || launch_fm_forward(c, s, rb, re, true, false) || launch_nfm_mlp(c, s, rb, re, rows) ||
                         launch_fm_backward(c, s, rb, re, true);
                    break;
            }
            rc = rc || (multi ? dist_post_step(c, s, slot, rows) : launch_apply(c, rows));
            break;
    }
    // a weighted slot's statistics are the weighted sums, computed from the step's predictions once its kernels are done,
    // when the caller reads them
    if (!rc && s.has_rw && weighted_stats) rc = launch_weighted_stats(c, s, rb, re);
    // change tracking: the rows the stepped entries name, behind the updater (several GPUs: the owner marks the rows it
    // served, dist_post_step)
    if (rc || (!multi && track_mark_entries(c, s, rb, re, nullptr, c->stream))) return 1;
    c->step++;
    return 0;
}

int lctr_train_step(lctr_ctx* c, int slot, int64_t rb, int64_t re, float* loss_sum, float* acc_cnt) {
    const uint64_t step = c ? c->step : 0;
    if (train_step_on(c, slot, rb, re, loss_sum || acc_cnt)) return 1;
    return read_stats(c, step, loss_sum, acc_cnt);
}

// The forward of lctr_score / lctr_predict on rows [rb, re) of the slot, with statistics off and the forward-only instances
// of the kernels that fuse a backward.  as_step (lctr_score): FFM runs the kernel the train step chooses, so the pCTR is
// the step's; otherwise (lctr_predict) the plain CTA-per-sample kernel.  The other models run the step's launchers for both.
// NFM and Wide&Deep run their rows in blocks of at most max(kScoreBlock, the rows the dense scratch already holds), which
// bounds c->z, the fp32 activations and the Wide&Deep source map whatever the slot's size.  On several GPUs the rows are
// already pulled into the cache.
constexpr int64_t kScoreBlock = 65536;
static int score_rows(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool as_step) {
    const bool compact = c->grad_path == GRAD_COMPACT;
    switch (c->cfg.model) {
        case LCTR_MODEL_FM:  // the order-free step's forward is MODE 0 of its kernel family
            return compact ? launch_fm_forward_tree(c, s, rb, re, false) : launch_fm_forward(c, s, rb, re, false, false);
        case LCTR_MODEL_FFM: return launch_ffm_score(c, s, rb, re, as_step);
        default: break;
    }
    const bool wnd = c->cfg.model == LCTR_MODEL_WND;
    const int64_t block = std::max<int64_t>(kScoreBlock, (int64_t)c->mlp_cap_rows);
    for (int64_t b = rb; b < re; b += block) {
        const int64_t e = std::min(re, b + block);
        if (mlp_reserve(c, e - b) || (wnd && wnd_reserve(c, e - b))) return 1;
        const int rc = wnd ? launch_wnd_forward(c, s, b, e)
                     : compact ? launch_nfm_forward_fused(c, s, b, e) : launch_fm_forward(c, s, b, e, true, false);
        if (rc || launch_dense_score(c, s, b, e)) return 1;
    }
    return 0;
}

// score_rows, and the pCTR to pctr.  On several GPUs a collective pull-only round (dist.cu): the owners serve the slot's
// rows from their shards into the batch-compact cache, the forward runs on that cache and the cache is released to the
// owners.  No push, merge or updater; the step counter does not advance.
static int forward_round(lctr_ctx* c, Slot& s, int slot, int64_t rb, int64_t re, bool as_step, float* pctr) {
    if (c->cfg.world > 1) {
        // the forward waits for the owners' rows as the step's does: in-kernel on the order-free path, behind a wait kernel
        // otherwise
        if (dist_pre_step(c, s, slot, c->grad_path == GRAD_COMPACT, false)) return 1;
        const int rc = score_rows(c, s, rb, re, as_step);
        if (dist_release(c)) return 1;  // also after a failed forward: the owners' next serve waits for it
        if (rc) return 1;
        if (dist_check_overflow(c)) return 1;  // a truncated key list gives no pCTR
    } else if (score_rows(c, s, rb, re, as_step)) {
        return 1;
    }
    if (pctr && re > rb) {
        LCTR_CUDA(cudaMemcpyAsync(pctr, s.pred + rb, (size_t)(re - rb) * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

int lctr_score(lctr_ctx* c, int slot, int64_t rb, int64_t re, float* pctr) {
    if (check_slot(c, "lctr_score", slot, rb, re, false)) return 1;
    return forward_round(c, c->slots[slot], slot, rb, re, true, pctr);
}

int lctr_train_batch(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                     const uint16_t* field, const float* val, const int32_t* label, float* loss_sum, float* acc_cnt) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(!c->keys, "lctr_train_batch: keyed context: upload with lctr_upload_batch_keys, then lctr_train_step");
    if (lctr_upload_batch(c, 0, rows, nnz, row_ptr, fid, field, val, label)) return 1;
    return lctr_train_step(c, 0, 0, rows, loss_sum, acc_cnt);
}

// ---- streamed training: copy stream + compute stream, two pipeline slots -------------------------------------
static int pipe_init(lctr_ctx* c) {
    if (c->copy_stream) return 0;
    LCTR_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    LCTR_CUDA(cudaStreamCreateWithFlags(&c->build_stream, cudaStreamNonBlocking));
    for (int i = 0; i < kPipe; i++) {
        LCTR_CUDA(cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming));
        LCTR_CUDA(cudaEventCreateWithFlags(&c->ev_computed[i], cudaEventDisableTiming));
        LCTR_CUDA(cudaEventCreateWithFlags(&c->ev_h2d[i], cudaEventDisableTiming));
    }
    for (int i = 0; i < kStatRing; i++) LCTR_CUDA(cudaEventCreateWithFlags(&c->ev_stat[i], cudaEventDisableTiming));
    return c->h_stat_ring.alloc(2 * kStatRing);
}

// Graph path of the streamed pipeline (FM, cfg.deterministic == 2, one GPU): per pipeline slot two captured graphs --
// `build` (slot header copy + the five grouping kernels, on the copy stream) and `step` (updater-parameter copy,
// forward, grouped backward + update, result copy, on the compute stream).  Kernels take the batch size from the
// device-side slot header and the updater parameters from device memory, so the graphs are static: a streamed step
// costs the host three cudaMemcpyAsync, two graph launches and four event calls instead of ~20 launches.
// *n = the kernel nodes of a captured graph
static int count_kernel_nodes(cudaGraph_t graph, int* n) {
    *n = 0;
    size_t count = 0;
    LCTR_CUDA(cudaGraphGetNodes(graph, nullptr, &count));
    std::vector<cudaGraphNode_t> nodes(count);
    LCTR_CUDA(cudaGraphGetNodes(graph, nodes.data(), &count));
    for (cudaGraphNode_t node : nodes) {
        cudaGraphNodeType t;
        LCTR_CUDA(cudaGraphNodeGetType(node, &t));
        *n += t == cudaGraphNodeTypeKernel;
    }
    return 0;
}

// weighted: the step graph takes the weighted kernel instances and ends with a weighted-statistics node over s.rw, which
// must hold cap_rows floats before the capture
static int pipe_graph_capture(lctr_ctx* c, int p, bool has_val, bool weighted) {
    PipeGraph& g = c->pipe_graph[p];
    Slot& s = c->slots[kNumSlots - kPipe + p];
    if (g.build) { cudaGraphExecDestroy(g.build); g.build = nullptr; }
    if (g.step) { cudaGraphExecDestroy(g.step); g.step = nullptr; }
    if (!g.h_stat && (g.d_hdr.alloc(2) || g.h_hdr.alloc(2) || g.d_opt.alloc(1) || g.h_opt.alloc(1) || g.d_stat.alloc(2) ||
                      g.h_stat.alloc(2)))
        return 1;
    s.has_val = has_val;
    s.has_rw = weighted;
    // the launchers pick their updater instance from the host copy at capture time: give it the context's updater
    memset(g.h_opt, 0, sizeof(OptParams));
    g.h_opt[0].opt = c->cfg.optimizer;
    cudaGraph_t graph;
    const bool fused = c->grad_path == GRAD_COMPACT;  // else device grouping (GRAD_FEATURE_MAJOR)
    // ---- build graph (copy stream)
    LCTR_CUDA(cudaStreamBeginCapture(c->copy_stream, cudaStreamCaptureModeThreadLocal));
    int rc = cudaMemcpyAsync(g.d_hdr, g.h_hdr, 2 * sizeof(int64_t), cudaMemcpyHostToDevice, c->copy_stream) != cudaSuccess;
    if (!rc) {
        if (fused) {  // labels widened, then the slot map of the batch (fm_fused.cu)
            rc = launch(c, {(unsigned)((s.cap_rows + 255) / 256), 256, 0, c->copy_stream}, label_to_float_kernel,
                        reinterpret_cast<int32_t*>(s.pred.get()), s.label, s.cap_rows, g.d_hdr) ||
                 fused_build_slot(c, s, c->copy_stream, g.d_hdr, s.cap_rows, s.cap_nnz);
        } else {
            rc = csc_build_device(c, s, c->copy_stream, reinterpret_cast<int32_t*>(s.pred.get()), g.d_hdr, s.cap_rows, s.cap_nnz);
        }
    }
    cudaError_t ce = cudaStreamEndCapture(c->copy_stream, &graph);  // always closes the capture, also on error paths
    if (rc || ce != cudaSuccess) { set_error("streamed pipeline: capture of the build graph failed (%s)", cudaGetErrorString(ce)); return 1; }
    if (count_kernel_nodes(graph, &g.build_kernels)) return 1;
    LCTR_CUDA(cudaGraphInstantiate(&g.build, graph, 0));
    cudaGraphDestroy(graph);
    // ---- step graph (compute stream)
    LCTR_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    rc = cudaMemcpyAsync(g.d_opt, g.h_opt, sizeof(OptParams), cudaMemcpyHostToDevice, c->stream) != cudaSuccess;
    if (!rc) {
        if (fused)
            rc = launch_fm_fused(c, s, 0, s.cap_rows, true, g.d_hdr, g.d_stat) ||
                 launch_apply_compact(c, s, s.cap_rows, g.h_opt, g.d_opt);
        else
            rc = launch_fm_forward_ex(c, s, 0, s.cap_rows, false, true, g.d_hdr, g.d_stat) ||
                 launch_fm_backward_devcsc_ex(c, s, 0, s.cap_rows, g.h_opt, g.d_opt);
        if (!rc && weighted)  // over what the forward wrote into d_stat
            rc = launch(c, {(unsigned)std::min<int64_t>((s.cap_rows + 255) / 256, (int64_t)c->sm_count * 4), 256, 0, c->stream},
                        weighted_stats_hdr_kernel, s.pred, s.label, s.rw, g.d_hdr, 0, c->stat_partial, c->stat_done, g.d_stat);
        if (!rc) rc = track_mark_entries(c, s, 0, 0, g.d_hdr, c->stream);
    }
    if (!rc) rc = cudaMemcpyAsync(g.h_stat, g.d_stat, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess;
    ce = cudaStreamEndCapture(c->stream, &graph);
    if (rc || ce != cudaSuccess) { set_error("streamed pipeline: capture of the step graph failed (%s)", cudaGetErrorString(ce)); return 1; }
    if (count_kernel_nodes(graph, &g.step_kernels)) return 1;
    LCTR_CUDA(cudaGraphInstantiate(&g.step, graph, 0));
    cudaGraphDestroy(graph);
    g.cap_rows = s.cap_rows; g.cap_nnz = s.cap_nnz; g.has_val = has_val; g.tracked = c->changed;
    g.weighted = weighted; g.rw = weighted ? s.rw.get() : nullptr;
    return 0;
}

static int train_batch_async_graph(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                                   const float* val, const int32_t* label, const float* weight, uint64_t* ticket) {
    const int p = (int)(c->pipe_issued % kPipe);
    const int slot = kNumSlots - kPipe + p;
    Slot& s = c->slots[slot];
    PipeGraph& g = c->pipe_graph[p];
    const bool fused = c->grad_path == GRAD_COMPACT;
    const bool weighted = weight != nullptr;
    if (rows > s.cap_rows || nnz > s.cap_nnz || !g.build || g.has_val != (val != nullptr) || g.cap_rows != s.cap_rows ||
        g.cap_nnz != s.cap_nnz || g.tracked != c->changed.get() || g.weighted != weighted || (weighted && g.rw != s.rw.get())) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->copy_stream));
        LCTR_CUDA(cudaStreamSynchronize(c->build_stream));
        if (rows > s.cap_rows || nnz > s.cap_nnz)  // head-room so that slightly larger batches do not re-capture
            if (slot_reserve(c, s, std::max(rows, s.cap_rows) + rows / 8 + 64, std::max(nnz, s.cap_nnz) + nnz / 8 + 1024)) return 1;
        if (fused ? fused_reserve(c, s, s.cap_nnz) : csc_reserve(c, s, s.cap_nnz)) return 1;
        if (weighted && s.cap_rw < s.cap_rows) {  // the graph captures the pointer: room for any batch the slot fits
            s.cap_rw = 0;
            if (alloc_group(sized(s.rw, (size_t)s.cap_rows))) return 1;
            s.cap_rw = s.cap_rows;
        }
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        if (pipe_graph_capture(c, p, val != nullptr, weighted)) return 1;
    }
    s.rows = rows; s.nnz = nnz; s.has_val = val != nullptr; s.has_field = false; s.has_rw = weighted;
    if (c->pipe_issued >= (uint64_t)kPipe) LCTR_CUDA(cudaStreamWaitEvent(c->copy_stream, c->ev_computed[p], 0));
    LCTR_CUDA(cudaMemcpyAsync(s.row_ptr, row_ptr, (size_t)(rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, c->copy_stream));
    LCTR_CUDA(cudaMemcpyAsync(s.fid, fid, (size_t)nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, c->copy_stream));
    if (val) LCTR_CUDA(cudaMemcpyAsync(s.val, val, (size_t)nnz * sizeof(float), cudaMemcpyHostToDevice, c->copy_stream));
    LCTR_CUDA(cudaMemcpyAsync(s.pred, label, (size_t)rows * sizeof(int32_t), cudaMemcpyHostToDevice, c->copy_stream));
    if (weighted) LCTR_CUDA(cudaMemcpyAsync(s.rw, weight, (size_t)rows * sizeof(float), cudaMemcpyHostToDevice, c->copy_stream));
    g.h_hdr[0] = rows; g.h_hdr[1] = nnz;
    // the batch's slot map is built on its own stream: the copy engine moves batch t+1 while the SMs build batch t's map (the
    // build kernels share scratch buffers, so they stay serialised among themselves -- on this one stream)
    LCTR_CUDA(cudaEventRecord(c->ev_h2d[p], c->copy_stream));
    LCTR_CUDA(cudaStreamWaitEvent(c->build_stream, c->ev_h2d[p], 0));
    if (launch_graph(c, g.build, g.build_kernels, c->build_stream)) return 1;
    LCTR_CUDA(cudaEventRecord(c->ev_copied[p], c->build_stream));
    LCTR_CUDA(cudaStreamWaitEvent(c->stream, c->ev_copied[p], 0));
    if (fused) fused_opt_params(c, rows, g.h_opt); else csc_opt_params(c, rows, g.h_opt);
    if (launch_graph(c, g.step, g.step_kernels, c->stream)) return 1;
    LCTR_CUDA(cudaEventRecord(c->ev_computed[p], c->stream));
    s.dev_csc = !fused;
    s.fused_valid = fused;
    g.ticket = c->step;
    *ticket = c->step++;
    c->pipe_issued++;
    return 0;
}

// lctr_train_batch_async, weighted when weight is not null
static int train_batch_async(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                             const uint16_t* field, const float* val, const int32_t* label, const float* weight,
                             uint64_t* ticket) {
    LCTR_CHECK(c && ticket, "null argument");
    LCTR_CHECK(!c->keys, "lctr_train_batch_async: the streamed pipeline takes no keyed batches (lctr_upload_batch_keys + lctr_train_step)");
    LCTR_CHECK(c->cfg.deterministic != 1, "streamed batches need cfg.deterministic 0 (RED scatter) or 2 (device grouping)");
    if (pipe_init(c)) return 1;
    LCTR_CHECK(c->pipe_issued - c->pipe_waited < (uint64_t)kPipe, "more than %d streamed batches outstanding: call lctr_wait first", kPipe);
    if (weight) {  // before anything is enqueued: a refused batch issues no ticket
        for (int64_t r = 0; r < rows; r++)
            LCTR_CHECK(std::isfinite(weight[r]) && weight[r] >= 0.f, "lctr_train_batch_weighted_async: weight %g of row %lld is "
                       "not a finite value >= 0", (double)weight[r], (long long)r);
    }
    if (c->cfg.model == LCTR_MODEL_FM && c->grad_path != GRAD_DENSE && c->cfg.world == 1 && !c->profiling && rows > 0 && nnz > 0)
        return train_batch_async_graph(c, rows, nnz, row_ptr, fid, val, label, weight, ticket);
    const int p = (int)(c->pipe_issued % kPipe);
    const int slot = kNumSlots - kPipe + p;
    Slot& s = c->slots[slot];
    if (weight && rows > s.cap_rw) {  // room for the weights first (a step may still read the old array)
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        s.cap_rw = 0;
        const int64_t cap = std::max(rows, s.cap_rows);
        if (alloc_group(sized(s.rw, (size_t)cap))) return 1;
        s.cap_rw = cap;
    }
    // the copy may only overwrite the slot once the step that last used it has finished
    if (c->pipe_issued >= (uint64_t)kPipe) LCTR_CUDA(cudaStreamWaitEvent(c->copy_stream, c->ev_computed[p], 0));
    if (c->pipe_issued >= 1) LCTR_CUDA(cudaStreamWaitEvent(c->copy_stream, c->ev_copied[(p + kPipe - 1) % kPipe], 0));  // a graph-path build of the
                                                                   // other slot (build_stream) shares the slot-map scratch
    if (upload_batch_on(c, c->copy_stream, slot, rows, nnz, row_ptr, fid, field, val, label)) return 1;
    if (weight && rows > 0) {
        LCTR_CUDA(cudaMemcpyAsync(s.rw, weight, (size_t)rows * sizeof(float), cudaMemcpyHostToDevice, c->copy_stream));
        s.has_rw = true;
    }
    LCTR_CUDA(cudaEventRecord(c->ev_copied[p], c->copy_stream));
    LCTR_CUDA(cudaStreamWaitEvent(c->stream, c->ev_copied[p], 0));
    const uint64_t step = c->step;
    // the ticket's statistics come from the ring: a weighted slot always writes its weighted ones there
    if (train_step_on(c, slot, 0, rows, true)) return 1;
    LCTR_CUDA(cudaEventRecord(c->ev_computed[p], c->stream));
    const int ri = (int)(step % kStatRing);
    LCTR_CUDA(cudaMemcpyAsync(c->h_stat_ring + 2 * ri, c->stats + 2 * ri, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaEventRecord(c->ev_stat[ri], c->stream));
    c->pipe_graph[p].ticket = ~0ull;
    *ticket = step;
    c->pipe_issued++;
    return 0;
}

int lctr_train_batch_async(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                           const uint16_t* field, const float* val, const int32_t* label, uint64_t* ticket) {
    return train_batch_async(c, rows, nnz, row_ptr, fid, field, val, label, nullptr, ticket);
}

int lctr_train_batch_weighted_async(lctr_ctx* c, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                                    const uint16_t* field, const float* val, const int32_t* label, const float* weight,
                                    uint64_t* ticket) {
    return train_batch_async(c, rows, nnz, row_ptr, fid, field, val, label, weight, ticket);
}

int lctr_wait(lctr_ctx* c, uint64_t ticket, float* loss_sum, float* acc_cnt) {
    LCTR_CHECK(c && c->copy_stream, "lctr_wait: no streamed batch was issued");
    LCTR_CHECK(ticket < c->step && c->step - ticket <= (uint64_t)kStatRing, "lctr_wait: ticket %llu is not outstanding",
               (unsigned long long)ticket);
    for (int p = 0; p < kPipe; p++) {
        if (c->pipe_graph[p].build && c->pipe_graph[p].ticket == ticket) {
            LCTR_CUDA(cudaEventSynchronize(c->ev_computed[p]));
            if (loss_sum) *loss_sum = (float)c->pipe_graph[p].h_stat[0];
            if (acc_cnt) *acc_cnt = (float)c->pipe_graph[p].h_stat[1];
            if (c->pipe_waited < c->pipe_issued) c->pipe_waited++;
            return 0;
        }
    }
    const int ri = (int)(ticket % kStatRing);
    LCTR_CUDA(cudaEventSynchronize(c->ev_stat[ri]));
    if (loss_sum) *loss_sum = (float)c->h_stat_ring[2 * ri];
    if (acc_cnt) *acc_cnt = (float)c->h_stat_ring[2 * ri + 1];
    if (c->pipe_waited < c->pipe_issued) c->pipe_waited++;
    return 0;
}

// forward_round over the whole slot, or one of the single-GPU predictors only lctr_predict has (the FM quirk predictor, the
// FFM parity predictor).  Every refusal comes before anything is launched and follows from the arguments and the
// configuration, so every rank that passes the same arguments refuses alike.
int lctr_predict(lctr_ctx* c, int slot, int quirk_sumvx_slot, float* pctr) {
    if (check_slot(c, "lctr_predict", slot, 0, 0, false)) return 1;  // (rows [0, 0) lie in every slot)
    Slot& s = c->slots[slot];
    const int model = c->cfg.model;
    LCTR_CHECK(model != LCTR_MODEL_NFM, "lctr_predict: the reference ships no NFM predictor (main.cpp:230-233)");
    LCTR_CHECK(quirk_sumvx_slot < 0 || model == LCTR_MODEL_WND || c->cfg.world == 1,
               "lctr_predict: quirk_sumvx_slot is single-GPU: the quirk predictor reads another slot's sumVX, which a sharded "
               "context does not keep for the rows of this slot (world %d)", c->cfg.world);
    LCTR_CHECK(model != LCTR_MODEL_WND || c->cfg.mlp_precision == LCTR_MLP_FP32, "forward-only dense layers run in the fp32 mode");
    int rc;
    if (model == LCTR_MODEL_FM && quirk_sumvx_slot >= 0) {
        LCTR_CHECK(quirk_sumvx_slot < kNumSlots, "quirk slot out of range");
        rc = launch_predict_quirk(c, s, c->slots[quirk_sumvx_slot]);
    } else if (model == LCTR_MODEL_FFM && c->cfg.deterministic == 1) {
        rc = launch_ffm_predict_inorder(c, s);  // parity mode: the reference's own pair loop order
    } else {
        // FM_Predict::Predict / Distributed_Algo_Abst::Predict (distributed_algo_abst.h:163-174): a forward over the slot
        return forward_round(c, s, slot, 0, s.rows, false, pctr);
    }
    if (rc) return 1;
    return pctr ? lctr_download_pred(c, slot, pctr) : 0;
}

int lctr_download_sumvx(lctr_ctx* c, int slot, float* out) {
    LCTR_CHECK(c && out, "null argument");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    LCTR_CHECK(s.sumvx, "model has no sumVX (FFM keeps it NULL, fm_predict.cpp:20)");
    LCTR_CUDA(cudaMemcpyAsync(out, s.sumvx, (size_t)s.rows * c->cfg.factor_cnt * sizeof(float), cudaMemcpyDeviceToHost,
                              c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}
int lctr_download_pred(lctr_ctx* c, int slot, float* out) {
    LCTR_CHECK(c && out, "null argument");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    LCTR_CUDA(cudaMemcpyAsync(out, s.pred, (size_t)s.rows * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_download_batch(lctr_ctx* c, int slot, int64_t* rows, int64_t* nnz, int64_t* row_ptr, uint32_t* fid, uint16_t* field,
                        float* val, float* label) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "slot %d out of range", slot);
    Slot& s = c->slots[slot];
    const size_t r = (size_t)s.rows, n = (size_t)s.nnz;
    if (rows) *rows = s.rows;
    if (nnz) *nnz = s.nnz;
    if (row_ptr && s.row_ptr) LCTR_CUDA(cudaMemcpyAsync(row_ptr, s.row_ptr, (r + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    if (n && fid) LCTR_CUDA(cudaMemcpyAsync(fid, s.fid, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    if (n && field) {
        if (s.has_field) LCTR_CUDA(cudaMemcpyAsync(field, s.field, n * sizeof(uint16_t), cudaMemcpyDeviceToHost, c->stream));
        else memset(field, 0, n * sizeof(uint16_t));
    }
    if (n && val) {
        if (s.has_val) LCTR_CUDA(cudaMemcpyAsync(val, s.val, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        else std::fill(val, val + n, 1.0f);
    }
    if (r && label) LCTR_CUDA(cudaMemcpyAsync(label, s.label, r * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_dense_grad_buffer(lctr_ctx* c, void** dev_ptr, size_t* n_floats) {
    LCTR_CHECK(c && dev_ptr && n_floats, "null argument");
    *dev_ptr = c->dense_grad;
    *n_floats = c->dense_grad_n;
    return 0;
}

int lctr_profile(lctr_ctx* c, int enable) {
    LCTR_CHECK(c, "null ctx");
    c->profiling = enable ? 1 : 0;
    return 0;
}
int lctr_profile_read(lctr_ctx* c, double* ms, int64_t* counts, int n, int reset) {
    LCTR_CHECK(c && ms && counts, "null argument");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i < c->prof_id.size(); i++) {
        float t = 0.f;
        cudaEventElapsedTime(&t, c->prof_ev[2 * i], c->prof_ev[2 * i + 1]);
        const int id = c->prof_id[i];
        if (id >= 0 && id < kNumProf) { c->prof_ms[id] += t; c->prof_cnt[id]++; }
        cudaEventDestroy(c->prof_ev[2 * i]); cudaEventDestroy(c->prof_ev[2 * i + 1]);
    }
    c->prof_ev.clear(); c->prof_id.clear();
    for (int i = 0; i < n && i < kNumProf; i++) { ms[i] = c->prof_ms[i]; counts[i] = c->prof_cnt[i]; }
    if (reset) for (int i = 0; i < kNumProf; i++) { c->prof_ms[i] = 0; c->prof_cnt[i] = 0; }
    return 0;
}

int64_t lctr_launch_count(const lctr_ctx* c) { return c ? c->launches : 0; }
void* lctr_stream(lctr_ctx* c) { return c ? (void*)c->stream : nullptr; }

}  // extern "C"
