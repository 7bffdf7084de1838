// lightctr_b200/csrc/checkpoint.cu -- binary dump / restore of everything a trainer needs to resume: W, V, the updater
// state (Adagrad accumulators | FTRL z,n | Adam m,v + its call counter), the dense layers with their Adagrad state and
// dropout masks, and the step counter.  SURVEY.md 8f-3: the reference's saveModel (fm_algo_abst.h:109-135, kept as text in
// the host shims) writes W and V only, so its optimizer state dies with the process; this is the device-side
// complement.  Also here: the binary CSR cache of a parsed libffm file (8f-2), so that the sscanf-per-token parse of
// fm_algo_abst.h:70-107 is paid once per file.
//
// Multi-GPU trainers (world > 1) write one shard file per rank ("LCTRCKS1"): the single-GPU header, a CkptShard, then the
// same sections over the shard's Fl local rows (local row l = global row l * world + rank) and the rank's own copy of the
// dense layers.  lctr_load_checkpoint reads a shard back into the same rank of the same world; lctr_load_checkpoint_shards
// loads a whole save into a context of any world, streaming the row sections through reshard_rows_kernel.
#include <stdio.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "keys.cuh"

namespace lctr {

struct CkptHeader {
    char magic[8];  // "LCTRCKP1" (one GPU) or "LCTRCKS1" (one rank's shard, a CkptShard follows)
    int32_t model, optimizer, n_layers, reserved;  // reserved: key_word(cfg) (0 for dense tables)
    uint64_t feature_cnt, field_cnt, factor_cnt, adam_iter, step;
    int32_t in[LCTR_MAX_LAYERS + 1], out[LCTR_MAX_LAYERS + 1];
};
struct CkptShard {
    int32_t world, rank;
    uint64_t rows;        // API rows of the whole table: feature_cnt (keyed: the capacity, the null row stays out)
    uint64_t local_rows;  // Fl: rows of each row section of the file
};
static_assert(sizeof(CkptHeader) == 136 && sizeof(CkptShard) == 24, "checkpoint headers are a file format");

// cfg.key_mode in the low byte, cfg.key_evict in bit 8: dense and untracked keyed files keep the value they always had
static int32_t key_word(const lctr_cfg& cfg) { return cfg.key_mode | (cfg.key_evict ? 0x100 : 0); }

static bool put(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
static bool get(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }

// device array <-> file through a bounded pinned-size staging buffer (tables can be tens of GB)
static int dev_to_file(lctr_ctx* c, FILE* f, const float* dev, size_t n) {
    std::vector<float> buf(std::min<size_t>(n, (size_t)16 << 20));
    for (size_t o = 0; o < n; o += buf.size()) {
        const size_t m = std::min(buf.size(), n - o);
        LCTR_CUDA(cudaMemcpyAsync(buf.data(), dev + o, m * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        LCTR_CHECK(put(f, buf.data(), m * sizeof(float)), "checkpoint: short write");
    }
    return 0;
}
static int file_to_dev(lctr_ctx* c, FILE* f, float* dev, size_t n) {
    std::vector<float> buf(std::min<size_t>(n, (size_t)16 << 20));
    for (size_t o = 0; o < n; o += buf.size()) {
        const size_t m = std::min(buf.size(), n - o);
        LCTR_CHECK(get(f, buf.data(), m * sizeof(float)), "checkpoint: short read");
        LCTR_CUDA(cudaMemcpyAsync(dev + o, buf.data(), m * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
    }
    return 0;
}

static bool same_trainer(const lctr_ctx* c, const CkptHeader& h) {
    bool same = h.model == c->cfg.model && h.optimizer == c->cfg.optimizer && h.n_layers == c->n_layers &&
                h.feature_cnt == c->F && h.field_cnt == c->cfg.field_cnt && h.factor_cnt == c->cfg.factor_cnt &&
                h.reserved == key_word(c->cfg);
    for (int l = 0; l < c->n_layers && same; l++) same = h.in[l] == c->layers[l].in && h.out[l] == c->layers[l].out;
    return same;
}

static size_t layer_floats(const lctr_ctx* c) {  // w, b, acc_w, acc_b, mask of every layer
    size_t n = 0;
    for (int l = 0; l < c->n_layers; l++) n += 2 * (size_t)c->layers[l].out * c->layers[l].in + 3 * (size_t)c->layers[l].out;
    return n;
}

// the tail every successful load shares: the dropout-mask flag, the counters
static int finish_load(lctr_ctx* c, const CkptHeader& h) {
    if (c->n_layers) {  // the masked code path of the tensor-core mode is keyed on "any mask entry == 0": recomputed, not accumulated
        c->mlp_has_mask = 0;
        for (int l = 0; l < c->n_layers; l++) {
            std::vector<float> m(c->layers[l].out);
            LCTR_CUDA(cudaMemcpy(m.data(), c->layers[l].mask, m.size() * sizeof(float), cudaMemcpyDeviceToHost));
            for (float v : m) if (v == 0.f) c->mlp_has_mask = 1;
        }
    }
    c->adam_iter = (size_t)h.adam_iter;
    c->step = h.step;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

// keyed loads give rows new numbers: slots translated before hold row ids of the old numbering (as after lctr_evict_keys)
static void mark_slots_stale(lctr_ctx* c) {
    for (int s = 0; s < kNumSlots; s++)
        if (c->slots[s].key_state != SLOT_KEYS_INVALID) c->slots[s].key_state = SLOT_KEYS_STALE;
}

static int log2_world(int w) { int s = 0; while ((1 << s) < w) s++; return s; }

// One file of a load, opened and checked against the context before anything is written: header, cfg, shard geometry,
// file length, and (keyed) its row -> key map, each key owned by the file's rank.
struct CkptFile {
    std::string path;
    FILE* f = nullptr;
    CkptHeader h;
    CkptShard s;             // a single-GPU file reads as world 1, rank 0
    long rows_at = 0;        // offset of the first row section
    std::vector<uint64_t> keys;
    CkptFile() = default;
    CkptFile(const CkptFile&) = delete;
    CkptFile& operator=(const CkptFile&) = delete;
    ~CkptFile() { if (f) fclose(f); }
    size_t arrays(const lctr_ctx* c) const { return c->s2W ? 3 : 2; }  // (W, V) pairs: parameters, s1, s2
    long layers_at(const lctr_ctx* c) const {
        return rows_at + (long)(arrays(c) * s.local_rows * (1 + c->rowlen) * sizeof(float));
    }
};

static int ckpt_open(lctr_ctx* c, const char* path, CkptFile& cf) {
    cf.path = path;
    cf.f = fopen(path, "rb");
    LCTR_CHECK(cf.f, "open file error! (%s)", path);
    const bool ok = get(cf.f, &cf.h, sizeof(cf.h));
    const bool shard = ok && memcmp(cf.h.magic, "LCTRCKS1", 8) == 0;
    LCTR_CHECK(shard || (ok && memcmp(cf.h.magic, "LCTRCKP1", 8) == 0), "%s is not a lightctr_b200 checkpoint", path);
    LCTR_CHECK(same_trainer(c, cf.h), "checkpoint %s was written by a different trainer (model/optimizer/feature_cnt/field_cnt/"
                                      "factor_cnt/layers/key_mode/key_evict)", path);
    const uint64_t rows = api_rows(c);
    if (shard) {
        LCTR_CHECK(get(cf.f, &cf.s, sizeof(cf.s)), "checkpoint %s: short shard header", path);
        const int W = cf.s.world;
        LCTR_CHECK(W >= 2 && W <= 64 && (W & (W - 1)) == 0 && cf.s.rank >= 0 && cf.s.rank < W && cf.s.rows == rows &&
                       cf.s.local_rows == (c->F + W - 1) / W,
                   "checkpoint %s: inconsistent shard header (rank %d of world %d, %llu rows, %llu local rows)", path, cf.s.rank, W,
                   (unsigned long long)cf.s.rows, (unsigned long long)cf.s.local_rows);
    } else {
        cf.s = CkptShard{1, 0, rows, c->F};
    }
    cf.rows_at = ftell(cf.f);
    long end = cf.layers_at(c) + (long)(layer_floats(c) * sizeof(float));
    if (c->keys) {
        uint64_t n = 0;
        const uint64_t owned = (rows + cf.s.world - 1 - cf.s.rank) / cf.s.world;  // global rows < rows this rank holds
        LCTR_CHECK(fseek(cf.f, end, SEEK_SET) == 0 && get(cf.f, &n, sizeof(n)) && n <= owned,
                   "checkpoint %s: missing or inconsistent key section", path);
        cf.keys.resize(n);
        LCTR_CHECK(get(cf.f, cf.keys.data(), n * sizeof(uint64_t)), "checkpoint %s: short read of the keys", path);
        const int shift = log2_world(cf.s.world);
        for (uint64_t i = 0; i < n; i++)
            LCTR_CHECK(cf.keys[i] != kEmptyKey && (int)owner_of_key(cf.keys[i], shift) == cf.s.rank,
                       "checkpoint %s: key %llu at row %llu is not owned by rank %d of world %d (corrupted or mismatched set)",
                       path, (unsigned long long)cf.keys[i], (unsigned long long)i, cf.s.rank, cf.s.world);
        end += (long)((1 + n) * sizeof(uint64_t)) * (keys_tracked(c) ? 2 : 1);  // + the clock and the stamps
    }
    long len = -1;
    if (fseek(cf.f, 0, SEEK_END) == 0) len = ftell(cf.f);
    LCTR_CHECK(len == end, "checkpoint %s: %ld bytes, its header describes %ld", path, len, end);
    LCTR_CHECK(fseek(cf.f, cf.rows_at, SEEK_SET) == 0, "checkpoint %s: seek failed", path);
    return 0;
}

// where row i of a staged chunk of source rows goes: the keyed map, or the dense rule (global row g = source local row *
// source world + source rank; mine when g % world == rank, at local row g / world)
struct ReshardRule {
    const uint32_t* map;  // keyed: destination row per chunk row, kNoRow = not mine; nullptr: the dense rule
    uint64_t l0, rows;    // first source row of the chunk, API rows of the table
    uint32_t src_world, src_rank, world, rank;
};
__device__ __forceinline__ uint32_t reshard_dest(const ReshardRule& r, size_t i) {
    if (r.map) return r.map[i];
    const uint64_t g = (r.l0 + i) * r.src_world + r.src_rank;
    if (g >= r.rows || g % r.world != r.rank) return kNoRow;
    return (uint32_t)(g / r.world);
}

// one staged chunk of a row section into this shard: a warp per row (16-byte accesses when rowlen % 4 == 0), or for the
// W-like sections of one float per row, a thread per row
template <bool VEC4>
__global__ void __launch_bounds__(256) reshard_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n,
                                                           size_t rowlen, ReshardRule r) {
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < n; i += nwarps) {
        const uint32_t d = reshard_dest(r, i);
        if (d == kNoRow) continue;
        if (VEC4) {
            const float4* s4 = reinterpret_cast<const float4*>(src + i * rowlen);
            float4* d4 = reinterpret_cast<float4*>(dst + (size_t)d * rowlen);
            for (size_t j = lane; j < rowlen / 4; j += 32) d4[j] = s4[j];
        } else {
            for (size_t j = lane; j < rowlen; j += 32) dst[(size_t)d * rowlen + j] = src[i * rowlen + j];
        }
    }
}
__global__ void __launch_bounds__(256) reshard_scalars_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n,
                                                              ReshardRule r) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t d = reshard_dest(r, i);
        if (d != kNoRow) dst[d] = src[i];
    }
}
__global__ void fill_kernel(float* p, size_t n, float v) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

// host + device staging of the resharding load: chunks of `rows` source rows (at most 16 M floats)
struct Stage {
    size_t rows = 0;
    std::vector<float> h;
    float* d = nullptr;
    uint32_t* dmap = nullptr;
    ~Stage() { cudaFree(d); cudaFree(dmap); }
};

// one row section (n source rows of `rowlen` floats) of an open file into dst, chunk by chunk
static int scatter_section(lctr_ctx* c, Stage& st, FILE* f, float* dst, size_t n, size_t rowlen, ReshardRule rule,
                           const uint32_t* map) {
    const size_t grid_cap = (size_t)c->sm_count * 16;
    for (size_t l0 = 0; l0 < n; l0 += st.rows) {
        const size_t m = std::min(st.rows, n - l0);
        LCTR_CHECK(get(f, st.h.data(), m * rowlen * sizeof(float)), "checkpoint: short read");
        LCTR_CUDA(cudaMemcpyAsync(st.d, st.h.data(), m * rowlen * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if (map) LCTR_CUDA(cudaMemcpyAsync(st.dmap, map + l0, m * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        rule.map = map ? st.dmap : nullptr;
        rule.l0 = l0;
        if (rowlen == 1) {
            reshard_scalars_kernel<<<(unsigned)std::max<size_t>(1, std::min((m + 255) / 256, grid_cap)), 256, 0, c->stream>>>(
                st.d, dst, m, rule);
        } else {
            const unsigned grid = (unsigned)std::max<size_t>(1, std::min((m + 7) / 8, grid_cap));
            if (rowlen % 4 == 0) reshard_rows_kernel<true><<<grid, 256, 0, c->stream>>>(st.d, dst, m, rowlen, rule);
            else reshard_rows_kernel<false><<<grid, 256, 0, c->stream>>>(st.d, dst, m, rowlen, rule);
        }
        c->launches++;
        LCTR_CUDA(cudaGetLastError());
        LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the host chunk is refilled next
    }
    return 0;
}

// same world, same rank: the sections land where they were read
static int load_shard_in_place(lctr_ctx* c, CkptFile& cf) {
    FILE* f = cf.f;
    const size_t nv = c->Fl * c->rowlen;
    int rc = file_to_dev(c, f, c->W, c->Fl) || file_to_dev(c, f, c->V, nv) || file_to_dev(c, f, c->s1W, c->Fl) ||
             file_to_dev(c, f, c->s1V, nv);
    if (!rc && c->s2W) rc = file_to_dev(c, f, c->s2W, c->Fl) || file_to_dev(c, f, c->s2V, nv);
    for (int l = 0; l < c->n_layers && !rc; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        rc = file_to_dev(c, f, L.w, nw) || file_to_dev(c, f, L.b, L.out) || file_to_dev(c, f, L.acc_w, nw) ||
             file_to_dev(c, f, L.acc_b, L.out) || file_to_dev(c, f, L.mask, L.out);
        if (!rc) rc = mlp_bf16_refresh(c, l);
    }
    if (!rc && c->keys) {
        rc = keys_restore(c, cf.keys.data(), cf.keys.size());
        mark_slots_stale(c);
    }
    return rc ? 1 : finish_load(c, cf.h);
}

// world > 1, lctr_load_checkpoint: the shard this rank of this world wrote
static int load_shard_same_world(lctr_ctx* c, const char* path) {
    CkptFile cf;
    if (ckpt_open(c, path, cf)) return 1;
    LCTR_CHECK(cf.s.world == c->cfg.world && cf.s.rank == c->cfg.rank,
               "checkpoint %s was written by rank %d of world %d, this context is rank %d of world %d (a save of another "
               "world loads through lctr_load_checkpoint_shards)", path, cf.s.rank, cf.s.world, c->cfg.rank, c->cfg.world);
    LCTR_CHECK(!c->keys || cf.keys.size() <= keys_capacity(c), "checkpoint %s: %zu keyed rows exceed the shard's capacity %zu",
               path, cf.keys.size(), keys_capacity(c));
    return load_shard_in_place(c, cf);
}

}  // namespace lctr

using namespace lctr;

extern "C" {

int lctr_save_checkpoint(lctr_ctx* c, const char* path) {
    LCTR_CHECK(c && path, "null argument");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // world > 1: only this rank's kernels, all on this stream, touch its shard
    const std::string tmp = std::string(path) + ".tmp";  // written beside the target and renamed: no torn checkpoint
    FILE* f = fopen(tmp.c_str(), "wb");
    LCTR_CHECK(f, "open file error! (%s)", tmp.c_str());
    const bool shard = c->cfg.world > 1;
    CkptHeader h;
    memset(&h, 0, sizeof(h));
    memcpy(h.magic, shard ? "LCTRCKS1" : "LCTRCKP1", 8);
    h.model = c->cfg.model; h.optimizer = c->cfg.optimizer; h.n_layers = c->n_layers;
    h.feature_cnt = c->F; h.field_cnt = c->cfg.field_cnt; h.factor_cnt = c->cfg.factor_cnt;
    h.adam_iter = c->adam_iter; h.step = c->step;
    h.reserved = key_word(c->cfg);
    for (int l = 0; l < c->n_layers; l++) { h.in[l] = c->layers[l].in; h.out[l] = c->layers[l].out; }
    int rc = put(f, &h, sizeof(h)) ? 0 : 1;
    if (!rc && shard) {
        const CkptShard s{c->cfg.world, c->cfg.rank, api_rows(c), c->Fl};
        rc = put(f, &s, sizeof(s)) ? 0 : 1;
    }
    const size_t nv = c->Fl * c->rowlen;  // Fl == F on one GPU
    const bool two = c->s2W != nullptr;
    rc = rc || dev_to_file(c, f, c->W, c->Fl) || dev_to_file(c, f, c->V, nv) || dev_to_file(c, f, c->s1W, c->Fl) ||
         dev_to_file(c, f, c->s1V, nv);
    if (!rc && two) rc = dev_to_file(c, f, c->s2W, c->Fl) || dev_to_file(c, f, c->s2V, nv);
    for (int l = 0; l < c->n_layers && !rc; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        rc = dev_to_file(c, f, L.w, nw) || dev_to_file(c, f, L.b, L.out) || dev_to_file(c, f, L.acc_w, nw) ||
             dev_to_file(c, f, L.acc_b, L.out) || dev_to_file(c, f, L.mask, L.out);
    }
    if (!rc && c->keys) {  // keyed tables: row count, then the key of every row (the table is rebuilt from it on load)
        std::vector<uint64_t> keys;
        rc = keys_download(c, keys);
        const uint64_t n = keys.size();
        if (!rc) rc = !(put(f, &n, sizeof(n)) && put(f, keys.data(), n * sizeof(uint64_t)));
        if (!rc && keys_tracked(c)) {  // key_evict = 1: the upload clock, then the stamp of every row
            std::vector<uint64_t> stamps;
            uint64_t clock = 0;
            rc = keys_download_stamps(c, n, stamps, &clock);
            if (!rc) rc = !(put(f, &clock, sizeof(clock)) && put(f, stamps.data(), n * sizeof(uint64_t)));
        }
    }
    if (fclose(f) != 0) rc = 1;
    if (rc) {
        remove(tmp.c_str());
        set_error("lctr_save_checkpoint: short write (%s)", tmp.c_str());
        return 1;
    }
    if (rename(tmp.c_str(), path) != 0) {
        remove(tmp.c_str());
        set_error("lctr_save_checkpoint: cannot rename %s to %s", tmp.c_str(), path);
        return 1;
    }
    return 0;
}

int lctr_load_checkpoint(lctr_ctx* c, const char* path) {
    LCTR_CHECK(c && path, "null argument");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (c->cfg.world > 1) return load_shard_same_world(c, path);
    FILE* f = fopen(path, "rb");
    LCTR_CHECK(f, "open file error! (%s)", path);
    CkptHeader h{};
    if (!get(f, &h, sizeof(h)) || memcmp(h.magic, "LCTRCKP1", 8) != 0) {
        const bool shard = memcmp(h.magic, "LCTRCKS1", 8) == 0;
        fclose(f);
        if (shard) set_error("%s is one rank's shard of a multi-GPU checkpoint: load the whole save with lctr_load_checkpoint_shards", path);
        else set_error("%s is not a lightctr_b200 checkpoint", path);
        return 1;
    }
    if (!same_trainer(c, h)) {
        fclose(f);
        set_error("checkpoint %s was written by a different trainer (model/optimizer/feature_cnt/field_cnt/factor_cnt/layers/key_mode/key_evict)", path);
        return 1;
    }
    const size_t nv = c->F * c->rowlen;
    const bool two = c->s2W != nullptr;
    int rc = file_to_dev(c, f, c->W, c->F) || file_to_dev(c, f, c->V, nv) || file_to_dev(c, f, c->s1W, c->F) ||
             file_to_dev(c, f, c->s1V, nv);
    if (!rc && two) rc = file_to_dev(c, f, c->s2W, c->F) || file_to_dev(c, f, c->s2V, nv);
    for (int l = 0; l < c->n_layers && !rc; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        rc = file_to_dev(c, f, L.w, nw) || file_to_dev(c, f, L.b, L.out) || file_to_dev(c, f, L.acc_w, nw) ||
             file_to_dev(c, f, L.acc_b, L.out) || file_to_dev(c, f, L.mask, L.out);
        if (!rc) rc = mlp_bf16_refresh(c, l);
    }
    if (!rc && c->keys) {
        uint64_t n = 0;
        std::vector<uint64_t> keys;
        if (!get(f, &n, sizeof(n)) || n > c->F - 1) {
            rc = 1;
            set_error("checkpoint %s: missing or inconsistent key section", path);
        } else {
            keys.resize(n);
            if (!get(f, keys.data(), n * sizeof(uint64_t))) { rc = 1; set_error("checkpoint %s: short read of the keys", path); }
            else rc = keys_restore(c, keys.data(), n);
        }
        if (!rc && keys_tracked(c)) {
            uint64_t clock = 0;
            std::vector<uint64_t> stamps(n);
            if (!get(f, &clock, sizeof(clock)) || !get(f, stamps.data(), n * sizeof(uint64_t))) {
                rc = 1;
                set_error("checkpoint %s: short read of the row stamps", path);
            } else {
                rc = keys_restore_stamps(c, stamps.data(), n, clock);
            }
        }
    }
    fclose(f);
    if (rc) return 1;
    return finish_load(c, h);
}

int lctr_load_checkpoint_shards(lctr_ctx* c, int n, const char* const* paths) {
    LCTR_CHECK(c && n >= 1 && paths, "lctr_load_checkpoint_shards: null argument or empty set");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const int world = c->cfg.world, me = c->cfg.rank;
    // 1. every check, before any device write
    std::vector<std::unique_ptr<CkptFile>> fs(n);
    for (int i = 0; i < n; i++) {
        LCTR_CHECK(paths[i], "lctr_load_checkpoint_shards: null path %d", i);
        fs[i].reset(new CkptFile());
        if (ckpt_open(c, paths[i], *fs[i])) return 1;
    }
    std::vector<CkptFile*> by_rank(n, nullptr);  // the files in rank order: the source order of keyed rows
    for (int i = 0; i < n; i++) {
        CkptFile& cf = *fs[i];
        LCTR_CHECK(cf.s.world == n, "lctr_load_checkpoint_shards: %s belongs to a save of world %d, the set has %d files", cf.path.c_str(),
                   cf.s.world, n);
        LCTR_CHECK(!by_rank[cf.s.rank], "lctr_load_checkpoint_shards: rank %d appears twice (%s, %s)", cf.s.rank,
                   by_rank[cf.s.rank]->path.c_str(), cf.path.c_str());
        by_rank[cf.s.rank] = &cf;
    }
    const CkptHeader& h0 = by_rank[0]->h;
    for (int r = 1; r < n; r++)
        LCTR_CHECK(by_rank[r]->h.step == h0.step && by_rank[r]->h.adam_iter == h0.adam_iter,
                   "lctr_load_checkpoint_shards: rank %d was saved at step %llu (adam_iter %llu), rank 0 at step %llu (adam_iter "
                   "%llu): not one save", r, (unsigned long long)by_rank[r]->h.step, (unsigned long long)by_rank[r]->h.adam_iter,
                   (unsigned long long)h0.step, (unsigned long long)h0.adam_iter);
    if (n == world) {  // the world is unchanged: this rank's own file, rows in place, its own layers
        CkptFile& mine = *by_rank[me];
        if (world == 1) {
            const std::string path = mine.path;
            fs.clear();
            if (lctr_load_checkpoint(c, path.c_str())) return 1;  // the single-GPU loader (stamps included)
            if (c->keys) mark_slots_stale(c);
            return 0;
        }
        LCTR_CHECK(!c->keys || mine.keys.size() <= keys_capacity(c), "checkpoint %s: %zu keyed rows exceed the shard's capacity %zu",
                   mine.path.c_str(), mine.keys.size(), keys_capacity(c));
        return load_shard_in_place(c, mine);
    }
    // the world changes: the dense layers must be one model
    const size_t nlf = layer_floats(c);
    std::vector<float> layers(nlf), other(nlf);
    for (int r = 0; r < n && nlf; r++) {
        CkptFile& cf = *by_rank[r];
        LCTR_CHECK(fseek(cf.f, cf.layers_at(c), SEEK_SET) == 0 && get(cf.f, r ? other.data() : layers.data(), nlf * sizeof(float)),
                   "checkpoint %s: short read of the dense layers", cf.path.c_str());
        LCTR_CHECK(r == 0 || memcmp(layers.data(), other.data(), nlf * sizeof(float)) == 0,
                   "lctr_load_checkpoint_shards: the dense layers of rank %d differ from rank 0's (per-rank layers, as Wide&Deep "
                   "trains them without a dense all-reduce: no rule picks one of them for world %d)", r, world);
    }
    // keyed: the keys this rank owns under its world, at rows 0..m-1 in source order
    std::vector<std::vector<uint32_t>> maps(c->keys ? n : 0);
    std::vector<uint64_t> mine;
    if (c->keys) {
        const int shift = log2_world(world);
        for (int r = 0; r < n; r++) {
            const CkptFile& cf = *by_rank[r];
            maps[r].assign(cf.s.local_rows, kNoRow);
            for (size_t l = 0; l < cf.keys.size(); l++)
                if ((int)owner_of_key(cf.keys[l], shift) == me) {
                    maps[r][l] = (uint32_t)mine.size();
                    mine.push_back(cf.keys[l]);
                }
        }
        LCTR_CHECK(mine.size() <= keys_capacity(c),
                   "lctr_load_checkpoint_shards: rank %d would hold %zu keys, its shard's capacity is %zu rows (nothing was changed)",
                   me, mine.size(), keys_capacity(c));
    }
    // 2. the writes: keyed shards start from the state lctr_create gives (rows past the keys stay so)
    const size_t nv = c->Fl * c->rowlen;
    if (c->keys) {
        const float s1 = (c->cfg.optimizer == LCTR_OPT_PS_ADAGRAD || c->cfg.optimizer == LCTR_OPT_PS_DCASGDA) ? 1e-7f : 0.f;
        const unsigned grid = (unsigned)c->sm_count * 4;
        LCTR_CUDA(cudaMemsetAsync(c->W, 0, c->Fl * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(c->V, 0, nv * sizeof(float), c->stream));
        fill_kernel<<<grid, 256, 0, c->stream>>>(c->s1W, c->Fl, s1);
        fill_kernel<<<grid, 256, 0, c->stream>>>(c->s1V, nv, s1);
        c->launches += 2;
        LCTR_CUDA(cudaGetLastError());
        if (c->s2W) {
            LCTR_CUDA(cudaMemsetAsync(c->s2W, 0, c->Fl * sizeof(float), c->stream));
            LCTR_CUDA(cudaMemsetAsync(c->s2V, 0, nv * sizeof(float), c->stream));
        }
    }
    Stage st;
    {
        size_t src_rows = 0;
        for (int r = 0; r < n; r++) src_rows = std::max<size_t>(src_rows, by_rank[r]->s.local_rows);
        st.rows = std::max<size_t>(1, std::min<size_t>(src_rows, ((size_t)16 << 20) / c->rowlen));
        st.h.resize(st.rows * c->rowlen);
        LCTR_CUDA(cudaMalloc((void**)&st.d, st.rows * c->rowlen * sizeof(float)));
        if (c->keys) LCTR_CUDA(cudaMalloc((void**)&st.dmap, st.rows * sizeof(uint32_t)));
    }
    float* dst[6] = {c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V};
    for (int r = 0; r < n; r++) {
        CkptFile& cf = *by_rank[r];
        LCTR_CHECK(fseek(cf.f, cf.rows_at, SEEK_SET) == 0, "checkpoint %s: seek failed", cf.path.c_str());
        const ReshardRule rule{nullptr, 0, api_rows(c), (uint32_t)n, (uint32_t)r, (uint32_t)world, (uint32_t)me};
        const uint32_t* map = c->keys ? maps[r].data() : nullptr;
        for (size_t a = 0; a < 2 * cf.arrays(c); a++)
            if (scatter_section(c, st, cf.f, dst[a], cf.s.local_rows, a % 2 ? c->rowlen : 1, rule, map)) return 1;
    }
    const float* src = layers.data();
    for (int l = 0; l < c->n_layers; l++) {
        MlpLayer& L = c->layers[l];
        const size_t nw = (size_t)L.out * L.in;
        float* parts[5] = {L.w, L.b, L.acc_w, L.acc_b, L.mask};
        const size_t sizes[5] = {nw, (size_t)L.out, nw, (size_t)L.out, (size_t)L.out};
        for (int p = 0; p < 5; p++) {
            LCTR_CUDA(cudaMemcpyAsync(parts[p], src, sizes[p] * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            src += sizes[p];
        }
        if (mlp_bf16_refresh(c, l)) return 1;
    }
    if (c->keys) {
        if (keys_restore(c, mine.data(), mine.size())) return 1;
        mark_slots_stale(c);
    }
    return finish_load(c, h0);
}

// ---- binary CSR cache of a parsed dataset -------------------------------------------------------------------------
int lctr_save_dataset_bin(const lctr_dataset* d, const char* path) {
    if (!d || !path) { set_error("lctr_save_dataset_bin: null argument"); return 1; }
    FILE* f = fopen(path, "wb");
    if (!f) { set_error("open file error! (%s)", path); return 1; }
    const char magic[8] = {'L', 'C', 'T', 'R', 'C', 'S', 'R', '1'};
    const uint64_t hdr[5] = {(uint64_t)d->rows, (uint64_t)d->nnz, (uint64_t)d->label_cnt, d->feature_cnt, d->field_cnt};
    bool ok = put(f, magic, 8) && put(f, hdr, sizeof(hdr)) && put(f, d->row_ptr, sizeof(int64_t) * (size_t)(d->rows + 1)) &&
              put(f, d->fid, sizeof(uint32_t) * (size_t)d->nnz) && put(f, d->field, sizeof(uint16_t) * (size_t)d->nnz) &&
              put(f, d->val, sizeof(float) * (size_t)d->nnz) && put(f, d->label, sizeof(int32_t) * (size_t)d->label_cnt);
    fclose(f);
    if (!ok) { set_error("lctr_save_dataset_bin: short write (%s)", path); return 1; }
    return 0;
}

int lctr_load_dataset_bin(const char* path, lctr_dataset** out) {
    if (!path || !out) { set_error("lctr_load_dataset_bin: null argument"); return 1; }
    FILE* f = fopen(path, "rb");
    if (!f) { set_error("open file error! (%s)", path); return 1; }
    char magic[8];
    uint64_t hdr[5];
    if (!get(f, magic, 8) || memcmp(magic, "LCTRCSR1", 8) != 0 || !get(f, hdr, sizeof(hdr))) {
        fclose(f);
        set_error("%s is not a lightctr_b200 CSR cache", path);
        return 1;
    }
    // the header is not trusted: the counts must be consistent with each other and with the length of the file
    long long flen = -1;
    {
        const long here = ftell(f);
        if (here >= 0 && fseek(f, 0, SEEK_END) == 0) { flen = ftell(f); fseek(f, here, SEEK_SET); }
    }
    const uint64_t rows = hdr[0], nnz = hdr[1], labels = hdr[2];
    const uint64_t kMax = (uint64_t)1 << 40;
    const bool sane = rows < kMax && nnz < kMax && labels < kMax && labels >= rows &&
                      (flen < 0 || (unsigned long long)flen == 8 + sizeof(hdr) + 8 * (rows + 1) + 10 * nnz + 4 * labels);
    if (!sane) {
        fclose(f);
        set_error("%s: inconsistent CSR cache header (rows %llu, nnz %llu, labels %llu, file %lld bytes)", path,
                  (unsigned long long)rows, (unsigned long long)nnz, (unsigned long long)labels, flen);
        return 1;
    }
    lctr_dataset* d = (lctr_dataset*)calloc(1, sizeof(lctr_dataset));
    if (!d) { fclose(f); set_error("lctr_load_dataset_bin: out of memory"); return 1; }
    d->rows = (int64_t)rows; d->nnz = (int64_t)nnz; d->label_cnt = (int64_t)labels;
    d->feature_cnt = hdr[3]; d->field_cnt = hdr[4];
    const size_t nn = d->nnz ? (size_t)d->nnz : 1, nl = d->label_cnt ? (size_t)d->label_cnt : 1;
    d->row_ptr = (int64_t*)malloc(sizeof(int64_t) * (size_t)(d->rows + 1));
    d->fid = (uint32_t*)malloc(sizeof(uint32_t) * nn);
    d->field = (uint16_t*)malloc(sizeof(uint16_t) * nn);
    d->val = (float*)malloc(sizeof(float) * nn);
    d->label = (int32_t*)malloc(sizeof(int32_t) * nl);
    if (!d->row_ptr || !d->fid || !d->field || !d->val || !d->label) {
        fclose(f); lctr_free_dataset(d);
        set_error("lctr_load_dataset_bin: out of memory for %llu entries", (unsigned long long)nnz);
        return 1;
    }
    bool ok = get(f, d->row_ptr, sizeof(int64_t) * (size_t)(d->rows + 1)) && get(f, d->fid, sizeof(uint32_t) * (size_t)d->nnz) &&
              get(f, d->field, sizeof(uint16_t) * (size_t)d->nnz) && get(f, d->val, sizeof(float) * (size_t)d->nnz) &&
              get(f, d->label, sizeof(int32_t) * (size_t)d->label_cnt);
    fclose(f);
    if (!ok) { lctr_free_dataset(d); set_error("lctr_load_dataset_bin: short read (%s)", path); return 1; }
    *out = d;
    return 0;
}

}  // extern "C"
