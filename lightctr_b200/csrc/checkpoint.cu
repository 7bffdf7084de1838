// lightctr_b200/csrc/checkpoint.cu -- binary dump / restore of everything a trainer needs to resume: W, V, the updater
// state (Adagrad accumulators | FTRL z,n | Adam m,v + its call counter), the dense layers with their Adagrad state and
// dropout masks, and the step counter.  SURVEY.md 8f-3: the reference's saveModel (fm_algo_abst.h:109-135, kept as text in
// the host shims) writes W and V only, so its optimizer state dies with the process; this is the device-side
// complement.  Also here: the binary CSR cache of a parsed libffm file (8f-2), so that the sscanf-per-token parse of
// fm_algo_abst.h:70-107 is paid once per file.
//
// Multi-GPU trainers (world > 1) write one shard file per rank ("LCTRCKS1"): the single-GPU header, a CkptShard, then the
// same sections over the shard's Fl local rows (local row l = global row l * world + rank) and the rank's own copy of the
// dense layers.  Every load reads through ckpt_open, which checks a file against the context before anything is written
// (a single-GPU file reads as rank 0 of world 1).  lctr_load_checkpoint then loads the file of this rank of this world in
// place, for every world; lctr_load_checkpoint_shards loads a whole save into a context of any world, streaming the row
// sections through reshard_rows_kernel when the world changes.
#include <stdio.h>
#include <string.h>

#include <algorithm>
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

// cfg.key_mode in the low byte, cfg.key_evict in bit 8, a host tier (cfg.key_host_rows > 0) in bit 9: dense, untracked and
// untiered keyed files keep the value they always had
static int32_t key_word(const lctr_cfg& cfg) {
    return cfg.key_mode | (cfg.key_evict ? 0x100 : 0) | (cfg.key_host_rows ? 0x200 : 0);
}
// bit 10: key admission was on (lctr_set_key_admission), and the file ends with its section.  Not part of the cfg, so it
// is compared apart from the other bits
constexpr int32_t kAdmissionBit = 0x400;

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
                (h.reserved & ~kAdmissionBit) == key_word(c->cfg);
    for (int l = 0; l < c->n_layers && same; l++) same = h.in[l] == c->layers[l].in && h.out[l] == c->layers[l].out;
    return same;
}

// The sections of a file after its header(s), in file order: the row sections over the file's rows, the parts of every
// layer, then for keyed tables the row count and the key of every row, for key_evict = 1 the upload clock and the stamp
// of every row, and for a host tier its row count n, the key and the stamp of each of its rows, then the row sections over
// those n rows, and with key admission (header bit 10) u32 min_count, u32 log2_width and the 4 * 2^log2_width u32
// counters of the sketch.  Everything that walks the format takes the row sections and the layer parts from these helpers.

// W, V, s1W, s1V[, s2W, s2V] of this rank's shard
struct RowSections {
    float* p[6];
    int n;  // 4, or 6 when the updater keeps s2
    size_t rowlen;
    size_t width(int a) const { return a % 2 ? rowlen : 1; }  // floats per row of section a
};
static RowSections row_sections(const lctr_ctx* c) {
    return {{c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V}, c->s2W ? 6 : 4, c->rowlen};
}
// the same sections over the host tier's arrays (pinned host memory)
static RowSections tier_sections(const lctr_ctx* c, const TierRows& tr) {
    RowSections rs = row_sections(c);
    for (int a = 0; a < 6; a++) rs.p[a] = tr.p[a];
    return rs;
}

// w, b, acc_w, acc_b, mask of one dense layer and their sizes in floats
struct LayerParts {
    float* p[5];
    size_t n[5];
};
static LayerParts layer_parts(const MlpLayer& L) {
    const size_t nw = (size_t)L.out * L.in, no = (size_t)L.out;
    return {{L.w, L.b, L.acc_w, L.acc_b, L.mask}, {nw, no, nw, no, no}};
}

static size_t row_floats(const lctr_ctx* c) {  // one row across the row sections
    const RowSections rs = row_sections(c);
    size_t n = 0;
    for (int a = 0; a < rs.n; a++) n += rs.width(a);
    return n;
}
static size_t layer_floats(const lctr_ctx* c) {  // every layer
    size_t n = 0;
    for (int l = 0; l < c->n_layers; l++)
        for (size_t m : layer_parts(c->layers[l]).n) n += m;
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
// file length, (keyed) its row -> key map, each key owned by the file's rank, and (key_evict = 1) the clock and stamps.
struct CkptFile {
    std::string path;
    FILE* f = nullptr;
    CkptHeader h;
    CkptShard s;             // a single-GPU file reads as world 1, rank 0
    long rows_at = 0;        // offset of the first row section
    std::vector<uint64_t> keys;
    uint64_t clock = 0;
    std::vector<uint64_t> stamps;
    std::vector<uint64_t> tier_keys, tier_stamps;  // host tier (cfg.key_host_rows > 0)
    long tier_rows_at = 0;                         // offset of its row sections
    bool adm = false;                              // key admission section (header bit 10)
    uint32_t adm_min = 0, adm_lw = 0;
    long adm_at = 0;                               // offset of its counters
    CkptFile() = default;
    CkptFile(const CkptFile&) = delete;
    CkptFile& operator=(const CkptFile&) = delete;
    ~CkptFile() { if (f) fclose(f); }
    long layers_at(const lctr_ctx* c) const { return rows_at + (long)(s.local_rows * row_floats(c) * sizeof(float)); }
};

static int ckpt_open(lctr_ctx* c, const char* path, CkptFile& cf) {
    cf.path = path;
    cf.f = fopen(path, "rb");
    LCTR_CHECK(cf.f, "open file error! (%s)", path);
    const bool ok = get(cf.f, &cf.h, sizeof(cf.h));
    const bool shard = ok && memcmp(cf.h.magic, "LCTRCKS1", 8) == 0;
    LCTR_CHECK(shard || (ok && memcmp(cf.h.magic, "LCTRCKP1", 8) == 0), "%s is not a lightctr_b200 checkpoint", path);
    LCTR_CHECK(same_trainer(c, cf.h), "checkpoint %s was written by a different trainer (model/optimizer/feature_cnt/field_cnt/"
                                      "factor_cnt/layers/key_mode/key_evict/key_host_rows)", path);
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
        LCTR_CHECK(fseek(cf.f, end, SEEK_SET) == 0 && get(cf.f, &n, sizeof(n)) && n <= owned_rows(rows, cf.s.world, cf.s.rank),
                   "checkpoint %s: missing or inconsistent key section", path);
        cf.keys.resize(n);
        LCTR_CHECK(get(cf.f, cf.keys.data(), n * sizeof(uint64_t)), "checkpoint %s: short read of the keys", path);
        const int shift = log2_world(cf.s.world);
        for (uint64_t i = 0; i < n; i++)
            LCTR_CHECK(cf.keys[i] != kEmptyKey && (int)owner_of_key(cf.keys[i], shift) == cf.s.rank,
                       "checkpoint %s: key %llu at row %llu is not owned by rank %d of world %d (corrupted or mismatched set)",
                       path, (unsigned long long)cf.keys[i], (unsigned long long)i, cf.s.rank, cf.s.world);
        end += (long)((1 + n) * sizeof(uint64_t));
        if (keys_tracked(c)) {
            cf.stamps.resize(n);
            LCTR_CHECK(get(cf.f, &cf.clock, sizeof(cf.clock)) && get(cf.f, cf.stamps.data(), n * sizeof(uint64_t)),
                       "checkpoint %s: short read of the row stamps", path);
            end += (long)((1 + n) * sizeof(uint64_t));
        }
        TierRows tr;
        if (keys_tier(c, &tr)) {
            uint64_t nt = 0;
            LCTR_CHECK(get(cf.f, &nt, sizeof(nt)) && nt <= tr.cap,
                       "checkpoint %s: missing host-tier section, or more rows than cfg.key_host_rows = %zu", path, tr.cap);
            cf.tier_keys.resize(nt);
            cf.tier_stamps.resize(nt);
            LCTR_CHECK(get(cf.f, cf.tier_keys.data(), nt * sizeof(uint64_t)) && get(cf.f, cf.tier_stamps.data(), nt * sizeof(uint64_t)),
                       "checkpoint %s: short read of the host tier's keys", path);
            // a key lives in at most one of the two tables
            std::vector<uint64_t> all(cf.keys);
            all.insert(all.end(), cf.tier_keys.begin(), cf.tier_keys.end());
            std::sort(all.begin(), all.end());
            LCTR_CHECK(std::adjacent_find(all.begin(), all.end()) == all.end() && (all.empty() || all.back() != kEmptyKey),
                       "checkpoint %s: a host-tier key is reserved or held twice", path);
            cf.tier_rows_at = end + (long)((1 + 2 * nt) * sizeof(uint64_t));
            end = cf.tier_rows_at + (long)(nt * row_floats(c) * sizeof(float));
        }
        if (cf.h.reserved & kAdmissionBit) {
            uint32_t s[2] = {0, 0};
            LCTR_CHECK(fseek(cf.f, end, SEEK_SET) == 0 && get(cf.f, s, sizeof(s)) && s[0] > 1 && s[1] >= 10 && s[1] <= 28,
                       "checkpoint %s: missing or inconsistent key admission section", path);
            cf.adm = true;
            cf.adm_min = s[0];
            cf.adm_lw = s[1];
            cf.adm_at = end + (long)sizeof(s);
            end = cf.adm_at + (long)(((size_t)4 << s[1]) * sizeof(uint32_t));
        }
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

// host + device staging of the resharding load: chunks of `rows` source rows (at most 16 M floats)
struct Stage {
    size_t rows = 0;
    std::vector<float> h;
    Buf<float> d;
    Buf<uint32_t> dmap;
};

// one row section (n source rows of `rowlen` floats) of an open file into dst, chunk by chunk
static int scatter_section(lctr_ctx* c, Stage& st, FILE* f, float* dst, size_t n, size_t rowlen, ReshardRule rule,
                           const uint32_t* map) {
    const size_t grid_cap = (size_t)c->sm_count * 16;
    for (size_t l0 = 0; l0 < n; l0 += st.rows) {
        const size_t m = std::min(st.rows, n - l0);
        LCTR_CHECK(get(f, st.h.data(), m * rowlen * sizeof(float)), "checkpoint: short read");
        auto chunk = [&]() -> int {
            LCTR_CUDA(cudaMemcpyAsync(st.d, st.h.data(), m * rowlen * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            if (map) LCTR_CUDA(cudaMemcpyAsync(st.dmap, map + l0, m * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
            rule.map = map ? st.dmap.get() : nullptr;
            rule.l0 = l0;
            return rowlen == 1
                ? launch(c, {(unsigned)std::max<size_t>(1, std::min((m + 255) / 256, grid_cap)), 256, 0, c->stream},
                         reshard_scalars_kernel, st.d, dst, m, rule)
                : launch(c, {(unsigned)std::max<size_t>(1, std::min((m + 7) / 8, grid_cap)), 256, 0, c->stream},
                         rowlen % 4 == 0 ? reshard_rows_kernel<true> : reshard_rows_kernel<false>, st.d, dst, m, rowlen, rule);
        };
        const int rc = chunk();
        // the host chunk is refilled next; after a failure the stage goes with the caller, while queued copies may read it
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        if (rc) return 1;
    }
    return 0;
}

// the key admission settings of a file against the context's: they must be equal (off = off), except that a context with
// admission off may be told to ignore the file's section (skip_when_off)
static int check_admission(const lctr_ctx* c, const CkptFile& cf, bool skip_when_off) {
    uint32_t mc = 0, lw = 0;
    const bool on = keys_admission(c, &mc, &lw);
    if (!on && skip_when_off) return 0;
    if (on == cf.adm && mc == cf.adm_min && lw == cf.adm_lw) return 0;
    char mine[64] = "off", theirs[64] = "off";
    if (on) snprintf(mine, sizeof(mine), "min_count %u, log2_width %u", mc, lw);
    if (cf.adm) snprintf(theirs, sizeof(theirs), "min_count %u, log2_width %u", cf.adm_min, cf.adm_lw);
    set_error("checkpoint %s was saved with key admission %s, this context has %s (lctr_set_key_admission must match; nothing "
              "was changed)", cf.path.c_str(), theirs, mine);
    return 1;
}

// a file ckpt_open checked, written by this rank of this world: the sections land where they were read
static int load_shard_in_place(lctr_ctx* c, CkptFile& cf) {
    LCTR_CHECK(!c->keys || cf.keys.size() <= keys_capacity(c), "checkpoint %s: %zu keyed rows exceed the shard's capacity %zu",
               cf.path.c_str(), cf.keys.size(), keys_capacity(c));
    const RowSections rs = row_sections(c);
    for (int a = 0; a < rs.n; a++)
        if (file_to_dev(c, cf.f, rs.p[a], c->Fl * rs.width(a))) return 1;
    for (int l = 0; l < c->n_layers; l++) {
        const LayerParts lp = layer_parts(c->layers[l]);
        for (int p = 0; p < 5; p++)
            if (file_to_dev(c, cf.f, lp.p[p], lp.n[p])) return 1;
        if (mlp_bf16_refresh(c, l)) return 1;
    }
    if (c->keys) {
        mark_slots_stale(c);
        if (keys_restore(c, cf.keys.data(), cf.keys.size())) return 1;
        if (keys_tracked(c) && keys_restore_stamps(c, cf.stamps.data(), cf.stamps.size(), cf.clock)) return 1;
        TierRows tr;
        if (keys_tier(c, &tr)) {  // straight into the pinned arrays, then a fresh index
            const size_t nt = cf.tier_keys.size();
            memcpy(tr.key, cf.tier_keys.data(), nt * sizeof(uint64_t));
            memcpy(tr.stamp, cf.tier_stamps.data(), nt * sizeof(uint64_t));
            const RowSections ts = tier_sections(c, tr);
            LCTR_CHECK(fseek(cf.f, cf.tier_rows_at, SEEK_SET) == 0, "checkpoint %s: seek failed", cf.path.c_str());
            for (int a = 0; a < ts.n; a++)
                LCTR_CHECK(get(cf.f, ts.p[a], nt * ts.width(a) * sizeof(float)), "checkpoint %s: short read of the host tier", cf.path.c_str());
            if (keys_tier_restore(c, nt)) return 1;
        }
        uint32_t mc, lw;
        if (cf.adm && keys_admission(c, &mc, &lw)) {  // check_admission made the settings equal
            std::vector<uint32_t> sketch((size_t)4 << lw);
            LCTR_CHECK(fseek(cf.f, cf.adm_at, SEEK_SET) == 0 && get(cf.f, sketch.data(), sketch.size() * sizeof(uint32_t)),
                       "checkpoint %s: short read of the key admission sketch", cf.path.c_str());
            if (keys_admission_restore(c, sketch.data())) return 1;
        }
    }
    return finish_load(c, cf.h);
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
    uint32_t adm[2];
    const bool admission = keys_admission(c, &adm[0], &adm[1]);
    h.reserved = key_word(c->cfg) | (admission ? kAdmissionBit : 0);
    for (int l = 0; l < c->n_layers; l++) { h.in[l] = c->layers[l].in; h.out[l] = c->layers[l].out; }
    int rc = put(f, &h, sizeof(h)) ? 0 : 1;
    if (!rc && shard) {
        const CkptShard s{c->cfg.world, c->cfg.rank, api_rows(c), c->Fl};
        rc = put(f, &s, sizeof(s)) ? 0 : 1;
    }
    const RowSections rs = row_sections(c);
    for (int a = 0; a < rs.n && !rc; a++) rc = dev_to_file(c, f, rs.p[a], c->Fl * rs.width(a));  // Fl == F on one GPU
    for (int l = 0; l < c->n_layers && !rc; l++) {
        const LayerParts lp = layer_parts(c->layers[l]);
        for (int p = 0; p < 5 && !rc; p++) rc = dev_to_file(c, f, lp.p[p], lp.n[p]);
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
        TierRows tr;
        if (!rc && keys_tier(c, &tr)) {  // host tier: row count, keys, stamps, then its row sections
            const uint64_t nt = tr.n;
            const RowSections ts = tier_sections(c, tr);
            rc = !(put(f, &nt, sizeof(nt)) && put(f, tr.key, nt * sizeof(uint64_t)) && put(f, tr.stamp, nt * sizeof(uint64_t)));
            for (int a = 0; a < ts.n && !rc; a++) rc = !put(f, ts.p[a], nt * ts.width(a) * sizeof(float));
        }
        if (!rc && admission) {  // key admission: min_count, log2_width, the sketch
            std::vector<uint32_t> sketch;
            rc = keys_admission_download(c, sketch);
            if (!rc) rc = !(put(f, adm, sizeof(adm)) && put(f, sketch.data(), sketch.size() * sizeof(uint32_t)));
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
    CkptFile cf;
    if (ckpt_open(c, path, cf)) return 1;
    LCTR_CHECK(cf.s.world == c->cfg.world && cf.s.rank == c->cfg.rank,
               "checkpoint %s was written by rank %d of world %d, this context is rank %d of world %d (a save of another "
               "world loads through lctr_load_checkpoint_shards)", path, cf.s.rank, cf.s.world, c->cfg.rank, c->cfg.world);
    if (check_admission(c, cf, false)) return 1;
    return load_shard_in_place(c, cf);
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
        if (check_admission(c, *fs[i], true)) return 1;  // a context with admission off skips the section
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
    if (n == world) return load_shard_in_place(c, *by_rank[me]);  // the world is unchanged: this rank's own file in place
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
    if (c->keys && reset_table_rows(c)) return 1;
    Stage st;
    {
        size_t src_rows = 0;
        for (int r = 0; r < n; r++) src_rows = std::max<size_t>(src_rows, by_rank[r]->s.local_rows);
        st.rows = std::max<size_t>(1, std::min<size_t>(src_rows, ((size_t)16 << 20) / c->rowlen));
        st.h.resize(st.rows * c->rowlen);
        if (st.d.alloc(st.rows * c->rowlen) || (c->keys && st.dmap.alloc(st.rows))) return 1;
    }
    const RowSections rs = row_sections(c);
    for (int r = 0; r < n; r++) {
        CkptFile& cf = *by_rank[r];
        LCTR_CHECK(fseek(cf.f, cf.rows_at, SEEK_SET) == 0, "checkpoint %s: seek failed", cf.path.c_str());
        const ReshardRule rule{nullptr, 0, api_rows(c), (uint32_t)n, (uint32_t)r, (uint32_t)world, (uint32_t)me};
        const uint32_t* map = c->keys ? maps[r].data() : nullptr;
        for (int a = 0; a < rs.n; a++)
            if (scatter_section(c, st, cf.f, rs.p[a], cf.s.local_rows, rs.width(a), rule, map)) return 1;
    }
    const float* src = layers.data();
    for (int l = 0; l < c->n_layers; l++) {
        const LayerParts lp = layer_parts(c->layers[l]);
        for (int p = 0; p < 5; p++) {
            LCTR_CUDA(cudaMemcpyAsync(lp.p[p], src, lp.n[p] * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            src += lp.n[p];
        }
        if (mlp_bf16_refresh(c, l)) return 1;
    }
    if (c->keys) {
        mark_slots_stale(c);
        if (keys_restore(c, mine.data(), mine.size())) return 1;
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
