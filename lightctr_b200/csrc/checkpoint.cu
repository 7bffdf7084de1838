// lightctr_b200/csrc/checkpoint.cu -- binary dump / restore of everything a trainer needs to resume: W, V, the updater
// state (Adagrad accumulators | FTRL z,n | Adam m,v + its call counter), the dense layers with their Adagrad state and
// dropout masks, and the step counter.  SURVEY.md 8f-3: the reference's saveModel (fm_algo_abst.h:109-135, kept as text in
// the host shims) writes W and V only, so its optimizer state dies with the process; this is the device-side
// complement.  Also here: the binary CSR cache of a parsed libffm file (8f-2), so that the sscanf-per-token parse of
// fm_algo_abst.h:70-107 is paid once per file.
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace lctr {

struct CkptHeader {
    char magic[8];  // "LCTRCKP1"
    int32_t model, optimizer, n_layers, reserved;  // reserved: key_word(cfg) (0 for dense tables)
    uint64_t feature_cnt, field_cnt, factor_cnt, adam_iter, step;
    int32_t in[LCTR_MAX_LAYERS + 1], out[LCTR_MAX_LAYERS + 1];
};

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

}  // namespace lctr

using namespace lctr;

extern "C" {

int lctr_save_checkpoint(lctr_ctx* c, const char* path) {
    LCTR_CHECK(c && path, "null argument");
    LCTR_CHECK(c->cfg.world == 1, "checkpoints are written per single-GPU trainer (world == 1)");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const std::string tmp = std::string(path) + ".tmp";  // written beside the target and renamed: no torn checkpoint
    FILE* f = fopen(tmp.c_str(), "wb");
    LCTR_CHECK(f, "open file error! (%s)", tmp.c_str());
    CkptHeader h;
    memset(&h, 0, sizeof(h));
    memcpy(h.magic, "LCTRCKP1", 8);
    h.model = c->cfg.model; h.optimizer = c->cfg.optimizer; h.n_layers = c->n_layers;
    h.feature_cnt = c->F; h.field_cnt = c->cfg.field_cnt; h.factor_cnt = c->cfg.factor_cnt;
    h.adam_iter = c->adam_iter; h.step = c->step;
    h.reserved = key_word(c->cfg);
    for (int l = 0; l < c->n_layers; l++) { h.in[l] = c->layers[l].in; h.out[l] = c->layers[l].out; }
    int rc = put(f, &h, sizeof(h)) ? 0 : 1;
    const size_t nv = c->F * c->rowlen;
    const bool two = c->s2W != nullptr;
    rc = rc || dev_to_file(c, f, c->W, c->F) || dev_to_file(c, f, c->V, nv) || dev_to_file(c, f, c->s1W, c->F) ||
         dev_to_file(c, f, c->s1V, nv);
    if (!rc && two) rc = dev_to_file(c, f, c->s2W, c->F) || dev_to_file(c, f, c->s2V, nv);
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
    LCTR_CHECK(c->cfg.world == 1, "checkpoints are read per single-GPU trainer (world == 1)");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    FILE* f = fopen(path, "rb");
    LCTR_CHECK(f, "open file error! (%s)", path);
    CkptHeader h;
    if (!get(f, &h, sizeof(h)) || memcmp(h.magic, "LCTRCKP1", 8) != 0) {
        fclose(f);
        set_error("%s is not a lightctr_b200 checkpoint", path);
        return 1;
    }
    bool same = h.model == c->cfg.model && h.optimizer == c->cfg.optimizer && h.n_layers == c->n_layers &&
                h.feature_cnt == c->F && h.field_cnt == c->cfg.field_cnt && h.factor_cnt == c->cfg.factor_cnt &&
                h.reserved == key_word(c->cfg);
    for (int l = 0; l < c->n_layers && same; l++) same = h.in[l] == c->layers[l].in && h.out[l] == c->layers[l].out;
    if (!same) {
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
