// lightctr_b200/csrc/loader.cpp -- host-side ingest: libffm text -> CSR, bit-exact w.r.t. the reference parser.
//
// Restates FM_Algo_Abst::loadDataRow (fm_algo_abst.h:70-107):
//   per line:  sscanf("%d%n") label, skip ONE separator char, then repeatedly
//              sscanf("%zu:%zu:%f%n") >= 2 -> (field, fid, val), skip one char;
//   feature_cnt = max(fid)+1 (:95); field_cnt only grows when the ctor passed > 0 (:96-98);
//   rows without features are skipped -- but their label was already appended (:90,101-103), which
//   shifts every later label; that quirk is reproduced (label_cnt >= rows).
// Well-formed tokens ("digits:digits:number") take a hand-written fast path (strtoul/strtof, the
// conversions scanf itself uses); anything else falls back to the very sscanf call of the reference,
// including its stale-%n / stale-val behaviour when only two fields parse (:92).
#include <ctype.h>
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/lightctr_b200.h"

namespace lctr {
void set_error(const char* fmt, ...);
}

namespace {

inline bool fast_token(const char* p, size_t* fieldid, size_t* fid, float* val, int* nchar) {
    const char* s = p;
    while (isspace((unsigned char)*s)) s++;
    if (!isdigit((unsigned char)*s)) return false;
    size_t a = 0;
    int nd = 0;
    while (isdigit((unsigned char)*s)) { a = a * 10 + (size_t)(*s - '0'); s++; if (++nd > 18) return false; }
    if (*s != ':') return false;
    s++;
    if (!isdigit((unsigned char)*s)) return false;
    size_t b = 0;
    nd = 0;
    while (isdigit((unsigned char)*s)) { b = b * 10 + (size_t)(*s - '0'); s++; if (++nd > 18) return false; }
    if (*s != ':') return false;
    s++;
    // %f: optional sign, digits with optional '.', optional exponent; keep the fast path to plain decimals
    const char* fs = s;
    if (*s == '-' || *s == '+') s++;
    if (!isdigit((unsigned char)*s) && *s != '.') return false;
    bool digits = false;
    while (isdigit((unsigned char)*s)) { s++; digits = true; }
    if (*s == '.') { s++; while (isdigit((unsigned char)*s)) { s++; digits = true; } }
    if (!digits) return false;
    if (*s == 'e' || *s == 'E' || *s == 'x' || *s == 'X' || isalpha((unsigned char)*s)) return false;  // let scanf decide
    char* endp = nullptr;
    const float v = strtof(fs, &endp);
    if (endp != s) return false;
    *fieldid = a; *fid = b; *val = v; *nchar = (int)(s - p);
    return true;
}

inline bool fast_label(const char* p, int* y, int* nchar) {
    const char* s = p;
    while (isspace((unsigned char)*s)) s++;
    bool neg = false;
    if (*s == '-' || *s == '+') { neg = *s == '-'; s++; }
    if (!isdigit((unsigned char)*s)) return false;
    long v = 0;
    int nd = 0;
    while (isdigit((unsigned char)*s)) { v = v * 10 + (*s - '0'); s++; if (++nd > 9) return false; }
    *y = (int)(neg ? -v : v);
    *nchar = (int)(s - p);
    return true;
}

// The parse itself, shared by the dense and the keyed loader.  Id = uint32_t: ids >= 2^32 are an error (the dense
// tables are indexed by them); Id = uint64_t: ids keep the full %zu width (keyed mode hashes them into rows).
template <typename Id>
struct Parsed {
    std::vector<int64_t> row_ptr{0};
    std::vector<Id> ids;
    std::vector<uint16_t> fields;
    std::vector<float> vals;
    std::vector<int32_t> labels;
    uint64_t feature_cnt = 0, field_cnt = 0;
};

template <typename Id>
static int parse_libffm(const char* path, Parsed<Id>& out) {
    FILE* f = fopen(path, "rb");
    if (!f) { lctr::set_error("open file error! (%s)", path); return 1; }  // fm_algo_abst.h:79-82
    std::string buf;
    {
        char tmp[1 << 16];
        size_t n;
        while ((n = fread(tmp, 1, sizeof(tmp), f)) > 0) buf.append(tmp, n);
    }
    fclose(f);
    std::vector<int64_t>& row_ptr = out.row_ptr;
    std::vector<Id>& fids = out.ids;
    std::vector<uint16_t>& fields = out.fields;
    std::vector<float>& vals = out.vals;
    std::vector<int32_t>& labels = out.labels;
    uint64_t& feature_cnt = out.feature_cnt;
    uint64_t& field_cnt = out.field_cnt;
    int nchar = 0, y = 0;
    size_t fid = 0, fieldid = 0;
    float val = 0;
    size_t pos = 0;
    const size_t N = buf.size();
    std::string line;
    bool more = N > 0;
    while (more) {
        // std::getline: up to '\n' (dropped).  A final line without '\n' is still processed; a trailing
        // empty read at EOF parses nothing.
        size_t nl = buf.find('\n', pos);
        if (nl == std::string::npos) { line.assign(buf, pos, N - pos); more = false; }
        else { line.assign(buf, pos, nl - pos); pos = nl + 1; if (pos >= N) more = false; }
        const char* base = line.c_str();
        const char* end = base + (int)line.length();
        const char* p = base;
        const size_t row_start = fids.size();
        bool got = fast_label(p, &y, &nchar);
        if (!got) got = sscanf(p, "%d%n", &y, &nchar) >= 1;
        if (got) {
            p += nchar + 1;
            labels.push_back(y);
            while (p < end) {
                if (!fast_token(p, &fieldid, &fid, &val, &nchar)) {
                    if (!(sscanf(p, "%zu:%zu:%f%n", &fieldid, &fid, &val, &nchar) >= 2)) break;
                }
                p += nchar + 1;
                if ((sizeof(Id) < 8 && fid >= (1ull << 32)) || fieldid >= (1ull << 16)) {
                    lctr::set_error("lctr_load_libffm: fid %zu / field %zu exceed the device index types (u32/u16)", fid, fieldid);
                    return 1;
                }
                fids.push_back((Id)fid);
                fields.push_back((uint16_t)fieldid);
                vals.push_back(val);
                if (fid + 1 > feature_cnt) feature_cnt = fid + 1;
                if (field_cnt > 0 && fieldid + 1 > field_cnt) field_cnt = fieldid + 1;
            }
        }
        if (fids.size() == row_start) continue;
        row_ptr.push_back((int64_t)fids.size());
    }
    return 0;
}

template <typename T>
static T* copy_out(const std::vector<T>& v) {
    T* p = (T*)malloc(sizeof(T) * (v.size() ? v.size() : 1));
    if (v.size()) memcpy(p, v.data(), sizeof(T) * v.size());
    return p;
}

}  // namespace

extern "C" int lctr_load_libffm(const char* path, uint64_t field_cnt, uint64_t feature_cnt, lctr_dataset** out) {
    if (!path || !out) { lctr::set_error("lctr_load_libffm: null argument"); return 1; }
    Parsed<uint32_t> r;
    r.feature_cnt = feature_cnt;
    r.field_cnt = field_cnt;
    if (parse_libffm(path, r)) return 1;
    lctr_dataset* d = (lctr_dataset*)calloc(1, sizeof(lctr_dataset));
    d->rows = (int64_t)r.row_ptr.size() - 1;
    d->nnz = (int64_t)r.ids.size();
    d->label_cnt = (int64_t)r.labels.size();
    d->feature_cnt = r.feature_cnt;
    d->field_cnt = r.field_cnt;
    d->row_ptr = copy_out(r.row_ptr);
    d->fid = copy_out(r.ids);
    d->field = copy_out(r.fields);
    d->val = copy_out(r.vals);
    d->label = copy_out(r.labels);
    *out = d;
    return 0;
}

extern "C" int lctr_load_libffm_keys(const char* path, uint64_t field_cnt, lctr_keyed_dataset** out) {
    if (!path || !out) { lctr::set_error("lctr_load_libffm_keys: null argument"); return 1; }
    Parsed<uint64_t> r;
    r.field_cnt = field_cnt;
    if (parse_libffm(path, r)) return 1;
    lctr_keyed_dataset* d = (lctr_keyed_dataset*)calloc(1, sizeof(lctr_keyed_dataset));
    d->rows = (int64_t)r.row_ptr.size() - 1;
    d->nnz = (int64_t)r.ids.size();
    d->label_cnt = (int64_t)r.labels.size();
    d->field_cnt = r.field_cnt;
    d->row_ptr = copy_out(r.row_ptr);
    d->key = copy_out(r.ids);
    d->field = copy_out(r.fields);
    d->val = copy_out(r.vals);
    d->label = copy_out(r.labels);
    *out = d;
    return 0;
}

extern "C" int lctr_free_keyed_dataset(lctr_keyed_dataset* d) {
    if (!d) return 0;
    free(d->row_ptr); free(d->key); free(d->field); free(d->val); free(d->label); free(d);
    return 0;
}

extern "C" int lctr_free_dataset(lctr_dataset* d) {
    if (!d) return 0;
    free(d->row_ptr); free(d->fid); free(d->field); free(d->val); free(d->label); free(d);
    return 0;
}
