// lightctr_b200/csrc/loader.cpp -- host-side ingest: libffm text -> CSR, bit-exact w.r.t. the reference parser.
//
// Restates FM_Algo_Abst::loadDataRow (fm_algo_abst.h:70-107):
//   per line:  sscanf("%d%n") label, skip ONE separator char, then repeatedly
//              sscanf("%zu:%zu:%f%n") >= 2 -> (field, fid, val), skip one char;
//   feature_cnt = max(fid)+1 (:95); field_cnt only grows when the ctor passed > 0 (:96-98);
//   rows without features are skipped -- but their label was already appended (:90,101-103), which
//   shifts every later label; that quirk is reproduced (label_cnt >= rows).
// Well-formed tokens ("digits:digits:number") take the fast grammar of libffm_grammar.h, which the device parser
// (text.cu) shares; anything else falls back to the very sscanf call of the reference, including its stale-%n /
// stale-val behaviour when only two fields parse (:92).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/lightctr_b200.h"
#include "libffm_grammar.h"
#include "loader.h"

namespace lctr {
void set_error(const char* fmt, ...);
}

namespace {

// A token: the shared grammar, strtof where its decimal conversion declines, and the reference's sscanf for the rest
// (including its stale-%n / stale-val behaviour when only two fields parse, fm_algo_abst.h:92).  false: the line ends.
inline bool read_token(const char* p, const char* end, size_t* fieldid, size_t* fid, float* val, int* nchar) {
    uint64_t a = 0, b = 0;
    float v = 0.f;
    int n = 0;
    const char* fs = nullptr;
    const int t = lctr::ffm::token(p, end, &a, &b, &v, &n, &fs);
    if (t == lctr::ffm::TOKEN_VALUE) {
        char* endp = nullptr;
        v = strtof(fs, &endp);
        if (endp != p + n) return sscanf(p, "%zu:%zu:%f%n", fieldid, fid, val, nchar) >= 2;
    } else if (t == lctr::ffm::TOKEN_NO) {
        return sscanf(p, "%zu:%zu:%f%n", fieldid, fid, val, nchar) >= 2;
    }
    *fieldid = a; *fid = b; *val = v; *nchar = n;
    return true;
}

// One line of the parse (fm_algo_abst.h:84-104), appended to out.  val / nchar: the state the reference's loop carries
// from token to token and from line to line.
template <typename Id>
static int parse_line_t(const char* base, size_t len, lctr::Parsed<Id>& out, float& val, int& nchar, uint64_t* bad_fid,
                        uint64_t* bad_field) {
    const char* end = base + (int)len;
    const char* p = base;
    const size_t row_start = out.ids.size();
    int y = 0;
    bool got = lctr::ffm::label(p, end, &y, &nchar);
    if (!got) got = sscanf(p, "%d%n", &y, &nchar) >= 1;
    if (got) {
        p += nchar + 1;
        out.labels.push_back(y);
        size_t fid = 0, fieldid = 0;
        while (p < end) {
            if (!read_token(p, end, &fieldid, &fid, &val, &nchar)) break;
            p += nchar + 1;
            if ((sizeof(Id) < 8 && fid >= (1ull << 32)) || fieldid >= (1ull << 16)) {
                *bad_fid = fid;
                *bad_field = fieldid;
                return 1;
            }
            out.ids.push_back((Id)fid);
            out.fields.push_back((uint16_t)fieldid);
            out.vals.push_back(val);
            if (fid + 1 > out.feature_cnt) out.feature_cnt = fid + 1;
            if (out.field_cnt > 0 && fieldid + 1 > out.field_cnt) out.field_cnt = fieldid + 1;
        }
    }
    if (out.ids.size() != row_start) out.row_ptr.push_back((int64_t)out.ids.size());
    return 0;
}

template <typename Id>
static int parse_libffm(const char* path, lctr::Parsed<Id>& out) {
    FILE* f = fopen(path, "rb");
    if (!f) { lctr::set_error("open file error! (%s)", path); return 1; }  // fm_algo_abst.h:79-82
    std::string buf;
    {
        char tmp[1 << 16];
        size_t n;
        while ((n = fread(tmp, 1, sizeof(tmp), f)) > 0) buf.append(tmp, n);
    }
    fclose(f);
    int nchar = 0;
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
        uint64_t fid = 0, fieldid = 0;
        if (parse_line_t(line.c_str(), line.length(), out, val, nchar, &fid, &fieldid)) {
            lctr::set_error("lctr_load_libffm: fid %zu / field %zu exceed the device index types (u32/u16)", (size_t)fid,
                            (size_t)fieldid);
            return 1;
        }
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

namespace lctr {
int parse_line(const char* line, size_t len, Parsed<uint64_t>& out, float& val, int& nchar, uint64_t* bad_fid,
               uint64_t* bad_field) {
    return parse_line_t(line, len, out, val, nchar, bad_fid, bad_field);
}
}  // namespace lctr

extern "C" int lctr_load_libffm(const char* path, uint64_t field_cnt, uint64_t feature_cnt, lctr_dataset** out) {
    if (!path || !out) { lctr::set_error("lctr_load_libffm: null argument"); return 1; }
    lctr::Parsed<uint32_t> r;
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
    lctr::Parsed<uint64_t> r;
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
