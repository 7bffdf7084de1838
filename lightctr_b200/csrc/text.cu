// lightctr_b200/csrc/text.cu -- libffm text parsed into a batch slot on the device (lctr_upload_libffm).
//
// The slots of a sequence of calls hold, bit for bit, what lctr_load_libffm gives on the concatenated text and
// lctr_upload_batch puts into a slot (keyed contexts: lctr_load_libffm_keys, then lctr_upload_batch_keys).  One call:
//   1. the text is copied into a staging buffer; text_count_kernel + text_scan_kernel count the '\n' of each 16 KB tile,
//      text_index_kernel writes where every line ends;
//   2. text_parse_kernel, one thread per line, parses the line against the fast grammar of libffm_grammar.h and records
//      its entry count, label and last value, or declines the whole line when one of its tokens is outside the grammar;
//      text_declined_kernel finds for each declined line the line whose value a two-field token there would keep;
//   3. one read of the totals (and of the declined list, when there is one): the host parses the declined lines with the
//      loader's own parser (loader.cpp) and sends their entries back; errors are raised here, naming the first line;
//   4. text_tile_kernel + text_scan_kernel + text_write_kernel place every line's entries (a second parse of the device
//      lines), row_ptr and labels -- keyed contexts parse the ids into the translate's key scratch;
//   5. the labels move into the slot, and the upload ends as every upload does (upload_tail, capi.cu).
// Across calls the context keeps what the reference's loop carries from line to line: the value a two-field token keeps,
// and the labels of featureless lines not yet given to a row (each such line shifts every later row's label).
#include <string.h>

#include <algorithm>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <string>
#include <vector>

#include "common.cuh"
#include "libffm_grammar.h"
#include "loader.h"

namespace lctr {
namespace {

constexpr int kTextThreads = 256;                                // threads per block of every text kernel
constexpr int kTextBytes = 64;                                   // bytes per thread of the line index
constexpr size_t kTextTile = (size_t)kTextThreads * kTextBytes;  // bytes per block of the line index
constexpr int kScanThreads = 512;
constexpr uint32_t kNoLine = 0xffffffffu;
enum : uint8_t { LINE_LABEL = 1, LINE_TOKENS = 2, LINE_DECLINED = 4 };
enum { ERR_INDEX = 0, ERR_FIELD = 1, ERR_FID = 2, ERR_KINDS = 3 };

struct TextTotals {
    unsigned long long lines;           // '\n' in the text
    unsigned long long nnz, max_id;     // over the lines the device parsed
    unsigned int rows, labels, declined, max_field, not_one;
    unsigned int err[ERR_KINDS];        // first line with: an id / field beyond u32 / u16, a field >= field_cnt, a fid >= F
    unsigned int end_dev;               // 1: the value the next call carries is end_val (else the host's)
    float end_val;
};
// a declined line [begin, end); dev = 1: the value its two-field tokens would keep is val, from a device line before it
struct Declined {
    uint32_t line, begin, end, dev;
    float val;
};
// a declined line as the host parsed it: its entries at [off, off + cnt) of the host arrays
struct HostLine {
    unsigned long long off;
    uint32_t cnt, line;
    int32_t label;
    uint32_t got;
};
struct Limits {
    unsigned long long F;   // dense contexts: ids must be below it
    uint32_t field_cnt;     // FFM / Wide&Deep: fields must be below it (0: not checked)
    bool dense;
};

// One line [b, e) against the fast grammar: false = declined.  Otherwise *got / *y is its label and emit(field, id, val)
// runs for each token in order.  A remainder of whitespace only ends the line, as sscanf returning EOF does; a line of
// whitespace only has no label.
template <typename Emit>
__device__ bool grammar_line(const char* b, const char* e, bool* got, int* y, Emit emit) {
    int nchar = 0;
    if (!ffm::label(b, e, y, &nchar)) {
        for (const char* s = b; s < e; s++)
            if (!ffm::is_space(*s)) return false;
        *got = false;
        return true;
    }
    *got = true;
    for (const char* p = b + nchar + 1; p < e; p += nchar + 1) {
        uint64_t f = 0, id = 0;
        float v = 0.f;
        const char* vb = nullptr;
        const int t = ffm::token(p, e, &f, &id, &v, &nchar, &vb);
        if (t == ffm::TOKEN_VALUE) return false;
        if (t == ffm::TOKEN_NO) {
            for (const char* s = p; s < e; s++)
                if (!ffm::is_space(*s)) return false;
            return true;
        }
        emit(f, id, v);
    }
    return true;
}

// '\n' bytes in [base, min(base + kTextBytes, bytes)); base is a multiple of kTextBytes (16 B loads)
__device__ __forceinline__ int newlines_at(const char* text, size_t base, size_t bytes) {
    int n = 0;
    if (base + kTextBytes <= bytes) {
        const uint4* p = reinterpret_cast<const uint4*>(text + base);
#pragma unroll
        for (int j = 0; j < kTextBytes / 16; j++) {
            const uint4 v = p[j];
            n += __popc(__vcmpeq4(v.x, 0x0a0a0a0au)) + __popc(__vcmpeq4(v.y, 0x0a0a0a0au)) +
                 __popc(__vcmpeq4(v.z, 0x0a0a0a0au)) + __popc(__vcmpeq4(v.w, 0x0a0a0a0au));
        }
        return n >> 3;  // __vcmpeq4 sets 8 bits per equal byte
    }
    for (size_t q = base; q < bytes; q++) n += text[q] == '\n';
    return n;
}

__global__ void text_count_kernel(const char* text, size_t bytes, unsigned long long* tile_cnt) {
    typedef cub::BlockReduce<int, kTextThreads> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const int n = newlines_at(text, (size_t)blockIdx.x * kTextTile + (size_t)threadIdx.x * kTextBytes, bytes);
    const int sum = Reduce(tmp).Sum(n);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = (unsigned long long)sum;
}

// exclusive prefix sums of a[0, n) (and b, when given) in place, one block; *total = the sum of a
__global__ void __launch_bounds__(kScanThreads) text_scan_kernel(unsigned long long* a, unsigned long long* b, uint32_t n, unsigned long long* total) {
    typedef cub::BlockScan<unsigned long long, kScanThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    unsigned long long ca = 0, cb = 0;  // every thread keeps the carries (the aggregates are broadcast by the scan)
    for (uint32_t base = 0; base < n; base += kScanThreads) {
        const uint32_t i = base + threadIdx.x;
        unsigned long long o, agg;
        Scan(tmp).ExclusiveSum(i < n ? a[i] : 0ull, o, agg);
        if (i < n) a[i] = o + ca;
        ca += agg;
        __syncthreads();
        if (b) {
            Scan(tmp).ExclusiveSum(i < n ? b[i] : 0ull, o, agg);
            if (i < n) b[i] = o + cb;
            cb += agg;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0 && total) *total = ca;
}

// line_end[l] = position of the l-th '\n'; tail_line != kNoLine: the text's last line ends at `bytes` without one
__global__ void text_index_kernel(const char* text, size_t bytes, const unsigned long long* tile_off, uint32_t* line_end,
                                  uint32_t tail_line) {
    typedef cub::BlockScan<int, kTextThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const size_t base = (size_t)blockIdx.x * kTextTile + (size_t)threadIdx.x * kTextBytes;
    const int n = newlines_at(text, base, bytes);
    int before;
    Scan(tmp).ExclusiveSum(n, before);
    if (n) {
        uint32_t k = (uint32_t)tile_off[blockIdx.x] + (uint32_t)before;
        const size_t e = base + kTextBytes < bytes ? base + kTextBytes : bytes;
        for (size_t q = base; q < e; q++)
            if (text[q] == '\n') line_end[k++] = (uint32_t)q;
    }
    if (tail_line != kNoLine && blockIdx.x == 0 && threadIdx.x == 0) line_end[tail_line] = (uint32_t)bytes;
}

// pass 1, a thread per line: entry count, label, last value and the errors of each line the grammar takes; the others
// go to the declined list (in any order: the host sorts it)
__global__ void text_parse_kernel(const char* text, const uint32_t* line_end, uint32_t nlines, Limits lim, uint32_t* cnt,
                                  int32_t* lab, uint8_t* flag, float* last, Declined* decl, TextTotals* tot) {
    __shared__ unsigned long long s_nnz, s_max_id;
    __shared__ unsigned int s_rows, s_labels, s_max_field, s_not_one;
    if (threadIdx.x == 0) { s_nnz = 0; s_max_id = 0; s_rows = 0; s_labels = 0; s_max_field = 0; s_not_one = 0; }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nlines) {
        const uint32_t b = i ? line_end[i - 1] + 1 : 0, e = line_end[i];
        uint32_t n = 0, max_field = 0, err = 0;
        unsigned long long max_id = 0;
        float v_last = 0.f;
        bool not_one = false, got = false;
        int y = 0;
        const bool ok = grammar_line(text + b, text + e, &got, &y, [&](uint64_t f, uint64_t id, float v) {
            n++;
            v_last = v;
            not_one |= v != 1.0f;
            max_id = max_id > id ? max_id : id;
            max_field = max_field > (uint32_t)f ? max_field : (uint32_t)f;
            if ((lim.dense && id >= (1ull << 32)) || f >= (1ull << 16)) err |= 1u << ERR_INDEX;
            if (lim.field_cnt && f >= lim.field_cnt) err |= 1u << ERR_FIELD;
            if (lim.dense && id >= lim.F) err |= 1u << ERR_FID;
        });
        if (!ok) {
            cnt[i] = 0;
            flag[i] = LINE_DECLINED;
            const unsigned int k = atomicAdd(&tot->declined, 1u);
            decl[k] = Declined{i, b, e, 0, 0.f};
        } else {
            cnt[i] = n;
            lab[i] = y;
            last[i] = v_last;
            flag[i] = (got ? LINE_LABEL : 0) | (n ? LINE_TOKENS : 0);
            for (int k = 0; k < ERR_KINDS; k++)
                if (err & (1u << k)) atomicMin(&tot->err[k], i);
            if (n) {
                atomicAdd(&s_nnz, (unsigned long long)n);
                atomicAdd(&s_rows, 1u);
                atomicMax(&s_max_id, max_id);
                atomicMax(&s_max_field, max_field);
                if (not_one) s_not_one = 1;
            }
            if (got) atomicAdd(&s_labels, 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_nnz) {
            atomicAdd(&tot->nnz, s_nnz);
            atomicAdd(&tot->rows, s_rows);
            atomicMax(&tot->max_id, s_max_id);
            atomicMax(&tot->max_field, s_max_field);
            if (s_not_one) atomicOr(&tot->not_one, 1u);
        }
        if (s_labels) atomicAdd(&tot->labels, s_labels);
    }
}

// The line whose last value a two-field token on line `from` keeps: the nearest line before it with tokens.  true with
// *v when that is a device line; false when it is a declined line (the host's running value) or there is none in this
// text (the value carried in from the previous call, which the host also holds).
__device__ bool value_before(uint32_t from, const uint8_t* flag, const float* last, float* v) {
    int64_t j = (int64_t)from - 1;
    while (j >= 0 && !(flag[j] & (LINE_TOKENS | LINE_DECLINED))) j--;
    if (j < 0 || (flag[j] & LINE_DECLINED)) return false;
    *v = last[j];
    return true;
}

// for k < declined: the value declined line k starts from; k == declined: the value the next call starts from
__global__ void text_declined_kernel(Declined* decl, TextTotals* tot, const uint8_t* flag, const float* last, uint32_t nlines) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x, n = tot->declined;
    if (k > n) return;
    float v = 0.f;
    const bool dev = value_before(k < n ? decl[k].line : nlines, flag, last, &v);
    if (k < n) {
        decl[k].dev = dev;
        decl[k].val = v;
    } else {
        tot->end_dev = dev;
        tot->end_val = v;
    }
}

// the host's parse of the declined lines into the per-line arrays
__global__ void text_fix_kernel(const HostLine* hl, uint32_t n, uint32_t* cnt, int32_t* lab, uint8_t* flag, uint32_t* hidx) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const HostLine h = hl[k];
    cnt[h.line] = h.cnt;
    lab[h.line] = h.label;
    flag[h.line] = LINE_DECLINED | (h.got ? LINE_LABEL : 0);
    hidx[h.line] = k;
}

// per tile of kTextThreads lines: entries, and rows << 32 | labels
__global__ void text_tile_kernel(const uint32_t* cnt, const uint8_t* flag, uint32_t nlines, unsigned long long* tile_nnz,
                                 unsigned long long* tile_rl) {
    typedef cub::BlockReduce<unsigned long long, kTextThreads> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long n = i < nlines ? cnt[i] : 0;
    const unsigned long long rl = i < nlines ? ((n ? 1ull << 32 : 0ull) | (flag[i] & LINE_LABEL ? 1ull : 0ull)) : 0ull;
    const unsigned long long a = Reduce(tmp).Sum(n);
    __syncthreads();
    const unsigned long long b = Reduce(tmp).Sum(rl);
    if (threadIdx.x == 0) { tile_nnz[blockIdx.x] = a; tile_rl[blockIdx.x] = b; }
}

struct TextOut {
    int64_t* row_ptr;
    uint32_t* fid;              // dense contexts
    unsigned long long* key;    // keyed contexts: the translate's key scratch
    uint16_t* field;
    float* val;                 // null: every value is 1.0f
    int32_t* labels;            // [queue | this text's labels]
};
struct HostEntries {
    const HostLine* hl;
    const uint32_t* hidx;
    const unsigned long long* id;
    const uint16_t* field;
    const float* val;
};

// pass 2, a thread per line: the line's offsets from the tile scans, then its row_ptr entry, label and entries (a second
// parse of a device line, a copy of the host's entries for a declined one)
__global__ void text_write_kernel(const char* text, const uint32_t* line_end, uint32_t nlines, const uint32_t* cnt,
                                  const uint8_t* flag, const int32_t* lab, HostEntries h, const unsigned long long* tile_nnz,
                                  const unsigned long long* tile_rl, uint32_t queued, TextOut o) {
    typedef cub::BlockScan<unsigned long long, kTextThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < nlines;
    const uint32_t n = in ? cnt[i] : 0;
    const uint8_t fl = in ? flag[i] : 0;
    unsigned long long off, rl;
    Scan(tmp).ExclusiveSum((unsigned long long)n, off);
    __syncthreads();
    Scan(tmp).ExclusiveSum((n ? 1ull << 32 : 0ull) | (fl & LINE_LABEL ? 1ull : 0ull), rl);
    off += tile_nnz[blockIdx.x];
    rl += tile_rl[blockIdx.x];
    if (i == 0) o.row_ptr[0] = 0;
    if (!in) return;
    if (fl & LINE_LABEL) o.labels[queued + (uint32_t)rl] = lab[i];
    if (n == 0) return;
    o.row_ptr[(rl >> 32) + 1] = (int64_t)(off + n);
    if (fl & LINE_DECLINED) {
        const HostLine hl = h.hl[h.hidx[i]];
        for (uint32_t j = 0; j < n; j++) {
            const unsigned long long id = h.id[hl.off + j];
            if (o.key) o.key[off + j] = id;
            else o.fid[off + j] = (uint32_t)id;
            o.field[off + j] = h.field[hl.off + j];
            if (o.val) o.val[off + j] = h.val[hl.off + j];
        }
        return;
    }
    const uint32_t b = i ? line_end[i - 1] + 1 : 0, e = line_end[i];
    bool got;
    int y;
    unsigned long long w = off;
    grammar_line(text + b, text + e, &got, &y, [&](uint64_t f, uint64_t id, float v) {
        if (o.key) o.key[w] = id;
        else o.fid[w] = (uint32_t)id;
        o.field[w] = (uint16_t)f;
        if (o.val) o.val[w] = v;
        w++;
    });
}

unsigned blocks_for(uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); }

}  // namespace

struct TextState {
    Buf<char> text;
    size_t cap_text = 0;
    Buf<unsigned long long> tile_a, tile_b;
    size_t cap_tiles = 0;
    Buf<uint32_t> line_end, cnt, hidx;
    Buf<int32_t> lab;
    Buf<uint8_t> flag;
    Buf<float> last;
    Buf<Declined> decl;
    size_t cap_lines = 0;
    Buf<TextTotals> tot;
    HostBuf<TextTotals> h_tot;
    Buf<HostLine> hl;
    size_t cap_hl = 0;
    Buf<unsigned long long> h_id;
    Buf<uint16_t> h_field;
    Buf<float> h_val;
    size_t cap_hent = 0;
    Buf<int32_t> labels;
    size_t cap_labels = 0;
    // what the reference's loop carries from line to line, as of the last call that succeeded
    float val = 0.f;              // the value a two-field token keeps
    std::vector<int32_t> queue;   // labels parsed but not yet given to a row (one per featureless line so far)
    int64_t lines = 0;            // lines consumed since LCTR_TEXT_BEGIN
};
void drop(TextState* p) { delete p; }

namespace {

// regrowth of one scratch group to n (n > cap), once the stream is done with it
template <typename... S>
int text_grow(lctr_ctx* c, size_t& cap, size_t n, S... s) {
    if (n <= cap) return 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const size_t m = std::max(n, cap + cap / 2);
    cap = 0;
    if (alloc_group(sized(s.b, m)...)) return 1;
    cap = m;
    return 0;
}
template <typename T>
struct Grow {
    Buf<T>& b;
};
template <typename T>
Grow<T> grow(Buf<T>& b) { return {b}; }

int text_upload(lctr_ctx* c, int slot, const char* text, size_t bytes, int flags, lctr_text_info* info) {
    TextState* t = c->text.get();
    Slot& s = c->slots[slot];
    const bool keyed = c->keys != nullptr, insert = !(flags & LCTR_TEXT_LOOKUP), begin = flags & LCTR_TEXT_BEGIN;
    const cudaStream_t st = c->stream;
    s.key_state = SLOT_KEYS_INVALID;  // until the whole upload has succeeded
    s.fused_valid = false;
    // the parser state this call starts from; committed to t only when it succeeds
    float val = begin ? 0.f : t->val;
    const std::vector<int32_t> queue = begin ? std::vector<int32_t>() : t->queue;
    const int64_t first_line = begin ? 0 : t->lines;
    // whole lines only: what follows the last '\n' waits for the next call, unless this text ends the file
    size_t consumed = bytes;
    if (!(flags & LCTR_TEXT_END)) {
        const void* nl = bytes ? memrchr(text, '\n', bytes) : nullptr;
        consumed = nl ? (size_t)((const char*)nl - text) + 1 : 0;
    }
    const bool tail = consumed && text[consumed - 1] != '\n';
    if (!t->tot && (t->tot.alloc(1) || t->h_tot.alloc(1))) return 1;
    TextTotals* h = t->h_tot;
    memset(h, 0, sizeof(TextTotals));
    for (int k = 0; k < ERR_KINDS; k++) h->err[k] = kNoLine;
    LCTR_CUDA(cudaMemcpyAsync(t->tot, h, sizeof(TextTotals), cudaMemcpyHostToDevice, st));
    uint32_t nlines = 0;
    const unsigned ntiles = blocks_for(consumed, (unsigned)kTextTile);
    if (consumed) {
        if (text_grow(c, t->cap_text, ntiles * kTextTile, grow(t->text)) ||
            text_grow(c, t->cap_tiles, ntiles + 1, grow(t->tile_a), grow(t->tile_b)))
            return 1;
        LCTR_CUDA(cudaMemcpyAsync(t->text, text, consumed, cudaMemcpyHostToDevice, st));
        {
            ProfScope prof(c, PROF_TEXT);
            if (launch(c, {ntiles, kTextThreads, 0, st}, text_count_kernel, t->text, consumed, t->tile_a) ||
                launch(c, {1, kScanThreads, 0, st}, text_scan_kernel, t->tile_a, nullptr, ntiles, &t->tot.get()->lines))
                return 1;
        }
        LCTR_CUDA(cudaMemcpyAsync(h, t->tot, sizeof(TextTotals), cudaMemcpyDeviceToHost, st));
        LCTR_CUDA(cudaStreamSynchronize(st));
        nlines = (uint32_t)h->lines + (tail ? 1 : 0);
    }
    // ---- pass 1
    if (nlines) {
        if (text_grow(c, t->cap_lines, nlines, grow(t->line_end), grow(t->cnt), grow(t->hidx), grow(t->lab), grow(t->flag),
                      grow(t->last), grow(t->decl)))
            return 1;
        const Limits lim{c->F, (c->cfg.model == LCTR_MODEL_FFM || c->cfg.model == LCTR_MODEL_WND) ? c->cfg.field_cnt : 0u, !keyed};
        ProfScope prof(c, PROF_TEXT);
        if (launch(c, {ntiles, kTextThreads, 0, st}, text_index_kernel, t->text, consumed, t->tile_a, t->line_end,
                   tail ? nlines - 1 : kNoLine) ||
            launch(c, {blocks_for(nlines, kTextThreads), kTextThreads, 0, st}, text_parse_kernel, t->text, t->line_end, nlines,
                   lim, t->cnt, t->lab, t->flag, t->last, t->decl, t->tot) ||
            launch(c, {blocks_for(nlines + 1ull, kTextThreads), kTextThreads, 0, st}, text_declined_kernel, t->decl, t->tot,
                   t->flag, t->last, nlines))
            return 1;
    }
    LCTR_CUDA(cudaMemcpyAsync(h, t->tot, sizeof(TextTotals), cudaMemcpyDeviceToHost, st));
    LCTR_CUDA(cudaStreamSynchronize(st));
    const TextTotals tot = *h;
    // ---- the declined lines, in order, through the loader's parser
    std::vector<Declined> decl(tot.declined);
    if (tot.declined) {
        LCTR_CUDA(cudaMemcpyAsync(decl.data(), t->decl, decl.size() * sizeof(Declined), cudaMemcpyDeviceToHost, st));
        LCTR_CUDA(cudaStreamSynchronize(st));
        std::sort(decl.begin(), decl.end(), [](const Declined& a, const Declined& b) { return a.line < b.line; });
    }
    const uint32_t field_cnt = (c->cfg.model == LCTR_MODEL_FFM || c->cfg.model == LCTR_MODEL_WND) ? c->cfg.field_cnt : 0u;
    uint32_t err[ERR_KINDS + 1];  // + the reserved key (keyed contexts)
    for (int k = 0; k < ERR_KINDS; k++) err[k] = tot.err[k];
    err[ERR_KINDS] = kNoLine;
    Parsed<uint64_t> hp;
    std::vector<HostLine> hl(decl.size());
    bool host_not_one = false;
    uint64_t host_max_id = 0, host_max_field = 0;
    std::string line;
    for (size_t k = 0; k < decl.size(); k++) {
        const Declined& d = decl[k];
        if (d.line > err[ERR_INDEX]) break;  // the loader stops at its first error
        if (d.dev) val = d.val;
        line.assign(text + d.begin, d.end - d.begin);
        const size_t e0 = hp.ids.size(), l0 = hp.labels.size();
        int nchar = 0;
        uint64_t bad_fid = 0, bad_field = 0;
        const bool index_err = parse_line(line.c_str(), line.size(), hp, val, nchar, &bad_fid, &bad_field) != 0;
        HostLine& x = hl[k];
        x.off = e0;
        x.cnt = (uint32_t)(hp.ids.size() - e0);
        x.line = d.line;
        x.got = hp.labels.size() > l0;
        x.label = x.got ? hp.labels.back() : 0;
        for (size_t j = e0; j < hp.ids.size(); j++) {
            const uint64_t id = hp.ids[j], f = hp.fields[j];
            if (!keyed && id >= (1ull << 32)) err[ERR_INDEX] = std::min(err[ERR_INDEX], d.line);
            if (field_cnt && f >= field_cnt) err[ERR_FIELD] = std::min(err[ERR_FIELD], d.line);
            if (!keyed && id >= c->F) err[ERR_FID] = std::min(err[ERR_FID], d.line);
            if (keyed && id == ~0ull) err[ERR_KINDS] = std::min(err[ERR_KINDS], d.line);
            host_not_one |= hp.vals[j] != 1.0f;
            host_max_id = std::max(host_max_id, id);
            host_max_field = std::max(host_max_field, f);
        }
        if (index_err) err[ERR_INDEX] = std::min(err[ERR_INDEX], d.line);
    }
    const long long ln0 = (long long)first_line + 1;  // line numbers count from 1 at LCTR_TEXT_BEGIN
    LCTR_CHECK(err[ERR_INDEX] == kNoLine, "lctr_upload_libffm: line %lld: a fid / field exceeds the device index types (u32/u16)",
               ln0 + err[ERR_INDEX]);
    LCTR_CHECK(err[ERR_FIELD] == kNoLine, "lctr_upload_libffm: line %lld: a field >= field_cnt %u", ln0 + err[ERR_FIELD], field_cnt);
    LCTR_CHECK(err[ERR_FID] == kNoLine, "lctr_upload_libffm: line %lld: a fid >= feature_cnt %zu", ln0 + err[ERR_FID], c->F);
    LCTR_CHECK(err[ERR_KINDS] == kNoLine, "lctr_upload_libffm: line %lld: key %llu is reserved (the empty marker of the key table)",
               ln0 + err[ERR_KINDS], ~0ull);
    if (tot.end_dev) val = tot.end_val;  // else the host's running value: the last line with tokens was declined, or none
    // ---- sizes, slot, host entries
    int64_t rows = tot.rows, labels = tot.labels;
    for (const HostLine& x : hl) { rows += x.cnt > 0; labels += x.got; }
    const int64_t nnz = (int64_t)(tot.nnz + hp.ids.size()), queued = (int64_t)queue.size();
    const bool has_val = tot.not_one || host_not_one;
    if (slot_fit(c, s, rows, nnz)) return 1;
    s.rows = rows; s.nnz = nnz;
    s.has_val = has_val;
    s.has_field = true;
    uint64_t* keys = nullptr;
    if (keyed && nnz && keys_scratch(c, (size_t)nnz, &keys)) return 1;
    if (text_grow(c, t->cap_labels, (size_t)(queued + labels) + 1, grow(t->labels)) ||
        text_grow(c, t->cap_hl, hl.size() + 1, grow(t->hl)) ||
        text_grow(c, t->cap_hent, hp.ids.size() + 1, grow(t->h_id), grow(t->h_field), grow(t->h_val)))
        return 1;
    if (queued) LCTR_CUDA(cudaMemcpyAsync(t->labels, queue.data(), queued * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (!hl.empty()) {
        LCTR_CUDA(cudaMemcpyAsync(t->hl, hl.data(), hl.size() * sizeof(HostLine), cudaMemcpyHostToDevice, st));
        if (!hp.ids.empty()) {
            const size_t n = hp.ids.size();
            LCTR_CUDA(cudaMemcpyAsync(t->h_id, hp.ids.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
            LCTR_CUDA(cudaMemcpyAsync(t->h_field, hp.fields.data(), n * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
            LCTR_CUDA(cudaMemcpyAsync(t->h_val, hp.vals.data(), n * sizeof(float), cudaMemcpyHostToDevice, st));
        }
    }
    // ---- pass 2
    if (nlines) {
        const unsigned nt = blocks_for(nlines, kTextThreads);
        if (text_grow(c, t->cap_tiles, nt + 1, grow(t->tile_a), grow(t->tile_b))) return 1;
        const HostEntries he{t->hl, t->hidx, t->h_id, t->h_field, t->h_val};
        const TextOut o{s.row_ptr, keyed ? nullptr : s.fid.get(), reinterpret_cast<unsigned long long*>(keys), s.field,
                        has_val ? s.val.get() : nullptr, t->labels};
        ProfScope prof(c, PROF_TEXT);
        if ((!hl.empty() && launch(c, {blocks_for(hl.size(), kTextThreads), kTextThreads, 0, st}, text_fix_kernel, t->hl,
                                   (uint32_t)hl.size(), t->cnt, t->lab, t->flag, t->hidx)) ||
            launch(c, {nt, kTextThreads, 0, st}, text_tile_kernel, t->cnt, t->flag, nlines, t->tile_a, t->tile_b) ||
            launch(c, {1, kScanThreads, 0, st}, text_scan_kernel, t->tile_a, t->tile_b, nt, nullptr) ||
            launch(c, {nt, kTextThreads, 0, st}, text_write_kernel, t->text, t->line_end, nlines, t->cnt, t->flag, t->lab, he,
                   t->tile_a, t->tile_b, (uint32_t)queued, o))
            return 1;
    } else {
        LCTR_CUDA(cudaMemsetAsync(s.row_ptr, 0, sizeof(int64_t), st));
    }
    // ---- labels: the first `rows` of [queue | this text's labels] go to the slot, the rest wait for later rows
    std::vector<int32_t> next((size_t)(queued + labels - rows));
    if (rows) LCTR_CUDA(cudaMemcpyAsync(s.pred, t->labels, rows * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (!next.empty())
        LCTR_CUDA(cudaMemcpyAsync(next.data(), t->labels + rows, next.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (keyed && keys_translate_scratch(c, nnz, insert, s.fid)) return 1;
    if (upload_tail(c, st, slot, rows, nnz, keyed, nullptr, nullptr, nullptr)) {
        s.key_state = SLOT_KEYS_INVALID;
        return 1;
    }
    LCTR_CUDA(cudaStreamSynchronize(st));
    s.key_state = insert ? SLOT_KEYS_OK : SLOT_KEYS_LOOKUP;
    t->val = val;
    t->queue.swap(next);
    t->lines = first_line + nlines;
    if (info) {
        info->rows = rows;
        info->nnz = s.nnz;
        info->lines = nlines;
        info->labels = labels;
        const uint64_t max_id = std::max<uint64_t>(tot.max_id, host_max_id);
        const uint64_t max_field = std::max<uint64_t>(tot.max_field, host_max_field);
        info->feature_cnt = nnz ? max_id + 1 : 0;
        info->field_cnt = nnz ? max_field + 1 : 0;
        info->host_lines = (int64_t)decl.size();
        info->consumed = consumed;
    }
    return 0;
}

}  // namespace
}  // namespace lctr

using namespace lctr;

extern "C" int lctr_upload_libffm(lctr_ctx* c, int slot, const char* text, size_t bytes, int flags, lctr_text_info* info) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(slot >= 0 && slot < kNumSlots, "lctr_upload_libffm: slot %d out of range (0..%d)", slot, kNumSlots - 1);
    LCTR_CHECK(text || bytes == 0, "lctr_upload_libffm: null text");
    LCTR_CHECK((flags & ~(LCTR_TEXT_BEGIN | LCTR_TEXT_END | LCTR_TEXT_LOOKUP)) == 0, "lctr_upload_libffm: unknown flags 0x%x", flags);
    LCTR_CHECK(c->cfg.world == 1, "lctr_upload_libffm: text uploads are single-GPU (world %d): parse the text with "
                                  "lctr_load_libffm[_keys] and upload each rank's share with lctr_upload_batch[_keys]", c->cfg.world);
    LCTR_CHECK(c->cfg.deterministic != 1, "lctr_upload_libffm: deterministic = 1 builds its feature-major view on the host from "
                                          "host arrays, which a text upload does not have (use deterministic 0 or 2, or "
                                          "lctr_load_libffm + lctr_upload_batch)");
    LCTR_CHECK(!(flags & LCTR_TEXT_LOOKUP) || c->keys, "lctr_upload_libffm: LCTR_TEXT_LOOKUP needs a keyed context "
                                                       "(key_mode = LCTR_KEYS_HASHED)");
    LCTR_CHECK(bytes < 0xffffffffull, "lctr_upload_libffm: %zu bytes of text; one call takes less than 4 GiB", bytes);
    if (!c->text) c->text.reset(new TextState());
    return text_upload(c, slot, text, bytes, flags, info);
}
