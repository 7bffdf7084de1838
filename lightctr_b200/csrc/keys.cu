// lightctr_b200/csrc/keys.cu -- keyed mode (cfg.key_mode = LCTR_KEYS_HASHED): batches carry 64-bit hashed feature keys and
// the library owns the key -> row map, creating and initialising a row the first time a key is met.  The reference has
// this capability on its distributed path only: its parameter server keys parameters by size_t in an unordered_map and
// creates a key on first touch (distribut/paramserver.h:315-339, :40-47; distributed_algo_abst.h:70-72).  Here the map is
// a device hash table and translation happens at upload, so a slot holds ordinary u32 row ids afterwards and every
// kernel of the dense path runs on it unchanged.
//
// Table: open addressing over T = 2^m >= 2 * capacity slots, each a u64 key (~0 = empty, so that key value is reserved)
// and a u32 row.  Home group = fmix64(key) mod (T / 16); probing walks whole 128-byte groups of 16 keys, one 16-lane
// tile per key (one coalesced load and two ballots per group).  Slots only ever go from empty to a key, so a group with
// an empty slot and no match ends a lookup.  fmix64 is the MurmurHash3 finaliser the reference uses for PS sharding
// (common/hash.h:51-58), without its 32-bit truncation.
//
// Upload (insert = 1) is three launches on the ctx stream:
//   1. key_insert_kernel: a tile that finds no match claims the first empty slot of the group with a 64-bit atomicCAS; the
//      winner takes a row from an atomicAdd counter and records it in the list of new rows.  A key met again in the same
//      batch finds the claimed slot with a plain load once the CAS has landed, so batch-local duplicates cost atomics only
//      while their first claim is in flight, and keys already in the table cost none.
//   2. key_init_kernel<TIERED = false>: one warp per new row (FFM rows are Fc * k floats) writes W = 0, V, and the
//      optimizer state lctr_create gives (s1 = initial_s1, s2 = 0).
//   3. key_find_kernel: the translated row of every entry into the slot's fid array -- a second launch, so no tile ever
//      waits on another tile's row inside a kernel.
// Lookup-only uploads (insert = 0) run step 3 alone: absent keys map to the null row (index capacity), all zeros and
// never updated, which drops a feature the model never trained on (the reference's rule, predict/fm_predict.cpp:122).
//
// Capacity: the claim that draws row >= capacity stores kNoRow for its key and raises a flag; the upload fails naming the
// capacity and the slot is unusable until it is uploaded again.  Keys inserted before keep their rows; a key stored with
// kNoRow fails every later insert-upload that meets it the same way, and looks up as absent.
//
// Lazy init of V: V[row][j] = scale * N(0,1), the Box-Muller of fill_params_kernel (capi.cu) with its element counter
// replaced by fmix64(key) * rowlen + j, and uniforms whose fp32 arithmetic is exact (u1 never reaches 1, where
// sqrt(-2 log u1) is steepest):
//     h = fmix64((fmix64(key) * rowlen + j) * 0x9E3779B97F4A7C15 + seed)          (all arithmetic mod 2^64)
//     u1 = ((h & 0x7fffff) + 0.5) * 2^-23,  u2 = ((h >> 24) & 0xffffff) * 2^-24    (fp32)
//     V = scale * sqrtf(-2 logf(u1)) * cosf(6.2831853 u2)
// so the values depend on (seed, key, j) only -- never on the row a key got or on the order keys arrived in.  This is a
// different stream from the reference's rand()-driven GaussRand (fm_algo_abst.h:62-65); only the scale default,
// 1 / sqrt(k), is the reference's.
//
// Several GPUs (world > 1): each rank's table is the shard of the keys it owns (top bits of fmix64(key), keys.cuh) with
// the capacity of the global rows < feature_cnt that rank holds; dist.cu translates the keys an upload sends each owner
// with the insert and init above, and the per-rank calls below take only the owned keys (lctr_upload_keyed_params) or
// return global rows (lctr_lookup_keys).
//
// Eviction (cfg.key_evict = 1; the reference's server map only grows, paramserver.h:315-339).  A host u64 clock advances
// once per insert-upload, and key_find_kernel<0> of that upload stores it into last_seen[row] of every entry it
// translates (plain stores: duplicates write the same value).  Untracked contexts pass a null stamp pointer, a uniform
// branch.  lctr_evict_keys then runs on the ctx stream:
//   survey     survivors of the max_idle rule and their largest age (two counters back to the host);
//   select     only when max_rows binds: exact radix select of the age of rank max_rows among the survivors, 16-bit
//              digits from the top significant bit of the largest age (usually one 65,536-bin pass), warp-aggregated
//              histogram + a one-block pick of the digit; the host reads back (digit, count below) per pass;
//   count/scan one flag per row, recomputed from the stamp wherever needed; per-1024-row counts, a one-block scan of
//              them, then E(r) = evicted rows below r for r in [0, n] and the evicted-row list ev[E(r)] = r;
//   export     gather of the evicted rows' key, W and V (before anything moves);
//   move       survivor r >= n_live goes to ev[(r - n_live) - (E(r) - E(n_live))], the holes below n_live in order:
//              sources all >= n_live, destinations all < n_live, so one launch moves every row with no ordering hazard;
//   reset      rows [n_live, n) back to the state lctr_create gives;
//   rebuild    table emptied and rows [0, n_live) re-inserted with row = index (key_insert_fixed_kernel).
// The per-row arrays that do not move: gW / gV and `touched` are zero between steps, fused->slot_of and touch_list are
// scratch written by each step before it reads them.  Slots hold row ids of the old numbering and become stale.
//
// Host tier (cfg.key_host_rows > 0, HostTier below): the evicted rows are first appended to the tier (tier_spill_kernel,
// after the export, before the move).  Uploads give a device row to a key the tier holds as to a new key (insert = 0:
// key_lookup_restore_kernel, for tier keys only); key_init_kernel<TIERED = true> then copies its row back in place of the
// lazy init and lists the tier row it released, and tier_compact closes the holes with evict_move_kernel.  The compaction is
// planned on the host from that list alone (the holes below the new end, sorted, and the scan of the window
// [n_live, n) above it), so its cost scales with the rows restored, never with the tier's size.  lctr_evict_host_tier
// runs the whole eviction on the tier's arrays, with scratch of the tier's size allocated for the call.
//
// Frequency admission (lctr_set_key_admission, one GPU, FM / FFM / NFM): a new key gets a row only once it has been met
// min_count times, counted in a count-min sketch of 4 rows of 2^w u32 counters in HBM, counter i of key x at
//     fmix64(x ^ ((i + 1) * 0x9E3779B97F4A7C15)) >> (64 - w)
// (the XOR keeps the cell independent of the table's low bits and the owner's top bits of fmix64(x)).  A key is present
// when the table holds it (with a row, or without one after a capacity overflow) or the tier holds it live.  An
// insert-upload then runs, in place of key_insert_kernel:
//   count   key_count_kernel: every entry of a key that is not present adds 1 to its 4 counters (entries, not distinct
//           keys, so the counts do not depend on order);
//   admit   key_admit_kernel: keys the tier holds, and keys whose smallest counter has reached min_count, go through
//           tile_insert (present keys find their slot and stop there); init / restore follow unchanged;
// and key_find_kernel<0> writes kNoRow, the drop marker, for a key still absent, counting dropped entries with one
// warp-aggregated atomic.  The host reads the count at the synchronise of read_flags.  When entries were dropped,
// keys_admission_compact (called by the upload once row_ptr / field / val are on the device, before the slot map) closes the
// gaps: D(i) = dropped entries below i by the eviction's count / scan / index kernels over the drop flags, then entry i
// moves to i - D(i) in scratch (copied back into the slot) and row_ptr[r] -= D(row_ptr[r]) in place.  Rows are never
// removed.  Counters are never cleared by eviction: an evicted key is admitted again at its next occurrence unless
// lctr_decay_key_admission (counter >>= shift, one grid-stride launch) or a new lctr_set_key_admission lowered its count.
#include <algorithm>
#include <vector>

#include <cooperative_groups.h>

#include "keys.cuh"

namespace lctr {

constexpr int kEvTile = 1024;  // rows per block of the eviction count / index kernels
constexpr int kEvBins = 1 << 16;  // radix-select digit

// grid of a warp-per-item kernel over m items (8 warps a block), and of a grid-stride kernel of one thread per item
static unsigned warp_grid(const lctr_ctx* c, size_t m) {
    return (unsigned)std::max<size_t>(1, std::min<size_t>((m + 7) / 8, (size_t)c->sm_count * 16));
}
static unsigned stride_grid(const lctr_ctx* c, size_t n) {
    return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)c->sm_count * 8));
}
// the instance of a row kernel for the context's rows: 16-byte accesses when rowlen % 4 == 0 (FM / NFM k % 4 == 0,
// FFM Fc * k % 4 == 0), scalar ones otherwise
template <class K>
static K by_rowlen(const lctr_ctx* c, K vec4, K scalar) {
    return (c->rowlen & 3) == 0 ? vec4 : scalar;
}

// the per-row arrays that move with a row
struct RowArrays {
    float *W, *V, *s1W, *s1V, *s2W, *s2V;
    unsigned long long *row_key, *last_seen;
};

// Hash index key -> row: open addressing over T = 2^m >= 2 * capacity slots of a u64 key (kEmptyKey = free) and a u32
// row, with three flag words whose meaning is the owner's ([1] is "full" for both) and their pinned mirror.  Both the
// key table and the host tier index their rows with one.
struct KeyIndex {
    Buf<unsigned long long> key;
    Buf<uint32_t> row;
    Buf<unsigned int> flags;
    HostBuf<unsigned int> h_flags;
    size_t T = 0;

    int clear(cudaStream_t st) {
        LCTR_CUDA(cudaMemsetAsync(key, 0xff, T * sizeof(unsigned long long), st));
        LCTR_CUDA(cudaMemsetAsync(row, 0xff, T * sizeof(uint32_t), st));
        LCTR_CUDA(cudaMemsetAsync(flags, 0, 3 * sizeof(unsigned int), st));
        return 0;
    }
    int alloc(size_t cap, cudaStream_t st) {
        T = kGroup;
        while (T < 2 * cap) T <<= 1;
        if (key.alloc(T) || row.alloc(T) || flags.alloc(3) || h_flags.alloc(3)) return 1;
        return clear(st);
    }
    // emptied, then key row_key[i] re-inserted with row i for i < n (v: this index's view); fails naming `what` when full
    int rebuild(lctr_ctx* c, const KeyView& v, const unsigned long long* row_key, size_t n, const char* what);
};

// Host tier (cfg.key_host_rows > 0): rows of evicted keys in pinned, device-mapped host memory, live rows [0, n), and an
// index key -> tier row in HBM (flags: [0] rows restored, [1] index full, [2] slots claimed by a spill).  Index slots go
// from empty to a key only; a restored key keeps its slot with kNoRow, so `used` (slots holding a key) counts live and
// dead slots, and the index is rebuilt from row_key[0, n) once it passes T / 2.
struct HostTier {
    RowArrays a{};                          // device-mapped host arrays of `cap` rows: views of the owners below
    MappedBuf<unsigned long long> row_key, last_seen;
    MappedBuf<float> p[6];                  // W, V, s1W, s1V, s2W, s2V
    KeyIndex ix;
    size_t cap = 0, n = 0, used = 0;
    // scratch of the compaction after a restore, sized with the key table's per-call scratch (at most one entry per new row)
    Buf<uint32_t> rel;                      // tier rows released by the current call, in no order
    Buf<uint32_t> wscan;                    // [m + 1] released rows in [n_live, n_live + i)
    Buf<uint32_t> holes;                    // released rows below n_live, ascending
};

// frequency admission (lctr_set_key_admission): the sketch, the counters of the last insert-upload, compaction scratch
constexpr int kSketchDepth = 4;
struct Admission {
    Buf<uint32_t> sketch;                   // [kSketchDepth << lw] counters
    uint32_t min_count = 0, lw = 0;
    Buf<unsigned long long> cnt;            // [3] dropped entries, admitted keys of the current upload, scan total (device)
    HostBuf<unsigned long long> h_cnt;      // pinned mirror of [0, 2)
    uint64_t dropped = 0, admitted = 0;     // of the last insert-upload
    uint64_t pending = 0;                   // entries of the upload in flight that keys_admission_compact removes
    // compaction scratch, grown on demand (per-call scratch: not counted by lctr_device_bytes)
    size_t cap = 0;
    Buf<uint32_t> scan, tiles, fid;
    Buf<uint16_t> field;
    Buf<float> val;
};

struct KeyTable {
    KeyIndex ix;                            // row kNoRow when the capacity was exhausted; flags: [0] capacity exhausted,
                                            // [1] table full, [2] new rows of this upload
    Buf<unsigned long long> row_key;        // [capacity] key of each row
    Buf<unsigned long long> count;          // rows claimed (may pass capacity: claims that got no row)
    Buf<uint32_t> new_rows;                 // rows created by this upload
    Buf<unsigned long long> d_keys;         // staging of the keys of one call
    Buf<int64_t> d_rows;                    // lookup results / fixed rows of one call
    size_t cap_scratch = 0;
    size_t cap = 0;
    unsigned long long seed = 0;
    float scale = 1.f;
    // key_evict = 1
    Buf<unsigned long long> last_seen;        // [capacity] clock of the insert-upload that last met the row
    unsigned long long clock = 0;             // insert-uploads so far
    // scratch of lctr_evict_keys, allocated by its first call
    Buf<uint32_t> ev_scan;                    // [capacity + 1] E(r)
    Buf<uint32_t> ev_rows;                    // [capacity] evicted rows, ascending
    Buf<uint32_t> ev_tiles;                   // [capacity / kEvTile + 1] per-tile counts -> offsets
    Buf<unsigned int> ev_hist;                // [65536] digit histogram of the radix select
    Buf<unsigned long long> ev_res;           // [4] counters read back by the host
    HostBuf<unsigned long long> h_res;        // pinned mirror
    std::unique_ptr<HostTier> tier;           // cfg.key_host_rows > 0
    std::unique_ptr<Admission> adm;           // lctr_set_key_admission with min_count > 1
};
void drop(KeyTable* p) { delete p; }

static KeyView view(const KeyTable* t) {
    return KeyView{t->ix.key, t->ix.row, t->row_key, t->count, t->ix.flags, t->new_rows, t->ix.T / kGroup, t->cap};
}
// the tier's index: row_key is the tier's (host) row -> key map; no row counter and no new-row list
static KeyView view(const HostTier* h) {
    return KeyView{h->ix.key, h->ix.row, h->a.row_key, nullptr, h->ix.flags, nullptr, h->ix.T / kGroup, h->cap};
}

// 1. claim a slot and a row for every key not yet in the table (one 16-lane tile per key)
__global__ void __launch_bounds__(256) key_insert_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;  // whole tiles leave together
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    tile_insert(t, keys[i], sub, gmask);
}

// keys with caller-chosen rows (lctr_upload_keyed_params): every key gets rows[i]; `record` appends the row to the new-row
// list for key_init_kernel.  rows == nullptr: key i gets row i and keys is the row -> key map itself (KeyIndex::rebuild),
// which is then left as it is.
__global__ void __launch_bounds__(256) key_insert_fixed_kernel(const unsigned long long* keys, const int64_t* __restrict__ rows,
                                                               int64_t n, KeyView t, int record) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    bool claimed;
    const long long pos = tile_claim(t, key, sub, gmask, &claimed);
    if (sub != 0) return;
    if (pos < 0) { t.flags[1] = 1u; return; }
    const uint32_t r = rows ? (uint32_t)rows[i] : (uint32_t)i;
    t.row[pos] = r;
    if (rows) t.row_key[r] = key;
    if (record) t.new_rows[atomicAdd(&t.flags[2], 1u)] = r;
}

__device__ __forceinline__ float key_gauss(unsigned long long hk, size_t rowlen, size_t j, unsigned long long seed, float scale) {
    const unsigned long long g = hk * (unsigned long long)rowlen + (unsigned long long)j;
    const unsigned long long h = fmix64(g * 0x9E3779B97F4A7C15ull + seed);
    // every step exact in fp32 up to logf / cosf; u1 lies in (0, 1) and is never 1
    const float u1 = ((float)(unsigned)(h & 0x7fffffu) + 0.5f) * 1.1920928955078125e-07f;  // 2^-23
    const float u2 = (float)(unsigned)((h >> 24) & 0xffffffu) * 5.9604644775390625e-08f;   // 2^-24
    return scale * sqrtf(-2.0f * logf(u1)) * cosf(6.2831853f * u2);
}

// lazy init of row r of key `key` by one warp: W = 0, V from the key, the optimizer state lctr_create gives
__device__ __forceinline__ void warp_lazy_init(const RowArrays& a, uint32_t r, unsigned long long key, size_t rowlen, float s1_init,
                                               unsigned long long seed, float scale, int lane) {
    const unsigned long long hk = fmix64(key);
    const size_t o = (size_t)r * rowlen;
    for (size_t j = lane; j < rowlen; j += 32) {
        a.V[o + j] = key_gauss(hk, rowlen, j, seed, scale);
        a.s1V[o + j] = s1_init;
        if (a.s2V) a.s2V[o + j] = 0.f;
    }
    if (lane == 0) {
        a.W[r] = 0.f;
        a.s1W[r] = s1_init;
        if (a.s2W) a.s2W[r] = 0.f;
    }
}

// copy of one rowlen-float row by a warp, dst row d <- src row s, 16-byte accesses when rowlen % 4 == 0 (rows are then
// 16-byte aligned); either side may be device-mapped host memory
template <bool VEC4>
__device__ __forceinline__ void warp_copy_row(float* __restrict__ dst, size_t d, const float* __restrict__ src, size_t s,
                                              size_t rowlen, int lane) {
    if (VEC4) {
        float4* d4 = reinterpret_cast<float4*>(dst + d * rowlen);
        const float4* s4 = reinterpret_cast<const float4*>(src + s * rowlen);
        for (size_t j = lane; j < rowlen / 4; j += 32) d4[j] = s4[j];
    } else {
        for (size_t j = lane; j < rowlen; j += 32) dst[d * rowlen + j] = src[s * rowlen + j];
    }
}

// every array of row s of `from` into row d of `to` (one warp)
template <bool VEC4>
__device__ __forceinline__ void warp_copy_all(const RowArrays& to, size_t d, const RowArrays& from, size_t s, size_t rowlen, int lane) {
    warp_copy_row<VEC4>(to.V, d, from.V, s, rowlen, lane);
    warp_copy_row<VEC4>(to.s1V, d, from.s1V, s, rowlen, lane);
    if (to.s2V) warp_copy_row<VEC4>(to.s2V, d, from.s2V, s, rowlen, lane);
    if (lane == 0) {
        to.W[d] = from.W[s];
        to.s1W[d] = from.s1W[s];
        if (to.s2W) to.s2W[d] = from.s2W[s];
        to.row_key[d] = from.row_key[s];
        to.last_seen[d] = from.last_seen[s];
    }
}

// 2. the rows created by this upload, one warp per row: the lazy init.  TIERED (the tier holds rows): a key found in the
//    tier index takes its row from host memory bit for bit (stamp included) instead, its index slot turns kNoRow and its
//    tier row joins the released list.
template <bool TIERED, bool VEC4>
__global__ void __launch_bounds__(256) key_init_kernel(KeyView t, KeyView h, RowArrays dev, RowArrays tier, size_t rowlen,
                                                       uint32_t* __restrict__ rel, float s1_init, unsigned long long seed,
                                                       float scale) {
    const unsigned n = t.flags[2];
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n; w += nwarps) {
        const uint32_t r = t.new_rows[w];
        const unsigned long long key = t.row_key[r];
        if constexpr (TIERED) {
            long long pos = -1;
            if (lane < kGroup) pos = tile_find(h, key, lane, 0xffffu);
            uint32_t tr = kNoRow;  // read by lane 0 alone, which later overwrites the word
            if (lane == 0 && pos >= 0) tr = h.row[pos];
            pos = __shfl_sync(~0u, pos, 0);
            tr = __shfl_sync(~0u, tr, 0);
            if (tr != kNoRow) {
                warp_copy_all<VEC4>(dev, r, tier, tr, rowlen, lane);
                if (lane == 0) {
                    h.row[pos] = kNoRow;
                    rel[atomicAdd(&h.flags[0], 1u)] = tr;
                }
                continue;
            }
        }
        warp_lazy_init(dev, r, key, rowlen, s1_init, seed, scale, lane);
    }
}

// 3'. lookup-only restore (one 16-lane tile per key): a key found live in the tier index claims a device row (the key
//     table's insert: new rows recorded for key_init_kernel, capacity flag past the capacity); others are left
__global__ void __launch_bounds__(256) key_lookup_restore_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t, KeyView h) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    const long long pos = tile_find(h, key, sub, gmask);
    if (pos < 0 || __ldg(h.row + pos) == kNoRow) return;  // whole tiles leave together
    tile_insert(t, key, sub, gmask);
}

// insert = 0, after the restore: a key still live in the tier whose device slot holds kNoRow was refused by the capacity,
// in this upload or an earlier one, and raises the capacity flag (an insert-upload's key_find_kernel raises it itself).
// A separate launch, so that no tile reads the row of a slot another tile of the same launch has just claimed.
__global__ void __launch_bounds__(256) key_tier_refused_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t, KeyView h) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    const long long pos = tile_find(t, key, sub, gmask);
    if (pos < 0 || __ldg(t.row + pos) != kNoRow) return;  // whole tiles leave together
    const long long hp = tile_find(h, key, sub, gmask);
    if (sub == 0 && hp >= 0 && h.row[hp] != kNoRow) t.flags[0] = 1u;
}

// spill of evicted device rows into tier rows base + i (warp per row, ascending old row, before anything moves), then the
// claim of each key's index slot; a dead slot of the same key is taken again
template <bool VEC4>
__global__ void __launch_bounds__(256) tier_spill_kernel(const uint32_t* __restrict__ ev_rows, size_t m, RowArrays dev, RowArrays tier,
                                                         size_t base, size_t rowlen, KeyView h) {
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < m; i += nwarps) {
        const size_t r = ev_rows[i], d = base + i;
        warp_copy_all<VEC4>(tier, d, dev, r, rowlen, lane);
        if (lane < kGroup) {
            bool claimed;
            const long long pos = tile_claim(h, dev.row_key[r], lane, 0xffffu, &claimed);
            if (lane == 0) {
                if (pos < 0) {
                    h.flags[1] = 1u;
                } else {
                    h.row[pos] = (uint32_t)d;
                    if (claimed) atomicAdd(&h.flags[2], 1u);
                }
            }
        }
    }
}

// 3. translation: MODE 0 -> u32 row per entry into a slot (absent: the null row; kNoRow: capacity flag + null row), and
//    with a stamp array (tracked context, insert-upload) last_seen[row] = clock; with a drop counter (admission on,
//    insert-upload) an absent key was not admitted: its entries get the drop marker kNoRow and are counted;
//    MODE 1 -> int64 row per key, -1 when absent or without a row
template <int MODE>
__global__ void __launch_bounds__(256) key_find_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t,
                                                       uint32_t* __restrict__ fid, int64_t* __restrict__ rows, int insert,
                                                       unsigned long long* __restrict__ last_seen, unsigned long long clock,
                                                       unsigned long long* __restrict__ dropped) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const long long pos = tile_find(t, keys[i], sub, gmask);
    if (sub != 0) return;
    const uint32_t r = pos >= 0 ? __ldg(t.row + pos) : kNoRow;
    if (MODE == 0) {
        if (dropped && pos < 0) {
            namespace cg = cooperative_groups;
            const cg::coalesced_group g = cg::coalesced_threads();
            if (g.thread_rank() == 0) atomicAdd(dropped, (unsigned long long)g.size());
            fid[i] = kNoRow;
            return;
        }
        if (r == kNoRow && insert) t.flags[pos >= 0 ? 0 : 1] = 1u;
        // hot rows appear in many entries of a batch: entries that find the stamp already written skip the store
        if (last_seen && r != kNoRow && __ldcg(last_seen + r) != clock) last_seen[r] = clock;
        fid[i] = r == kNoRow ? (uint32_t)t.cap : r;
    } else {
        rows[i] = r == kNoRow ? -1 : (int64_t)r;
    }
}

// parameters of rows given by index: warp per key
__global__ void __launch_bounds__(256) key_scatter_params_kernel(const int64_t* __restrict__ rows, int64_t n, const float* __restrict__ Win,
                                                                 const float* __restrict__ Vin, float* __restrict__ W, float* __restrict__ V,
                                                                 size_t rowlen) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x / 32);
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < n; i += nwarps) {
        const size_t r = (size_t)rows[i];
        if (Vin) warp_copy_row<false>(V, r, Vin, (size_t)i, rowlen, lane);
        if (Win && lane == 0) W[r] = Win[i];
    }
}

// stamps of rows given by index (lctr_upload_keyed_params)
__global__ void __launch_bounds__(256) key_stamp_rows_kernel(const int64_t* __restrict__ rows, int64_t n,
                                                             unsigned long long* __restrict__ last_seen, unsigned long long clock) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        last_seen[rows[i]] = clock;
}

// ---- frequency admission ----------------------------------------------------------------------------------------------
// counter i of a key: row i of the sketch, column from the top lw bits of a hash independent of the table's
__device__ __forceinline__ size_t sketch_cell(unsigned long long key, int i, unsigned lw) {
    return ((size_t)i << lw) + (size_t)(fmix64(key ^ ((unsigned long long)(i + 1) * 0x9E3779B97F4A7C15ull)) >> (64 - lw));
}

// the tier holds the key live (all lanes of the tile)
__device__ __forceinline__ bool tier_holds(const KeyView& h, unsigned long long key, int sub, unsigned gmask) {
    const long long hp = tile_find(h, key, sub, gmask);
    return hp >= 0 && __ldg(h.row + hp) != kNoRow;
}

// count: every entry of a key that is not present adds 1 to its kSketchDepth counters (lanes 0..3 of its tile)
__global__ void __launch_bounds__(256) key_count_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t, KeyView h,
                                                        int tiered, uint32_t* __restrict__ sketch, unsigned lw) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    if (tile_find(t, key, sub, gmask) >= 0) return;  // whole tiles leave together
    if (tiered && tier_holds(h, key, sub, gmask)) return;
    if (sub < kSketchDepth) atomicAdd(sketch + sketch_cell(key, sub, lw), 1u);
}

// admit + insert: keys the tier holds, and keys whose smallest counter reached min_count, go through tile_insert (a present
// key finds its slot and stops there); admitted counts the slots claimed for keys the tier did not hold
__global__ void __launch_bounds__(256) key_admit_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t, KeyView h,
                                                        int tiered, const uint32_t* __restrict__ sketch, unsigned lw,
                                                        unsigned min_count, unsigned long long* __restrict__ admitted) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    const bool restore = tiered && tier_holds(h, key, sub, gmask);
    if (!restore) {
        unsigned v = sub < kSketchDepth ? __ldg(sketch + sketch_cell(key, sub, lw)) : ~0u;
        for (int o = kGroup / 2; o; o >>= 1) v = min(v, __shfl_xor_sync(gmask, v, o));
        if (v < min_count) return;  // whole tiles leave together
    }
    if (tile_insert(t, key, sub, gmask) && !restore && sub == 0) atomicAdd(admitted, 1ull);
}

// every counter >>= shift (shift in [1, 32]); n % 4 == 0
__global__ void __launch_bounds__(256) sketch_decay_kernel(uint4* __restrict__ sketch, size_t n4, unsigned shift) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        uint4 v = sketch[i];
        if (shift >= 32) v = make_uint4(0u, 0u, 0u, 0u);
        else v = make_uint4(v.x >> shift, v.y >> shift, v.z >> shift, v.w >> shift);
        sketch[i] = v;
    }
}

// the kept entries into their dense positions i - D(i) of the scratch arrays (field / val may be null), and
// row_ptr[r] -= D(row_ptr[r]) in place; scan[i] = D(i), entries dropped below i, for i in [0, n]
__global__ void __launch_bounds__(256) admit_compact_kernel(const uint32_t* __restrict__ fid, const uint16_t* __restrict__ field,
                                                            const float* __restrict__ val, size_t n, const uint32_t* __restrict__ scan,
                                                            int64_t* __restrict__ row_ptr, size_t rows, uint32_t* __restrict__ fid2,
                                                            uint16_t* __restrict__ field2, float* __restrict__ val2) {
    const size_t m = n > rows + 1 ? n : rows + 1;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x) {
        if (i < n) {
            const uint32_t f = fid[i];
            if (f != kNoRow) {
                const size_t d = i - scan[i];
                fid2[d] = f;
                if (field) field2[d] = field[i];
                if (val) val2[d] = val[i];
            }
        }
        if (i <= rows) row_ptr[i] -= (int64_t)scan[row_ptr[i]];
    }
}

// ---- eviction ----------------------------------------------------------------------------------------------------------
// a row leaves when its age exceeds max_idle, or (limit) reaches the cutoff a* of the max_rows rule
struct EvictRule {
    unsigned long long clock, max_idle, cut;
    int limit;
};
__device__ __forceinline__ bool row_evicted(const EvictRule& e, unsigned long long stamp) {
    const unsigned long long age = e.clock - stamp;
    return age > e.max_idle || (e.limit && age >= e.cut);
}


// res[0] += rows with age <= max_idle, res[1] = max(res[1], their largest age)
__global__ void __launch_bounds__(256) evict_survey_kernel(const unsigned long long* __restrict__ last_seen, size_t n,
                                                           unsigned long long clock, unsigned long long max_idle,
                                                           unsigned long long* __restrict__ res) {
    unsigned long long cnt = 0, mx = 0;
    for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (size_t)gridDim.x * blockDim.x) {
        const unsigned long long age = clock - last_seen[r];
        if (age <= max_idle) { cnt++; mx = age > mx ? age : mx; }
    }
    for (int o = 16; o; o >>= 1) {
        cnt += __shfl_xor_sync(~0u, cnt, o);
        const unsigned long long m = __shfl_xor_sync(~0u, mx, o);
        mx = m > mx ? m : mx;
    }
    if ((threadIdx.x & 31) == 0 && cnt) {
        atomicAdd(res, cnt);
        atomicMax(res + 1, mx);
    }
}

// one radix-select pass: histogram of digit (age >> shift) & (2^width - 1) over the survivors whose bits above
// pshift equal prefix (pshift >= 64: no condition).  Ages cluster on a few values, so lanes with the same digit add once.
__global__ void __launch_bounds__(256) evict_hist_kernel(const unsigned long long* __restrict__ last_seen, size_t n,
                                                         unsigned long long clock, unsigned long long max_idle, int shift,
                                                         int width, int pshift, unsigned long long prefix,
                                                         unsigned int* __restrict__ hist) {
    const int lane = threadIdx.x & 31;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t r0 = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); r0 < n; r0 += stride) {  // warp-uniform
        const size_t r = r0 + lane;
        bool in = false;
        unsigned bin = 0;
        if (r < n) {
            const unsigned long long age = clock - last_seen[r];
            in = age <= max_idle && (pshift >= 64 || (age >> pshift) == prefix);
            bin = (unsigned)(age >> shift) & ((1u << width) - 1u);
        }
        const unsigned act = __ballot_sync(~0u, in);
        if (in) {
            const unsigned peers = __match_any_sync(act, bin);
            if (lane == __ffs(peers) - 1) atomicAdd(hist + bin, (unsigned)__popc(peers));
        }
    }
}

// the digit holding rank `rank` (0-based, ascending): res[0] = digit, res[1] = count of the smaller digits
__global__ void __launch_bounds__(1024) evict_pick_kernel(const unsigned int* __restrict__ hist, int nbins,
                                                          unsigned long long rank, unsigned long long* __restrict__ res) {
    __shared__ unsigned long long part[1024];
    const int per = (nbins + 1023) / 1024;
    const int b0 = (int)threadIdx.x * per, b1 = min(b0 + per, nbins);
    unsigned long long s = 0;
    for (int b = b0; b < b1; b++) s += hist[b];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const unsigned long long v = threadIdx.x >= (unsigned)o ? part[threadIdx.x - o] : 0ull;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    const unsigned long long incl = part[threadIdx.x], excl = incl - s;
    if (excl <= rank && rank < incl) {  // exactly one thread: rank < total
        unsigned long long below = excl;
        for (int b = b0; b < b1; b++) {
            const unsigned long long h = hist[b];
            if (rank < below + h) { res[0] = (unsigned long long)b; res[1] = below; break; }
            below += h;
        }
    }
}

// inclusive scan of one value per thread over a 1024-thread block; *total = the block's sum
__device__ __forceinline__ unsigned block_scan_incl(unsigned v, unsigned* ws, unsigned* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(~0u, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) ws[w] = x;
    __syncthreads();
    if (w == 0) {
        unsigned s = ws[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(~0u, s, o);
            if (lane >= o) s += y;
        }
        ws[lane] = s;
    }
    __syncthreads();
    const unsigned out = x + (w ? ws[w - 1] : 0u);
    *total = ws[31];
    __syncthreads();  // ws is reused by the next call
    return out;
}

// the flag the count / scan / index kernels below act on: a row the eviction rule frees, or an entry admission dropped
struct EvictFlag {
    const unsigned long long* last_seen;
    EvictRule e;
    __device__ __forceinline__ bool operator()(size_t r) const { return row_evicted(e, last_seen[r]); }
};
struct DropFlag {
    const uint32_t* fid;
    __device__ __forceinline__ bool operator()(size_t i) const { return fid[i] == kNoRow; }
};

// flagged positions per tile of kEvTile (tiles cover [0, n])
template <class Flag>
__global__ void __launch_bounds__(kEvTile) evict_count_kernel(Flag flag, size_t n, uint32_t* __restrict__ tiles) {
    const size_t r = (size_t)blockIdx.x * kEvTile + threadIdx.x;
    const int cnt = __syncthreads_count(r < n && flag(r));
    if (threadIdx.x == 0) tiles[blockIdx.x] = (uint32_t)cnt;
}

// tile counts -> exclusive offsets in place (one block); res[0] = evicted rows in all
__global__ void __launch_bounds__(1024) evict_scan_tiles_kernel(uint32_t* __restrict__ tiles, size_t ntiles,
                                                                unsigned long long* __restrict__ res) {
    __shared__ unsigned ws[32];
    unsigned carry = 0;
    for (size_t base = 0; base < ntiles; base += 1024) {
        const size_t i = base + threadIdx.x;
        const unsigned v = i < ntiles ? tiles[i] : 0u;
        unsigned tot;
        const unsigned incl = block_scan_incl(v, ws, &tot);
        if (i < ntiles) tiles[i] = carry + incl - v;
        carry += tot;
    }
    if (threadIdx.x == 0) res[0] = carry;
}

// E(r) = flagged positions below r, for r in [0, n], and (ev_rows non-null) the list ev_rows[E(r)] = r of the flagged ones
template <class Flag>
__global__ void __launch_bounds__(kEvTile) evict_index_kernel(Flag flag, size_t n, const uint32_t* __restrict__ tiles,
                                                              uint32_t* __restrict__ scan, uint32_t* __restrict__ ev_rows) {
    __shared__ unsigned ws[32];
    const size_t r = (size_t)blockIdx.x * kEvTile + threadIdx.x;
    const unsigned f = r < n && flag(r);
    unsigned tot;
    const unsigned E = tiles[blockIdx.x] + block_scan_incl(f, ws, &tot) - f;
    if (r <= n) scan[r] = E;
    if (f && ev_rows) ev_rows[E] = (uint32_t)r;
}

// export of the evicted rows (warp per row): key, W, V into dense device buffers, each may be null
__global__ void __launch_bounds__(256) evict_export_kernel(const uint32_t* __restrict__ ev_rows, size_t m, const unsigned long long* __restrict__ row_key,
                                                           const float* __restrict__ W, const float* __restrict__ V, size_t rowlen,
                                                           unsigned long long* __restrict__ keys_out, float* __restrict__ W_out,
                                                           float* __restrict__ V_out) {
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < m; i += nwarps) {
        const size_t r = ev_rows[i];
        if (V_out) warp_copy_row<false>(V_out, i, V, r, rowlen, lane);
        if (lane == 0) {
            if (keys_out) keys_out[i] = row_key[r];
            if (W_out) W_out[i] = W[r];
        }
    }
}

template <bool VEC4>
__device__ __forceinline__ void warp_fill_row(float* __restrict__ a, size_t d, size_t rowlen, float v, int lane) {
    if (VEC4) {
        float4* dst = reinterpret_cast<float4*>(a + d * rowlen);
        for (size_t j = lane; j < rowlen / 4; j += 32) dst[j] = make_float4(v, v, v, v);
    } else {
        for (size_t j = lane; j < rowlen; j += 32) a[d * rowlen + j] = v;
    }
}

// survivors at or above n_live into the holes below it (warp per row of [n_live, n); evicted rows there skip).  wscan[i]
// = E(n_live + i) for i in [0, n - n_live]: the window of the scan above n_live; holes = the rows that leave, ascending
// (only those below n_live are read)
template <bool VEC4>
__global__ void __launch_bounds__(256) evict_move_kernel(RowArrays a, size_t rowlen, size_t n_live, size_t n,
                                                         const uint32_t* __restrict__ wscan, const uint32_t* __restrict__ holes) {
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    const uint32_t e_live = wscan[0];
    for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n - n_live; w += nwarps) {
        const size_t r = n_live + w;
        const uint32_t E = wscan[w];
        if (wscan[w + 1] != E) continue;  // evicted
        const size_t d = holes[w - (E - e_live)];
        warp_copy_all<VEC4>(a, d, a, r, rowlen, lane);
    }
}

// after a tier move: the index slot of every moved row names its new row (one 16-lane tile per row of [n_live, n))
__global__ void __launch_bounds__(256) tier_reindex_kernel(KeyView h, size_t n_live, size_t n, const uint32_t* __restrict__ wscan,
                                                           const uint32_t* __restrict__ holes) {
    const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (w >= n - n_live) return;
    const size_t r = n_live + w;
    const uint32_t E = wscan[w];
    if (wscan[w + 1] != E) return;  // left the tier
    const size_t d = holes[w - (E - wscan[0])];
    const int sub = threadIdx.x & (kGroup - 1);
    const long long pos = tile_find(h, h.row_key[r], sub, 0xffffu << (threadIdx.x & 16));
    if (sub == 0 && pos >= 0) h.row[pos] = (uint32_t)d;
}

// rows [lo, hi) back to the state lctr_create gives (warp per row)
template <bool VEC4>
__global__ void __launch_bounds__(256) evict_reset_kernel(RowArrays a, size_t rowlen, size_t lo, size_t hi, float s1_init) {
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
    for (size_t r = lo + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; r < hi; r += nwarps) {
        warp_fill_row<VEC4>(a.V, r, rowlen, 0.f, lane);
        warp_fill_row<VEC4>(a.s1V, r, rowlen, s1_init, lane);
        if (a.s2V) warp_fill_row<VEC4>(a.s2V, r, rowlen, 0.f, lane);
        if (lane == 0) {
            a.W[r] = 0.f;
            a.s1W[r] = s1_init;
            if (a.s2W) a.s2W[r] = 0.f;
            a.row_key[r] = kEmptyKey;
            a.last_seen[r] = 0;
        }
    }
}

static unsigned tile_grid(int64_t n) { return (unsigned)std::max<int64_t>(1, (n * kGroup + 255) / 256); }

int KeyIndex::rebuild(lctr_ctx* c, const KeyView& v, const unsigned long long* row_key, size_t n, const char* what) {
    if (clear(c->stream)) return 1;
    if (n) {
        if (launch(c, {tile_grid((int64_t)n), 256, 0, c->stream}, key_insert_fixed_kernel, row_key, nullptr, (int64_t)n, v, 0))
            return 1;
    }
    LCTR_CUDA(cudaMemcpyAsync(h_flags, flags, 3 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    LCTR_CHECK(!h_flags[1], "%s %zu keys", what, n);
    return 0;
}

// room for n keys in the per-call scratch of the key table and of the tier compaction, grown by half at least
int scratch_reserve(lctr_ctx* c, size_t n) {
    KeyTable* t = c->keys.get();
    if (n <= t->cap_scratch) return 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const size_t cap = std::max(n, t->cap_scratch + t->cap_scratch / 2);
    HostTier* h = t->tier.get();
    t->cap_scratch = 0;
    if (h) { h->rel.reset(); h->wscan.reset(); h->holes.reset(); }
    if (alloc_group(sized(t->d_keys, cap), sized(t->d_rows, cap), sized(t->new_rows, cap))) return 1;
    if (h && alloc_group(sized(h->rel, cap), sized(h->wscan, cap + 1), sized(h->holes, cap))) {  // a call restores
        t->d_keys.reset(); t->d_rows.reset(); t->new_rows.reset();                                // <= 1 row per new row
        return 1;
    }
    t->cap_scratch = cap;
    return 0;
}

// the compaction scratch of admission for n entries
static int admission_scratch(Admission* a, size_t cap) {
    a->cap = 0;
    if (alloc_group(sized(a->scan, cap + 1), sized(a->tiles, cap / kEvTile + 1), sized(a->fid, cap), sized(a->field, cap),
                    sized(a->val, cap)))
        return 1;
    a->cap = cap;
    return 0;
}

// the scratch of lctr_evict_keys for a table of cap rows; h_res, allocated last, marks it complete
static int evict_scratch(KeyTable* t, size_t cap) {
    return alloc_group(sized(t->ev_scan, cap + 1), sized(t->ev_rows, cap), sized(t->ev_tiles, cap / kEvTile + 1),
                       sized(t->ev_hist, (size_t)kEvBins), sized(t->ev_res, 4), sized(t->h_res, 4));
}

static RowArrays device_rows(lctr_ctx* c) {
    return RowArrays{c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V, c->keys->row_key, c->keys->last_seen};
}

// tiered contexts whose tier holds rows restore the keys it holds instead of initialising them
static bool tier_live(const KeyTable* t) { return t->tier && t->tier->n > 0; }

// the rows the last insert recorded (at most max_new), initialised or restored from the tier
int init_new_rows(lctr_ctx* c, int64_t max_new) {
    KeyTable* t = c->keys.get();
    const bool tiered = tier_live(t);
    const auto kernel = tiered ? by_rowlen(c, key_init_kernel<true, true>, key_init_kernel<true, false>) : key_init_kernel<false, false>;
    HostTier* h = tiered ? t->tier.get() : nullptr;
    if (launch(c, {warp_grid(c, (size_t)max_new), 256, 0, c->stream}, kernel, view(t), h ? view(h) : KeyView{}, device_rows(c),
               h ? h->a : RowArrays{}, c->rowlen, h ? h->rel.get() : nullptr, initial_s1(c->cfg), t->seed, t->scale)) return 1;
    return 0;
}

// the key table's flags and, on a tiered context, the tier's, with one synchronisation; admission: also the counters of
// an insert-upload
static int read_flags(lctr_ctx* c, bool admission = false) {
    KeyTable* t = c->keys.get();
    LCTR_CUDA(cudaMemcpyAsync(t->ix.h_flags, t->ix.flags, 3 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    if (t->tier)
        LCTR_CUDA(cudaMemcpyAsync(t->tier->ix.h_flags, t->tier->ix.flags, 3 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    if (admission)
        LCTR_CUDA(cudaMemcpyAsync(t->adm->h_cnt, t->adm->cnt, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

static uint64_t rows_in_use(lctr_ctx* c, int* rc) {
    unsigned long long n = 0;
    *rc = cudaMemcpyAsync(&n, c->keys->count, sizeof(n), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
          cudaStreamSynchronize(c->stream) != cudaSuccess;
    if (*rc) set_error("key table: cannot read the row count");
    return std::min<uint64_t>(n, c->keys->cap);
}

int check_keys_reserved(const uint64_t* keys, int64_t n, const char* who) {
    for (int64_t i = 0; i < n; i++)
        LCTR_CHECK(keys[i] != kEmptyKey, "%s: key %llu at entry %lld is reserved (the empty marker of the key table)", who,
                   (unsigned long long)keys[i], (long long)i);
    return 0;
}

int keys_alloc(lctr_ctx* c) {
    c->keys.reset(new KeyTable());
    KeyTable* t = c->keys.get();
    // several GPUs: this rank's shard holds the global rows l * world + rank below feature_cnt (dist.cu: placement)
    t->cap = owned_rows(c->F - 1, c->cfg.world, c->cfg.rank);
    t->scale = (float)(1.0 / sqrt((double)c->cfg.factor_cnt));
    if (t->ix.alloc(t->cap, c->stream) || t->row_key.alloc(t->cap) || t->count.alloc(1)) return 1;
    LCTR_CUDA(cudaMemsetAsync(t->count, 0, sizeof(unsigned long long), c->stream));
    if (c->cfg.key_evict) {
        if (t->last_seen.alloc(t->cap)) return 1;
        LCTR_CUDA(cudaMemsetAsync(t->last_seen, 0, t->cap * sizeof(unsigned long long), c->stream));
    }
    if (c->cfg.key_host_rows) {
        t->tier.reset(new HostTier());
        HostTier* h = t->tier.get();
        h->cap = c->cfg.key_host_rows;
        if (h->ix.alloc(h->cap, c->stream)) return 1;
        // rows in pinned host memory mapped into the device address space: kernels read and write them over PCIe
        const size_t R = h->cap, nv = R * c->rowlen;
        const size_t np[6] = {R, nv, R, nv, c->s2W ? R : 0, c->s2W ? nv : 0};
        bool ok = !h->row_key.alloc(R) && !h->last_seen.alloc(R);
        for (int i = 0; i < 6 && ok; i++) ok = !h->p[i].alloc(np[i]);
        LCTR_CHECK(ok, "lctr_create: cannot allocate %llu rows of pinned host memory (cfg.key_host_rows)",
                   (unsigned long long)h->cap);
        memset(h->row_key, 0, R * sizeof(unsigned long long));
        memset(h->last_seen, 0, R * sizeof(unsigned long long));
        for (int i = 0; i < 6; i++)
            if (np[i]) memset(h->p[i], 0, np[i] * sizeof(float));
        h->a = RowArrays{h->p[0], h->p[1], h->p[2], h->p[3], h->p[4], h->p[5], h->row_key, h->last_seen};
    }
    return 0;
}

bool keys_tracked(const lctr_ctx* c) { return c->keys && c->keys->last_seen; }

static int tier_rebuild(lctr_ctx* c);

bool keys_tier(const lctr_ctx* c, TierRows* out) {
    if (!c->keys || !c->keys->tier) return false;
    const HostTier* h = c->keys->tier.get();
    *out = TierRows{h->a.row_key, h->a.last_seen, {h->a.W, h->a.V, h->a.s1W, h->a.s1V, h->a.s2W, h->a.s2V}, h->n, h->cap};
    return true;
}

int keys_tier_restore(lctr_ctx* c, uint64_t n) {
    HostTier* h = c->keys->tier.get();
    LCTR_CHECK(n <= h->cap, "checkpoint: %llu host-tier rows exceed cfg.key_host_rows = %zu", (unsigned long long)n, h->cap);
    h->n = (size_t)n;
    return tier_rebuild(c);
}

KeyView keys_view(lctr_ctx* c) { return view(c->keys.get()); }
size_t keys_capacity(const lctr_ctx* c) { return c->keys->cap; }

size_t keys_bytes(const lctr_ctx* c) {
    const KeyTable* t = c->keys.get();
    if (!t) return 0;
    return t->ix.T * (sizeof(unsigned long long) + sizeof(uint32_t)) + t->cap * sizeof(unsigned long long) +
           (t->last_seen ? t->cap * sizeof(unsigned long long) : 0) +
           (t->tier ? t->tier->ix.T * (sizeof(unsigned long long) + sizeof(uint32_t)) : 0) +
           (t->adm ? ((size_t)kSketchDepth << t->adm->lw) * sizeof(uint32_t) : 0);
}

// the tier index emptied and rows [0, n) re-inserted with row = index
static int tier_rebuild(lctr_ctx* c) {
    HostTier* h = c->keys->tier.get();
    if (h->ix.rebuild(c, view(h), h->a.row_key, h->n, "host tier: index full while re-inserting")) return 1;
    h->used = h->n;
    return 0;
}

// survivors at or above n_live into the holes below it, for the rows of one table (wscan, holes: evict_move_kernel)
static int launch_move(lctr_ctx* c, const RowArrays& a, size_t n_live, size_t n, const uint32_t* wscan, const uint32_t* holes) {
    if (launch(c, {warp_grid(c, n - n_live), 256, 0, c->stream}, by_rowlen(c, evict_move_kernel<true>, evict_move_kernel<false>),
               a, c->rowlen, n_live, n, wscan, holes)) return 1;
    return 0;
}

// ascending order of distinct values below 2^32: LSD radix sort, three passes of 11 bits
static void radix_sort_u32(std::vector<uint32_t>& v) {
    std::vector<uint32_t> tmp(v.size());
    for (int shift = 0; shift < 32; shift += 11) {
        size_t cnt[2049] = {0};
        for (uint32_t x : v) cnt[((x >> shift) & 2047) + 1]++;
        for (int b = 0; b < 2048; b++) cnt[b + 1] += cnt[b];
        for (uint32_t x : v) tmp[cnt[(x >> shift) & 2047]++] = x;
        v.swap(tmp);
    }
}

// after an upload that restored rows (tier flags read back): the m released rows leave the tier, and the survivors of the
// window [n_live, n) fill the holes below n_live by eviction's rule (the j-th survivor, ascending, into the j-th hole,
// ascending).  Planned on the host from the released list: O(m) copies and work (the sort is a radix sort), then one
// move and one reindex launch over the window; nothing reads the rest of the tier.
static int tier_compact(lctr_ctx* c) {
    HostTier* h = c->keys->tier.get();
    if (!h || !h->ix.h_flags[0]) return 0;
    const size_t m = h->ix.h_flags[0], n = h->n, n_live = n - m;
    std::vector<uint32_t> rel(m), holes;
    LCTR_CUDA(cudaMemcpyAsync(rel.data(), h->rel, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    std::vector<uint32_t> wscan(m + 1, 0);  // first as flags of the window, then its exclusive scan
    for (uint32_t r : rel) {
        if (r >= n_live) wscan[r - n_live] = 1;
        else holes.push_back(r);
    }
    radix_sort_u32(holes);
    uint32_t e = 0;
    for (size_t i = 0; i <= m; i++) {
        const uint32_t f = wscan[i];
        wscan[i] = e;
        e += f;
    }
    LCTR_CUDA(cudaMemcpyAsync(h->wscan, wscan.data(), (m + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    if (!holes.empty())
        LCTR_CUDA(cudaMemcpyAsync(h->holes, holes.data(), holes.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    if (launch_move(c, h->a, n_live, n, h->wscan, h->holes)) return 1;
    if (launch(c, {tile_grid((int64_t)m), 256, 0, c->stream}, tier_reindex_kernel, view(h), n_live, n, h->wscan, h->holes))
        return 1;
    LCTR_CUDA(cudaMemsetAsync(h->ix.flags, 0, 3 * sizeof(unsigned int), c->stream));
    h->ix.h_flags[0] = 0;
    h->n = n_live;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the host vectors above are the copies' sources
    return 0;
}

// keys of one upload (host) -> rows in fid (device, n entries): the keys copied into the scratch, then translated there.
// keys_translate_scratch: the translation of the n keys a caller has put into the scratch (keys_scratch); insert: create and initialise rows for new keys first.  Tiered:
// new keys the tier holds are restored from it; insert = 0 gives rows to the keys the tier holds, and to no other.
// Admission on, insert = 1: count + admit replace the insert, entries of keys not admitted get the drop marker, and the
// dropped count is left for keys_admission_compact.
int keys_translate(lctr_ctx* c, const uint64_t* h_keys, int64_t n, bool insert, uint32_t* fid) {
    uint64_t* d_keys = nullptr;
    if (n > 0) {
        if (keys_scratch(c, (size_t)n, &d_keys)) return 1;
        LCTR_CUDA(cudaMemcpyAsync(d_keys, h_keys, (size_t)n * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream));
    }
    return keys_translate_scratch(c, n, insert, fid);
}

int keys_scratch(lctr_ctx* c, size_t n, uint64_t** d_keys) {
    if (scratch_reserve(c, n)) return 1;
    *d_keys = reinterpret_cast<uint64_t*>(c->keys->d_keys.get());
    return 0;
}

int keys_translate_scratch(lctr_ctx* c, int64_t n, bool insert, uint32_t* fid) {
    KeyTable* t = c->keys.get();
    Admission* adm = insert ? t->adm.get() : nullptr;
    if (insert) t->clock++;  // the clock counts insert-uploads, empty ones included
    if (t->adm) t->adm->pending = 0;
    if (adm) adm->dropped = adm->admitted = 0;
    if (n == 0) return 0;
    LCTR_CUDA(cudaMemsetAsync(t->ix.flags, 0, 3 * sizeof(unsigned int), c->stream));
    if (adm) LCTR_CUDA(cudaMemsetAsync(adm->cnt, 0, 2 * sizeof(unsigned long long), c->stream));
    const bool restoring = tier_live(t);
    {
        ProfScope prof(c, PROF_KEYS);
        if (insert || restoring) {
            if (adm) {
                const KeyView hv = restoring ? view(t->tier.get()) : KeyView{};
                if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_count_kernel, t->d_keys, n, view(t), hv, restoring,
                           adm->sketch, adm->lw)) return 1;
                if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_admit_kernel, t->d_keys, n, view(t), hv, restoring,
                           adm->sketch, adm->lw, adm->min_count, adm->cnt + 1)) return 1;
            } else if (insert) {
                if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_insert_kernel, t->d_keys, n, view(t))) return 1;
            } else {
                if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_lookup_restore_kernel, t->d_keys, n, view(t), view(t->tier.get())))
                    return 1;
            }
            if (init_new_rows(c, std::min<int64_t>(n, (int64_t)t->cap))) return 1;
            if (!insert) {
                if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_tier_refused_kernel, t->d_keys, n, view(t), view(t->tier.get())))
                    return 1;
            }
        }
        if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_find_kernel<0>, t->d_keys, n, view(t), fid, nullptr, insert ? 1 : 0,
                   insert ? t->last_seen.get() : nullptr, t->clock, adm ? adm->cnt.get() : nullptr)) return 1;
    }
    if (read_flags(c, adm != nullptr)) return 1;
    if (adm) {
        adm->dropped = adm->pending = adm->h_cnt[0];
        adm->admitted = adm->h_cnt[1];
    }
    if (restoring && tier_compact(c)) return 1;  // before any failure below: restored rows have left the tier either way
    LCTR_CHECK(!t->ix.h_flags[1], "key table: no free slot on a probe path (%zu slots for capacity %zu)", t->ix.T, t->cap);
    LCTR_CHECK(!t->ix.h_flags[0], "key table: capacity of %zu rows (cfg.feature_cnt) exhausted; the batch's new keys do not fit",
               t->cap);
    return 0;
}

// after keys_translate dropped entries of the slot's batch (row_ptr, fid, field, val on the device): the kept entries in
// order, the new row_ptr, *nnz = the kept count.  Nothing runs when no entry was dropped.
int keys_admission_compact(lctr_ctx* c, Slot& s, cudaStream_t st, int64_t rows, int64_t* nnz) {
    Admission* a = c->keys ? c->keys->adm.get() : nullptr;
    if (!a || !a->pending) return 0;
    const size_t n = (size_t)*nnz, kept = n - a->pending;
    a->pending = 0;
    if (n > a->cap) {
        LCTR_CUDA(cudaStreamSynchronize(st));
        if (admission_scratch(a, std::max(n, a->cap + a->cap / 2))) return 1;
    }
    const uint16_t* field = s.has_field ? s.field.get() : nullptr;
    const float* val = s.has_val ? s.val.get() : nullptr;
    {
        ProfScope prof(c, PROF_KEYS);
        const size_t ntiles = n / kEvTile + 1;  // tiles cover [0, n]: D(n) is read for row_ptr[rows] = n
        if (launch(c, {(unsigned)ntiles, kEvTile, 0, st}, evict_count_kernel<DropFlag>, DropFlag{s.fid}, n, a->tiles)) return 1;
        if (launch(c, {1, 1024, 0, st}, evict_scan_tiles_kernel, a->tiles, ntiles, a->cnt + 2)) return 1;
        if (launch(c, {(unsigned)ntiles, kEvTile, 0, st}, evict_index_kernel<DropFlag>, DropFlag{s.fid}, n, a->tiles, a->scan, nullptr))
            return 1;
        if (launch(c, {stride_grid(c, std::max(n, (size_t)rows + 1)), 256, 0, st}, admit_compact_kernel, s.fid, field, val, n,
                   a->scan, s.row_ptr, (size_t)rows, a->fid, field ? a->field.get() : nullptr, val ? a->val.get() : nullptr)) return 1;
    }
    if (kept) {
        LCTR_CUDA(cudaMemcpyAsync(s.fid, a->fid, kept * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
        if (field) LCTR_CUDA(cudaMemcpyAsync(s.field, a->field, kept * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
        if (val) LCTR_CUDA(cudaMemcpyAsync(s.val, a->val, kept * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    *nnz = (int64_t)kept;
    return 0;
}

static int lookup_dev(lctr_ctx* c, const uint64_t* keys, int64_t n) {
    KeyTable* t = c->keys.get();
    if (scratch_reserve(c, (size_t)n)) return 1;
    LCTR_CUDA(cudaMemcpyAsync(t->d_keys, keys, (size_t)n * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream));
    if (launch(c, {tile_grid(n), 256, 0, c->stream}, key_find_kernel<1>, t->d_keys, n, view(t), nullptr, t->d_rows, 0, nullptr, 0,
               nullptr)) return 1;
    return 0;
}

// rebuild from a row -> key array (checkpoint restore): key i gets row i, parameters are left as they are
int keys_restore(lctr_ctx* c, const uint64_t* row_key, uint64_t n) {
    KeyTable* t = c->keys.get();
    LCTR_CHECK(n <= t->cap, "checkpoint: %llu keyed rows exceed the capacity %zu", (unsigned long long)n, t->cap);
    const unsigned long long cnt = n;
    LCTR_CUDA(cudaMemcpyAsync(t->count, &cnt, sizeof(cnt), cudaMemcpyHostToDevice, c->stream));
    if (n) LCTR_CUDA(cudaMemcpyAsync(t->row_key, row_key, n * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream));
    return t->ix.rebuild(c, view(t), t->row_key, (size_t)n, "checkpoint: key table full while restoring");
}

int keys_download(lctr_ctx* c, std::vector<uint64_t>& out) {
    int rc = 0;
    const uint64_t n = rows_in_use(c, &rc);
    if (rc) return 1;
    out.resize(n);
    if (n) LCTR_CUDA(cudaMemcpyAsync(out.data(), c->keys->row_key, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int keys_download_stamps(lctr_ctx* c, uint64_t n, std::vector<uint64_t>& stamps, uint64_t* clock) {
    KeyTable* t = c->keys.get();
    stamps.resize(n);
    *clock = t->clock;
    if (n) LCTR_CUDA(cudaMemcpyAsync(stamps.data(), t->last_seen, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int keys_restore_stamps(lctr_ctx* c, const uint64_t* stamps, uint64_t n, uint64_t clock) {
    KeyTable* t = c->keys.get();
    LCTR_CHECK(n <= t->cap, "checkpoint: %llu stamps exceed the capacity %zu", (unsigned long long)n, t->cap);
    LCTR_CUDA(cudaMemsetAsync(t->last_seen, 0, t->cap * sizeof(uint64_t), c->stream));
    if (n) LCTR_CUDA(cudaMemcpyAsync(t->last_seen, stamps, n * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    t->clock = clock;
    return 0;
}

static int read_res(lctr_ctx* c, int n) {
    KeyTable* t = c->keys.get();
    LCTR_CUDA(cudaMemcpyAsync(t->h_res, t->ev_res, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

// the age of rank `rank` (0-based, ascending) among the rows of age <= max_idle, of which the largest is max_age
static int radix_select_age(lctr_ctx* c, const unsigned long long* last_seen, size_t n, unsigned long long max_idle,
                            unsigned long long max_age, unsigned long long rank, unsigned long long* out) {
    KeyTable* t = c->keys.get();
    const int bits = std::max(1, 64 - __builtin_clzll(max_age | 1ull));
    const unsigned grid = stride_grid(c, n);
    unsigned long long prefix = 0;
    int pshift = 64, shift = bits;  // bits above `bits` are zero for every survivor: no prefix condition on the first pass
    while (shift > 0) {
        const int width = std::min(16, shift);
        shift -= width;
        LCTR_CUDA(cudaMemsetAsync(t->ev_hist, 0, ((size_t)1 << width) * sizeof(unsigned int), c->stream));
        if (launch(c, {grid, 256, 0, c->stream}, evict_hist_kernel, last_seen, n, t->clock, max_idle, shift, width, pshift,
                   prefix, t->ev_hist)) return 1;
        if (launch(c, {1, 1024, 0, c->stream}, evict_pick_kernel, t->ev_hist, 1 << width, rank, t->ev_res)) return 1;
        if (read_res(c, 2)) return 1;
        prefix = (prefix << width) | t->h_res[0];
        rank -= t->h_res[1];
        pshift = shift;
    }
    *out = prefix;
    return 0;
}

// one table as the eviction sees it: the device table or the host tier (rows [0, n), scratch sized for its capacity)
struct EvTable {
    RowArrays a;
    size_t n;
    uint32_t *scan, *rows, *tiles;
};

// survey, select, count and scan of the stamp rule against the upload clock: *m rows of the table leave by rule *l
static int evict_plan(lctr_ctx* c, const EvTable& tb, uint64_t max_idle, uint64_t max_rows, EvictRule* e, size_t* m) {
    KeyTable* t = c->keys.get();
    const size_t n = tb.n;
    // 1 + 2: the rule
    LCTR_CUDA(cudaMemsetAsync(t->ev_res, 0, 2 * sizeof(unsigned long long), c->stream));
    if (launch(c, {stride_grid(c, n), 256, 0, c->stream}, evict_survey_kernel, tb.a.last_seen, n, t->clock, max_idle, t->ev_res))
        return 1;
    if (read_res(c, 2)) return 1;
    const unsigned long long survivors = t->h_res[0], max_age = t->h_res[1];
    *e = EvictRule{t->clock, max_idle, 0ull, 0};
    if (survivors > max_rows) {
        if (radix_select_age(c, tb.a.last_seen, n, max_idle, max_age, max_rows, &e->cut)) return 1;
        e->limit = 1;
    }
    // count and scan
    const size_t ntiles = n / kEvTile + 1;  // tiles cover [0, n]: E(n) is needed too
    if (launch(c, {(unsigned)ntiles, kEvTile, 0, c->stream}, evict_count_kernel<EvictFlag>, EvictFlag{tb.a.last_seen, *e}, n, tb.tiles))
        return 1;
    if (launch(c, {1, 1024, 0, c->stream}, evict_scan_tiles_kernel, tb.tiles, ntiles, t->ev_res)) return 1;
    if (read_res(c, 1)) return 1;
    *m = (size_t)t->h_res[0];
    return 0;
}

// E(r) and the list of the m rows that leave, then their key, W and V into the caller's buffers (each may be null)
static int evict_index_export(lctr_ctx* c, const EvTable& tb, const EvictRule& e, size_t m, uint64_t* keys_out, float* W_out,
                              float* V_out) {
    if (launch(c, {(unsigned)(tb.n / kEvTile + 1), kEvTile, 0, c->stream}, evict_index_kernel<EvictFlag>, EvictFlag{tb.a.last_seen, e}, tb.n,
               tb.tiles, tb.scan, tb.rows)) return 1;
    if (!(keys_out || W_out || V_out)) return 0;
    Buf<unsigned long long> dK;
    Buf<float> dW, dV;
    if (dK.alloc(keys_out ? m : 0) || dW.alloc(W_out ? m : 0) || dV.alloc(V_out ? m * c->rowlen : 0)) return 1;
    auto copy_out = [&]() -> int {
        if (launch(c, {warp_grid(c, m), 256, 0, c->stream}, evict_export_kernel, tb.rows, m, tb.a.row_key, tb.a.W, tb.a.V,
                   c->rowlen, dK, dW, dV))
            return 1;
        if (dK) LCTR_CUDA(cudaMemcpyAsync(keys_out, dK, m * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
        if (dW) LCTR_CUDA(cudaMemcpyAsync(W_out, dW, m * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (dV) LCTR_CUDA(cudaMemcpyAsync(V_out, dV, m * c->rowlen * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        return 0;
    };
    const int rc = copy_out();
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the queued work reads the staging, which goes on return
    return rc;
}

bool keys_admission(const lctr_ctx* c, uint32_t* min_count, uint32_t* log2_width) {
    const Admission* a = c->keys ? c->keys->adm.get() : nullptr;
    *min_count = a ? a->min_count : 0;
    *log2_width = a ? a->lw : 0;
    return a != nullptr;
}

int keys_admission_download(lctr_ctx* c, std::vector<uint32_t>& sketch) {
    const Admission* a = c->keys->adm.get();
    sketch.resize((size_t)kSketchDepth << a->lw);
    LCTR_CUDA(cudaMemcpyAsync(sketch.data(), a->sketch, sketch.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int keys_admission_restore(lctr_ctx* c, const uint32_t* sketch) {
    Admission* a = c->keys->adm.get();
    LCTR_CUDA(cudaMemcpyAsync(a->sketch, sketch, ((size_t)kSketchDepth << a->lw) * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    a->dropped = a->admitted = a->pending = 0;
    return 0;
}

// the m rows of the device table's eviction list appended to the tier at rows [n, n + m), keys claimed in its index
static int tier_spill(lctr_ctx* c, const EvTable& dev, size_t m) {
    HostTier* h = c->keys->tier.get();
    KeyIndex& ix = h->ix;
    LCTR_CUDA(cudaMemsetAsync(ix.flags, 0, 3 * sizeof(unsigned int), c->stream));
    if (launch(c, {warp_grid(c, m), 256, 0, c->stream}, by_rowlen(c, tier_spill_kernel<true>, tier_spill_kernel<false>), dev.rows,
               m, dev.a, h->a, h->n, c->rowlen, view(h))) return 1;
    LCTR_CUDA(cudaMemcpyAsync(ix.h_flags, ix.flags, 3 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    h->n += m;
    h->used += ix.h_flags[2];
    LCTR_CUDA(cudaMemsetAsync(ix.flags, 0, 3 * sizeof(unsigned int), c->stream));
    // a full probe path (never expected below T / 2 used slots) or more than T / 2 slots in use: a fresh index
    if (ix.h_flags[1] || 2 * h->used > ix.T) return tier_rebuild(c);
    return 0;
}

}  // namespace lctr

using namespace lctr;

extern "C" {

int lctr_lookup_keys(lctr_ctx* c, int64_t n, const uint64_t* keys, int64_t* rows) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_lookup_keys: the context was not created with key_mode = LCTR_KEYS_HASHED");
    LCTR_CHECK(n >= 0 && (n == 0 || (keys && rows)), "lctr_lookup_keys: null argument");
    if (n == 0) return 0;
    if (lookup_dev(c, keys, n)) return 1;
    LCTR_CUDA(cudaMemcpyAsync(rows, c->keys->d_rows, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (c->cfg.world > 1)  // local row l of this rank is global row l * world + rank; keys it does not hold stay -1
        for (int64_t i = 0; i < n; i++)
            if (rows[i] >= 0) rows[i] = rows[i] * c->cfg.world + c->cfg.rank;
    return 0;
}

int lctr_download_keys(lctr_ctx* c, uint64_t* keys, uint64_t cap, uint64_t* n_rows) {
    LCTR_CHECK(c && n_rows, "null argument");
    LCTR_CHECK(c->keys, "lctr_download_keys: the context was not created with key_mode = LCTR_KEYS_HASHED");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    int rc = 0;
    const uint64_t n = rows_in_use(c, &rc);
    if (rc) return 1;
    *n_rows = n;
    if (!keys) return 0;
    LCTR_CHECK(cap >= n, "lctr_download_keys: room for %llu keys, the table has %llu rows", (unsigned long long)cap,
               (unsigned long long)n);
    if (n) LCTR_CUDA(cudaMemcpyAsync(keys, c->keys->row_key, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

static int upload_keyed_params_local(lctr_ctx* c, int64_t n, const uint64_t* keys, const float* W, const float* V);

int lctr_upload_keyed_params(lctr_ctx* c, int64_t n, const uint64_t* keys, const float* W, const float* V) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_upload_keyed_params: the context was not created with key_mode = LCTR_KEYS_HASHED");
    LCTR_CHECK(n >= 0 && (n == 0 || keys), "lctr_upload_keyed_params: null argument");
    if (n == 0) return 0;
    if (check_keys_reserved(keys, n, "lctr_upload_keyed_params")) return 1;
    {
        std::vector<uint64_t> sorted(keys, keys + n);
        std::sort(sorted.begin(), sorted.end());
        const auto d = std::adjacent_find(sorted.begin(), sorted.end());
        LCTR_CHECK(d == sorted.end(), "lctr_upload_keyed_params: key %llu appears more than once", (unsigned long long)*d);
    }
    if (c->cfg.world <= 1) return upload_keyed_params_local(c, n, keys, W, V);
    // several GPUs: only the keys this rank owns, in array order, so the same call on every rank seeds the sharded table
    int shift = 0;
    while ((1 << shift) < c->cfg.world) shift++;
    std::vector<uint64_t> mk;
    std::vector<float> mw, mv;
    for (int64_t i = 0; i < n; i++) {
        if (owner_of_key(keys[i], shift) != (unsigned)c->cfg.rank) continue;
        mk.push_back(keys[i]);
        if (W) mw.push_back(W[i]);
        if (V) mv.insert(mv.end(), V + (size_t)i * c->rowlen, V + (size_t)(i + 1) * c->rowlen);
    }
    if (mk.empty()) return 0;
    return upload_keyed_params_local(c, (int64_t)mk.size(), mk.data(), W ? mw.data() : nullptr, V ? mv.data() : nullptr);
}

// the keys of one rank's table (all of them on one GPU), validated by the caller
static int upload_keyed_params_local(lctr_ctx* c, int64_t n, const uint64_t* keys, const float* W, const float* V) {
    KeyTable* t = c->keys.get();
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (lookup_dev(c, keys, n)) return 1;
    std::vector<int64_t> rows((size_t)n);
    LCTR_CUDA(cudaMemcpyAsync(rows.data(), t->d_rows, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    int rc = 0;
    const uint64_t used = rows_in_use(c, &rc);
    if (rc) return 1;
    // absent keys: consecutive rows in array order
    std::vector<uint64_t> new_keys;
    std::vector<int64_t> new_rows;
    for (int64_t i = 0; i < n; i++)
        if (rows[(size_t)i] < 0) {
            rows[(size_t)i] = (int64_t)(used + new_keys.size());
            new_keys.push_back(keys[i]);
            new_rows.push_back(rows[(size_t)i]);
        }
    LCTR_CHECK(used + new_keys.size() <= t->cap, "lctr_upload_keyed_params: %zu new keys do not fit the capacity of %zu rows (%llu in use)",
               new_keys.size(), t->cap, (unsigned long long)used);
    const int64_t m = (int64_t)new_keys.size();
    if (m) {
        LCTR_CUDA(cudaMemsetAsync(t->ix.flags, 0, 3 * sizeof(unsigned int), c->stream));
        LCTR_CUDA(cudaMemcpyAsync(t->d_keys, new_keys.data(), (size_t)m * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
        LCTR_CUDA(cudaMemcpyAsync(t->d_rows, new_rows.data(), (size_t)m * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
        if (launch(c, {tile_grid(m), 256, 0, c->stream}, key_insert_fixed_kernel, t->d_keys, t->d_rows, m, view(t), 1)) return 1;
        const bool restoring = tier_live(t);  // tier keys bring their optimizer state back
        if (init_new_rows(c, m)) return 1;
        const unsigned long long cnt = used + (uint64_t)m;
        LCTR_CUDA(cudaMemcpyAsync(t->count, &cnt, sizeof(cnt), cudaMemcpyHostToDevice, c->stream));
        if (read_flags(c)) return 1;
        if (restoring && tier_compact(c)) return 1;
        LCTR_CHECK(!t->ix.h_flags[1], "lctr_upload_keyed_params: key table full");
    }
    if (t->last_seen || W || V)
        LCTR_CUDA(cudaMemcpyAsync(t->d_rows, rows.data(), (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (t->last_seen) {  // every named row counts as met at the current clock
        if (launch(c, {stride_grid(c, (size_t)n), 256, 0, c->stream}, key_stamp_rows_kernel, t->d_rows, n, t->last_seen, t->clock))
            return 1;
    }
    if (W || V) {
        Buf<float> dW, dV;
        if (dW.alloc(W ? (size_t)n : 0) || dV.alloc(V ? (size_t)n * c->rowlen : 0)) return 1;
        auto scatter = [&]() -> int {
            if (W) LCTR_CUDA(cudaMemcpyAsync(dW, W, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            if (V) LCTR_CUDA(cudaMemcpyAsync(dV, V, (size_t)n * c->rowlen * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            return launch(c, {warp_grid(c, (size_t)n), 256, 0, c->stream}, key_scatter_params_kernel, t->d_rows, n, dW, dV, c->W,
                          c->V, c->rowlen);
        };
        const int rc = scatter();
        LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the queued work reads the staging, which goes with this block
        if (rc) return 1;
    }
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_set_key_init(lctr_ctx* c, uint64_t seed, float scale) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_set_key_init: the context was not created with key_mode = LCTR_KEYS_HASHED");
    c->keys->seed = seed;
    c->keys->scale = scale;
    return 0;
}

int lctr_set_key_admission(lctr_ctx* c, uint32_t min_count, uint32_t log2_width) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_set_key_admission: the context was not created with key_mode = LCTR_KEYS_HASHED (a dense context "
                        "has no keys to admit)");
    LCTR_CHECK(c->cfg.world <= 1, "lctr_set_key_admission: world = %d: admission is single-GPU (the requester's slot map is "
                                  "built before the owners translate, so it cannot drop entries)", c->cfg.world);
    LCTR_CHECK(c->cfg.model != LCTR_MODEL_WND, "lctr_set_key_admission: Wide&Deep reads the first id of each field, and dropping "
                                               "entries would change which id that is");
    KeyTable* t = c->keys.get();
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    if (min_count <= 1) {  // off: the context behaves and launches as one that never set it
        t->adm.reset();
        return 0;
    }
    LCTR_CHECK(log2_width >= 10 && log2_width <= 28, "lctr_set_key_admission: log2_width = %u outside [10, 28]", log2_width);
    if (!t->adm || t->adm->lw != log2_width) {
        t->adm.reset();
        auto a = std::make_unique<Admission>();
        a->lw = log2_width;
        if (a->sketch.alloc((size_t)kSketchDepth << log2_width) || a->cnt.alloc(3) || a->h_cnt.alloc(2)) {
            set_error("lctr_set_key_admission: cannot allocate a sketch of %llu bytes (admission is off)",
                      (unsigned long long)(((size_t)kSketchDepth << log2_width) * sizeof(uint32_t)));
            return 1;
        }
        t->adm = std::move(a);
    }
    Admission* a = t->adm.get();
    a->min_count = min_count;
    a->dropped = a->admitted = a->pending = 0;
    LCTR_CUDA(cudaMemsetAsync(a->sketch, 0, ((size_t)kSketchDepth << a->lw) * sizeof(uint32_t), c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_decay_key_admission(lctr_ctx* c, uint32_t shift) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys && c->keys->adm, "lctr_decay_key_admission: admission is off (lctr_set_key_admission with min_count > 1 "
                                        "turns it on)");
    LCTR_CHECK(shift >= 1 && shift <= 32, "lctr_decay_key_admission: shift = %u outside [1, 32]", shift);
    const Admission* a = c->keys->adm.get();
    const size_t n4 = ((size_t)kSketchDepth << a->lw) / 4;
    if (launch(c, {stride_grid(c, n4), 256, 0, c->stream}, sketch_decay_kernel, reinterpret_cast<uint4*>(a->sketch.get()), n4, shift))
        return 1;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
}

int lctr_key_admission_stats(lctr_ctx* c, uint64_t* dropped_entries, uint64_t* admitted_keys) {
    LCTR_CHECK(c, "null ctx");
    LCTR_CHECK(c->keys, "lctr_key_admission_stats: the context was not created with key_mode = LCTR_KEYS_HASHED");
    const Admission* a = c->keys->adm.get();
    if (dropped_entries) *dropped_entries = a ? a->dropped : 0;
    if (admitted_keys) *admitted_keys = a ? a->admitted : 0;
    return 0;
}

int lctr_evict_keys(lctr_ctx* c, uint64_t max_idle, uint64_t max_rows, uint64_t* keys_out, float* W_out, float* V_out,
                    uint64_t cap_out, uint64_t* n_evicted) {
    LCTR_CHECK(c && n_evicted, "null argument");
    LCTR_CHECK(c->keys, "lctr_evict_keys: the context was not created with key_mode = LCTR_KEYS_HASHED");
    LCTR_CHECK(c->keys->last_seen, "lctr_evict_keys: the context was not created with key_evict = 1 (rows record no last use)");
    KeyTable* t = c->keys.get();
    *n_evicted = 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    int rc = 0;
    const size_t n = rows_in_use(c, &rc);
    if (rc) return 1;
    if (n == 0) return 0;
    if (!t->h_res && evict_scratch(t, t->cap)) return 1;
    const EvTable tb{device_rows(c), n, t->ev_scan, t->ev_rows, t->ev_tiles};
    EvictRule e;
    size_t m = 0;
    if (evict_plan(c, tb, max_idle, max_rows, &e, &m)) return 1;
    if (m == 0) return 0;  // nothing leaves: the table, its rows and the slots stay as they are
    const bool exporting = keys_out || W_out || V_out;
    LCTR_CHECK(!exporting || cap_out >= m, "lctr_evict_keys: room for %llu evicted rows, %zu would leave (nothing was changed)",
               (unsigned long long)cap_out, m);
    HostTier* h = t->tier.get();
    LCTR_CHECK(!h || h->n + m <= h->cap, "lctr_evict_keys: %zu rows would leave for the host tier, which holds %zu rows "
               "(cfg.key_host_rows) with %zu free (nothing was changed)", m, h ? h->cap : 0, h ? h->cap - h->n : 0);
    const size_t n_live = n - m;
    if (evict_index_export(c, tb, e, m, keys_out, W_out, V_out)) return 1;  // gathered before anything moves
    if (h && tier_spill(c, tb, m)) return 1;

    // move, reset, rebuild
    if (launch_move(c, tb.a, n_live, n, t->ev_scan + n_live, t->ev_rows)) return 1;
    if (launch(c, {warp_grid(c, m), 256, 0, c->stream}, by_rowlen(c, evict_reset_kernel<true>, evict_reset_kernel<false>), tb.a,
               c->rowlen, n_live, n, initial_s1(c->cfg))) return 1;
    const unsigned long long cnt = n_live;
    LCTR_CUDA(cudaMemcpyAsync(t->count, &cnt, sizeof(cnt), cudaMemcpyHostToDevice, c->stream));
    if (t->ix.rebuild(c, view(t), t->row_key, n_live, "lctr_evict_keys: key table full while re-inserting")) return 1;
    for (int s = 0; s < kNumSlots; s++)  // their row ids belong to the old numbering
        if (c->slots[s].key_state != SLOT_KEYS_INVALID) c->slots[s].key_state = SLOT_KEYS_STALE;
    *n_evicted = m;
    return 0;
}

int lctr_evict_host_tier(lctr_ctx* c, uint64_t max_idle, uint64_t max_rows, uint64_t* keys_out, float* W_out, float* V_out,
                         uint64_t cap_out, uint64_t* n_evicted) {
    LCTR_CHECK(c && n_evicted, "null argument");
    LCTR_CHECK(c->keys && c->keys->tier, "lctr_evict_host_tier: the context was not created with a host tier (cfg.key_host_rows)");
    HostTier* h = c->keys->tier.get();
    *n_evicted = 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    const size_t n = h->n;
    if (n == 0) return 0;
    if (!c->keys->h_res && evict_scratch(c->keys.get(), c->keys->cap)) return 1;
    // scratch of the tier's size for this call only: a tier eviction reads every tier row anyway
    Buf<uint32_t> scan, rows, tiles;
    if (scan.alloc(n + 1) || rows.alloc(n) || tiles.alloc(n / kEvTile + 1)) return 1;
    auto evict = [&]() -> int {
        const EvTable tb{h->a, n, scan, rows, tiles};
        EvictRule e;
        size_t m = 0;
        if (evict_plan(c, tb, max_idle, max_rows, &e, &m)) return 1;
        if (m == 0) return 0;
        LCTR_CHECK(!(keys_out || W_out || V_out) || cap_out >= m,
                   "lctr_evict_host_tier: room for %llu evicted rows, %zu would leave (nothing was changed)", (unsigned long long)cap_out, m);
        if (evict_index_export(c, tb, e, m, keys_out, W_out, V_out)) return 1;
        if (launch_move(c, h->a, n - m, n, scan + (n - m), rows)) return 1;
        h->n = n - m;
        if (tier_rebuild(c)) return 1;
        *n_evicted = m;
        return 0;
    };
    const int rc = evict();
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the queued work reads the scratch, which goes on return
    return rc;
}

int lctr_download_host_tier(lctr_ctx* c, uint64_t* keys, float* W, float* V, uint64_t cap, uint64_t* n_rows) {
    LCTR_CHECK(c && n_rows, "null argument");
    LCTR_CHECK(c->keys && c->keys->tier, "lctr_download_host_tier: the context was not created with a host tier (cfg.key_host_rows)");
    LCTR_CUDA(cudaStreamSynchronize(c->stream));  // the tier's rows change only on the ctx stream
    const HostTier* h = c->keys->tier.get();
    *n_rows = h->n;
    if (!keys && !W && !V) return 0;
    LCTR_CHECK(cap >= h->n, "lctr_download_host_tier: room for %llu rows, the tier holds %zu", (unsigned long long)cap, h->n);
    if (keys) memcpy(keys, h->a.row_key, h->n * sizeof(uint64_t));
    if (W) memcpy(W, h->a.W, h->n * sizeof(float));
    if (V) memcpy(V, h->a.V, h->n * c->rowlen * sizeof(float));
    return 0;
}

}  // extern "C"
