// lightctr_b200/csrc/keys.cuh -- device helpers of the keyed mode shared by keys.cu (the key table of a context) and
// dist.cu (the per-batch dedupe of a requester and the owner-side translation of the multi-GPU keyed exchange).
#pragma once
#include "common.cuh"

namespace lctr {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr uint32_t kNoRow = 0xffffffffu;
constexpr int kGroup = 16;  // slots per 128-byte probe group

struct KeyView {
    unsigned long long* key;
    uint32_t* row;
    unsigned long long* row_key;
    unsigned long long* count;
    unsigned int* flags;
    uint32_t* new_rows;
    size_t ngroups, cap;
};

__host__ __device__ __forceinline__ unsigned long long fmix64(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}

// rank that owns a key on `world` = 2^shift ranks: the TOP bits of fmix64(key).  The owner's table picks the home group
// from the low bits of the same hash, so the two choices stay independent.
__host__ __device__ __forceinline__ unsigned owner_of_key(unsigned long long key, int shift) {
    return shift ? (unsigned)(fmix64(key) >> (64 - shift)) : 0u;
}

// Finds the slot of `key` or claims one for it.  Returns the slot, or -1 when the table has no free slot left on the
// probe path.  *claimed: this tile's CAS put the key there (all lanes).  Table words are read with ld.cg: other tiles of
// the same launch insert concurrently, and a stale "empty" is corrected by the CAS that follows it.
__device__ __forceinline__ long long tile_claim(const KeyView& t, unsigned long long key, int sub, unsigned gmask, bool* claimed) {
    const size_t home = (size_t)(fmix64(key) & (t.ngroups - 1));
    *claimed = false;
    for (size_t step = 0; step < t.ngroups; step++) {
        const size_t base = ((home + step) & (t.ngroups - 1)) * kGroup;
        unsigned long long k = __ldcg(t.key + base + sub);
        while (true) {
            const unsigned hit = __ballot_sync(gmask, k == key) & gmask;
            if (hit) return (long long)(base + ((__ffs(hit) - 1) & (kGroup - 1)));
            const unsigned empty = __ballot_sync(gmask, k == kEmptyKey) & gmask;
            if (!empty) break;
            const int leader = __ffs(empty) - 1, lsub = leader & (kGroup - 1);
            unsigned long long old = 0;
            if ((int)(threadIdx.x & 31) == leader) old = atomicCAS(t.key + base + lsub, kEmptyKey, key);
            old = __shfl_sync(gmask, old, leader);
            if (old == kEmptyKey) { *claimed = true; return (long long)(base + lsub); }
            if (old == key) return (long long)(base + lsub);
            if (sub == lsub) k = old;  // lost the slot to another key: look at the group again
        }
    }
    return -1;
}

// read-only probe (no insert may run concurrently): slot of `key` or -1
__device__ __forceinline__ long long tile_find(const KeyView& t, unsigned long long key, int sub, unsigned gmask) {
    if (key == kEmptyKey) return -1;
    const size_t home = (size_t)(fmix64(key) & (t.ngroups - 1));
    for (size_t step = 0; step < t.ngroups; step++) {
        const size_t base = ((home + step) & (t.ngroups - 1)) * kGroup;
        const unsigned long long k = __ldg(t.key + base + sub);
        const unsigned hit = __ballot_sync(gmask, k == key) & gmask;
        if (hit) return (long long)(base + ((__ffs(hit) - 1) & (kGroup - 1)));
        if (__ballot_sync(gmask, k == kEmptyKey) & gmask) return -1;
    }
    return -1;
}

// one key of an insert (a whole 16-lane tile calls it): a tile that finds no match claims the first empty slot of the
// group; the winner takes a row from the counter and records it in the list of new rows, or stores kNoRow and raises the
// capacity flag when the counter has passed the capacity.  flags: [0] capacity exhausted, [1] table full, [2] new rows.
// Returns whether this tile claimed the key's slot (all lanes).
__device__ __forceinline__ bool tile_insert(const KeyView& t, unsigned long long key, int sub, unsigned gmask) {
    bool claimed;
    const long long pos = tile_claim(t, key, sub, gmask, &claimed);
    if (sub != 0) return claimed;
    if (pos < 0) { t.flags[1] = 1u; return false; }
    if (!claimed) return false;
    const unsigned long long r = atomicAdd(t.count, 1ull);
    if (r < t.cap) {
        t.row[pos] = (uint32_t)r;
        t.row_key[r] = key;
        t.new_rows[atomicAdd(&t.flags[2], 1u)] = (uint32_t)r;
    } else {
        t.row[pos] = kNoRow;
        t.flags[0] = 1u;
    }
    return true;
}

// host side of keys.cu used by dist.cu: the context's key table as a view, room for `n` keys (and new rows) in its
// scratch, and the lazy init of the rows the last insert recorded (one launch)
KeyView keys_view(lctr_ctx* c);
int scratch_reserve(lctr_ctx* c, size_t n);
int init_new_rows(lctr_ctx* c, int64_t max_new);
size_t keys_capacity(const lctr_ctx* c);

}  // namespace lctr
