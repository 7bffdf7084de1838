// lightctr_b200/csrc/dist.cu -- multi-GPU sparse exchange over NVLink peer memory (one process per GPU).
//
// Replaces the reference's Parameter-Server round trips: Pull::sync of the batch's unique keys
// (distribut/pull.h:43-68; unique-key build distributed_algo_abst.h:181-195) and Push::sync of the per-key
// gradients (distribut/push.h:36-51) with the owner applying the update (distribut/paramserver.h:181-310).
// Differences we state rather than reproduce (SURVEY.md 8e): synchronous instead of SSP-async, fp32 instead of
// fp16 on the wire, no |g| thresholding of pushes, owner = fid mod R instead of the murmur DHT ring.
//
// Tables are owner-sharded: row f lives on rank f % R at shard-local index f / R.  Every rank maps ONE buffer of every
// peer through CUDA IPC, its arena (flags, key inboxes, parameter cache, gradient inboxes): owners write rows into their
// requesters' caches and requesters push gradient rows into their owners' inboxes, so no rank reads or writes a peer's
// table shard.  Per-rank memory is the shard plus O(keys of a batch): the compute kernels work on a BATCH-COMPACT cache
// (row = slot of the batch's key set, fm_fused.cu's slot map) instead of full-size copies of the tables.
//
//   upload (depends only on the batch; on the upload stream, overlaps the previous step)
//     slot map of my batch (mark / compact / assign) and, per owner o, the list of the shard-local rows o owns, written
//     straight into o's key inbox with posted stores + a generation flag (send_keys_kernel).  From then on a row of the
//     exchange is addressed by p = o * cap_pair + its position in that list, by requester and owner alike: the entries of
//     the batch are re-indexed to p (remap_entries_kernel), so the cache rows of one owner and the gradient rows for one
//     owner are CONTIGUOUS and both transfers are long coalesced streams instead of scattered 64 B packets.
//   step
//     1 serve   OWNER-driven pull: I read the key lists my peers posted and WRITE the rows they asked for into their
//               caches (posted peer stores instead of read round trips), then raise "rows delivered" on each peer
//                                                                                                (serve_pull_kernel)
//     2 compute the single-GPU kernels on the cache; the first one waits (in-kernel) for every owner's flag
//     3 push    owner by owner, my gradient rows [gV | gW] (hot replicas folded) stream into the owner's gradient inbox
//               at the positions of the list it received -- no slot reservation, no atomics on the wire; then "pushes
//               landed" flags                                                                    (push_rows_kernel)
//     4 owner   inbox rows are added into update_g with local REDs (waits for the flags)          (merge_kernel)
//               sparse updater on the shard                                                      (opt.cu)
// Keyed contexts (cfg.key_mode = LCTR_KEYS_HASHED) change the upload only: the batch's keys are deduped into batch-local
// ids, the lists carry the keys, and each owner translates them into its shard's rows before the step (see "keyed upload").
// Launches per step: 6; the barriers between the phases are flags written at the tail of one kernel and polled at the
// head of the next -- no barrier launches, no host involvement.
//
// Pull-only rounds (lctr_predict: serve + forward, no push / merge / updater, no owner-side union build) and the cache
// release.  Invariant: no owner writes into requester r's cache for epoch e+1 until r's kernels of epoch e have stopped
// reading it.  In a training round this follows from the push: owner o serves e+1 only after its merge of e (stream order),
// the merge waited for r's "pushes landed" flag, and r's push runs after r's compute has finished with the cache.  A
// pull-only round has no push, so r ends it with release_cache_kernel, launched behind its forward (ordinary stream order:
// every read of the cache has completed), which raises FLAG_RELEASED = e on every owner.  The next round's serve is
// preceded by a wait for FLAG_RELEASED >= e from every requester -- only when the previous round was pull-only, which
// every rank knows because rounds are collective.  Two training rounds in a row issue exactly the launches and waits they
// did before pull-only rounds existed; a round after a pull-only one issues one extra (one-block) wait launch.
// Empty shares: a rank that uploads 0 rows (or 0 entries) still posts its key lists, empty, with the generation flag, so
// its peers' serve never waits for lists that would not come; it then serves, predicts 0 rows and pushes no gradients.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "keys.cuh"
#include "opt.cuh"

namespace lctr {

constexpr int kMaxWorld = 8;
constexpr int kHotRepD = kHotRep, kHotMaxD = kHotMax;

struct Peer {
    unsigned char* arena;  // the only buffer ranks share (lctr_ipc_export)
};
struct PeerTable { Peer p[kMaxWorld]; };

// byte offsets inside the arena (identical on every rank)
struct ArenaLayout {
    size_t flags;        // u64 [4 + kNumSlots][kMaxWorld]: row 0 rows delivered, 1 pushes landed, 2 keyed statuses, 3 cache
                         // released (pull-only rounds), 4 + s keys of slot s
    size_t key_inbox;    // [kNumSlots][2][world] regions (2: parity of the slot's upload generation -- a list may still be read
                         // by a slower owner's merge when its sender already uploads the slot's next batch):
                         // 64 B header {u32 count, u32 requester status (keyed)} + cap_pair x uint2 {row, requester slot}
                         // (+ keyed contexts: cap_pair x u64 keys at key_keys)
    size_t key_region;   // bytes per region
    size_t key_keys;     // keyed: offset of the key array inside a region
    size_t cacheW;       // world * cap_pair floats (row p)
    size_t cacheV;       // world * cap_pair x rowlen floats
    size_t grad_inbox;   // [world] regions of cap_pair x recw floats
    size_t grad_region;  // bytes per region
    size_t total;
};
enum { FLAG_PULLED = 0, FLAG_PUSHED = 1, FLAG_XLATED = 2, FLAG_RELEASED = 3, FLAG_KEYS = 4 };
// statuses of a keyed upload (code << 8 | rank): raised by every owner on every requester in FLAG_XLATED as seq << 16 | status
enum { XS_OK = 0, XS_REFUSED = 1, XS_INBOX = 2, XS_TIMEOUT = 3, XS_CAPACITY = 4, XS_TABLE_FULL = 5 };
// bound of every wait of the keyed upload: ~4 s at the H100's boost clock (longer at lower clocks)
constexpr long long kXlateWaitCycles = 1ll << 33;

struct DistState {
    int rank = 0, world = 1, shift = 0;
    Buf<unsigned char> arena;
    ArenaLayout A;
    PeerTable peers;
    size_t cap_keys = 0, cap_pair = 0;
    int recw = 0;                     // floats per gradient-inbox record: rowlen + 4 ([gV | gW | pad])
    size_t rows_x = 0;                // world * cap_pair: rows of the exchange index space p
    Buf<unsigned int> send_cnt;       // [kMaxWorld] records appended per owner by the running send_keys
    Buf<unsigned int> seg_cnt;        // [kNumSlots][kMaxWorld]: keys per owner of each slot's batch
    Buf<uint32_t> opos;               // [kNumSlots][cap_keys]: exchange row p of each of my slots
    Buf<uint32_t> hot_p;              // [kNumSlots][rows_x]: replica block of hot exchange rows (fused kernels), else ~0
    Buf<unsigned int> done_ctr;       // [4] last-block counters
    Buf<int> overflow;                // device flag: a key list outgrew cap_pair
    Buf<float> cgV, cgW;              // [rows_x][rowlen], [rows_x]: compact gradient rows of the non-fused kernels
    // owner side of the fused FM / NFM step: the UNION of the key lists the requesters sent for a slot's batch, built once per
    // upload, and for every union row its position in each requester's list (~0: not asked for) -- the updater walks it and
    // sums the gradient inboxes itself (no dense update_g, no touched map, no O(F / R) scan per step)
    Buf<uint32_t> own_uniq;           // [kNumSlots][cap_own] shard-local rows
    Buf<unsigned int> n_own;          // [kNumSlots]
    Buf<uint32_t> own_pos;            // [kNumSlots][world][cap_own]
    Buf<uint32_t> posmap;             // [world][Fl] scratch: list position of a row in requester q's current list (self-validating)
    Buf<uint8_t> own_mark;            // permuted byte map over the shard (128 * own_T)
    size_t cap_own = 0, own_T = 0;
    unsigned long long own_gen[kNumSlots] = {0};
    void* opened[kMaxWorld] = {nullptr};  // peers' arenas mapped by lctr_ipc_import
    bool imported = false;
    unsigned long long epoch = 0;
    unsigned long long released = 0; // epoch of the last round when it was pull-only (its requesters release their caches), else 0
    unsigned long long gen[kNumSlots] = {0};
    size_t bytes = 0;                 // device memory this module allocated
    // keyed contexts (cfg.key_mode = LCTR_KEYS_HASHED): requester-side dedupe of a batch's keys into batch-local ids u,
    // an open-addressing table of bt_T >= 2 * cap_keys slots cleared by the list of the slots it claimed
    bool keyed = false;
    Buf<unsigned long long> bt_key;           // [bt_T] slot keys, kEmptyKey = free
    Buf<uint32_t> bt_row;                     // [bt_T] batch-local id of the slot's key
    Buf<uint32_t> bt_claimed;                 // [bt_T] slots claimed by the running dedupe
    Buf<unsigned long long> bt_cnt;           // keys claimed (the batch's U when <= cap_keys)
    Buf<unsigned int> bt_flags;               // [3] U > cap_keys, table full, (unused)
    Buf<unsigned long long> batch_key;        // [cap_keys] key of batch-local id u
    Buf<unsigned long long> bt_stage;         // the batch's keys, one per entry
    size_t bt_T = 0, bt_stage_cap = 0;
    Buf<unsigned int> xstat;                  // owner side: status of the running translation (wait kernel -> the others)
    Buf<unsigned long long> xres;             // [kMaxWorld] status every owner raised for this rank's upload
    unsigned long long xseq = 0;              // keyed uploads so far (the same on every rank: the upload is collective)
    bool posted = false;                      // this upload's lists (or its refusal) are out
};
void drop(DistState* p) { delete p; }

__device__ __forceinline__ unsigned long long* flag_ptr(unsigned char* arena, const ArenaLayout& A, int row, int col) {
    return reinterpret_cast<unsigned long long*>(arena + A.flags) + (size_t)row * kMaxWorld + col;
}
// System-scope fences are executed by the few threads that poll / raise flags, never by whole CTAs: membar.sys drains the
// issuing SM's outstanding peer traffic, so hundreds of CTAs x 256 threads doing it would serialise every kernel behind
// its own fences.  The CTA barrier before / after
// makes the fence cumulative over the other threads' accesses (PTX memory model: causality order through bar.sync).
__device__ __forceinline__ void wait_flags(unsigned char* my_arena, const ArenaLayout& A, int row, int world,
                                           unsigned long long value) {
    if ((int)threadIdx.x < world) {
        const volatile unsigned long long* f = flag_ptr(my_arena, A, row, threadIdx.x);
        while (*f < value) __nanosleep(40);
        // acquire side: the flag lives in MY memory, whose point of coherence is my L2 -- the peer's row stores landed
        // there before its flag store became visible, and nothing of this kernel has read those rows yet
        __threadfence();
    }
    __syncthreads();
}
// every block: one thread fences the block's stores and counts in; the last block raises flag[row][me] = value on every peer
__device__ int g_dbg_mode = 0;  // LCTR_DIST_DEBUG bit0: serve_pull skips the row copies (timing experiment only)
// Blocks fence their stores at DEVICE scope and count in; only the last block (which has observed every other block's
// count) issues the system-scope fence before raising the flags -- cumulativity carries the other blocks' peer stores
// along.  One membar.sys per kernel instead of one per CTA (LCTR_DIST_FENCE=sys restores the per-block system fences; the
// choice was timed on B200s and has not been re-measured on H100s).
__device__ int g_block_fence_sys = 0;
__device__ __forceinline__ void raise_flags_last_block(const PeerTable& P, const ArenaLayout& A, int row, int me, int world,
                                                       unsigned long long value, unsigned int* ctr) {
    __shared__ bool last;
    __syncthreads();
    if (threadIdx.x == 0) {
        if (g_block_fence_sys) __threadfence_system(); else __threadfence();
        last = atomicAdd(ctr, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last && (int)threadIdx.x < world) {
        __threadfence_system();
        volatile unsigned long long* f = flag_ptr(P.p[threadIdx.x].arena, A, row, me);
        *f = value;
        if (threadIdx.x == 0) *ctr = 0;
        __threadfence_system();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// upload: per owner, the list of shard-local rows -> the owner's key inbox; rows of the exchange are then addressed by
// p = owner * cap_pair + position in that list, on both sides
// ---------------------------------------------------------------------------------------------------------------
// KEYED: uniq holds batch-local ids u; the owner comes from the top bits of fmix64(batch_key[u]), the pair is posted as
// {~0 (translated by the owner), requester slot} and the key goes to the key array of the same region
template <bool KEYED>
__global__ void __launch_bounds__(256)
send_keys_kernel(const uint32_t* __restrict__ uniq, const unsigned int* __restrict__ n_uniq, PeerTable P, ArenaLayout A,
                 int me, int world, int slot, int shift, unsigned cap_pair, unsigned int* __restrict__ send_cnt,
                 uint32_t* __restrict__ opos, int* __restrict__ overflow, const unsigned long long* __restrict__ batch_key) {
    __shared__ unsigned s_cnt[kMaxWorld], s_base[kMaxWorld];
    const unsigned n = *n_uniq;
    const unsigned mask = (unsigned)world - 1;
    for (unsigned c0 = blockIdx.x * blockDim.x; c0 < n; c0 += gridDim.x * blockDim.x) {
        if (threadIdx.x < kMaxWorld) s_cnt[threadIdx.x] = 0;
        __syncthreads();
        const unsigned i = c0 + threadIdx.x;
        uint32_t f = 0;
        unsigned o = 0, rk = 0;
        unsigned long long key = 0;
        if (i < n) {
            f = uniq[i];
            if (KEYED) {
                key = batch_key[f];
                o = owner_of_key(key, shift);
            } else {
                o = f & mask;
            }
            rk = atomicAdd(&s_cnt[o], 1u);
        }
        __syncthreads();
        if (threadIdx.x < world && s_cnt[threadIdx.x]) s_base[threadIdx.x] = atomicAdd(&send_cnt[threadIdx.x], s_cnt[threadIdx.x]);
        __syncthreads();
        if (i < n) {
            const unsigned j = s_base[o] + rk;
            if (j < cap_pair) {
                unsigned char* region = P.p[o].arena + A.key_inbox + ((size_t)slot * world + me) * A.key_region;
                uint2* pairs = reinterpret_cast<uint2*>(region + 64);
                if (KEYED) {
                    pairs[j] = make_uint2(kNoRow, i);
                    reinterpret_cast<unsigned long long*>(region + A.key_keys)[j] = key;
                } else {
                    pairs[j] = make_uint2(f >> shift, i);
                }
                opos[i] = o * cap_pair + j;
            } else {
                *overflow = 1;  // reported at the next host synchronisation; the row index stays in bounds
                opos[i] = o * cap_pair;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) __threadfence_system();  // after the loop's last CTA barrier: cumulative over the CTA's stores
}
// counts into the owners' headers (and kept locally for the push), counters re-armed, then the generation flag of
// (slot, me) on every owner.  Keyed contexts (overflow != nullptr) also post the requester status in hdr[1]: 1 = this rank
// refused its batch (the lists are empty), 2 = a list outgrew its region.
__global__ void send_keys_finish_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot, int flag_slot, unsigned cap_pair,
                                        unsigned int* send_cnt, unsigned int* seg_cnt, unsigned long long gen,
                                        const int* overflow, int refused) {
    const int o = threadIdx.x;
    __threadfence_system();
    if (o < world) {
        unsigned int* hdr = reinterpret_cast<unsigned int*>(P.p[o].arena + A.key_inbox + ((size_t)slot * world + me) * A.key_region);
        const unsigned n = refused ? 0u : min(send_cnt[o], cap_pair);
        hdr[0] = n;
        if (overflow) hdr[1] = refused ? 1u : (*overflow ? 2u : 0u);
        seg_cnt[o] = n;
        send_cnt[o] = 0;
        __threadfence_system();
        volatile unsigned long long* f = flag_ptr(P.p[o].arena, A, FLAG_KEYS + flag_slot, me);
        *f = gen;
    }
    __threadfence_system();
}
// entries: slot -> exchange row p (plain index of the parameter cache; gradient index unless the slot is hot); and the
// replica block of every hot exchange row
__global__ void __launch_bounds__(256)
remap_entries_kernel(const int64_t* __restrict__ hdr, int64_t nnz_arg, const uint32_t* __restrict__ opos,
                     uint32_t* __restrict__ ent_pslot, uint32_t* __restrict__ ent_slot, const uint32_t* __restrict__ hot_of,
                     const unsigned int* __restrict__ n_uniq, uint32_t* __restrict__ hot_p) {
    const int64_t nnz = hdr ? hdr[1] : nnz_arg;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i < nnz; i += nt) {
        const uint32_t pp = opos[ent_pslot[i]];
        ent_pslot[i] = pp;
        if (!(ent_slot[i] & kHotBit)) ent_slot[i] = pp;
    }
    if (hot_p) {
        const unsigned n = *n_uniq;
        for (int64_t i = t0; i < n; i += nt) {
            const uint32_t h = hot_of[i];
            if (h != 0xffffffffu) hot_p[opos[i]] = h;
        }
    }
}
// undo the hot marks of the previous batch of the slot (hot_p is all ~0 between uploads)
__global__ void __launch_bounds__(256)
clear_hot_p_kernel(const uint32_t* __restrict__ opos_prev, const uint32_t* __restrict__ hot_of_prev, unsigned n_prev,
                   uint32_t* __restrict__ hot_p) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n_prev; i += gridDim.x * blockDim.x)
        if (hot_of_prev[i] != 0xffffffffu) hot_p[opos_prev[i]] = 0xffffffffu;
}

// ---------------------------------------------------------------------------------------------------------------
// keyed upload (cfg.key_mode = LCTR_KEYS_HASHED).  Requester: the batch's keys -> batch-local ids u in [0, U) (the slot
// map and the send run on them unchanged, batch_key[u] gives the owner and the key that travels).  Owner: every key it
// received -> its local row (claimed and lazily initialised on first sight), written into pairs[j].x of its own inbox, so
// that serve / merge / union / updater kernels run unmodified; then a status flag on every requester.  Owner-side only,
// posted stores only: no rank probes or inserts into a peer's table.
// ---------------------------------------------------------------------------------------------------------------
// dedupe: claim a slot per distinct key; the claimer takes the next id and records the slot for the clear
__global__ void __launch_bounds__(256) batch_insert_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t,
                                                           uint32_t* __restrict__ claimed_slots) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;  // whole tiles leave together
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned long long key = keys[i];
    bool claimed;
    const long long pos = tile_claim(t, key, sub, gmask, &claimed);
    if (sub != 0) return;
    if (pos < 0) { t.flags[1] = 1u; return; }
    if (!claimed) return;
    const unsigned long long u = atomicAdd(t.count, 1ull);  // < table slots: every claim holds its own slot
    claimed_slots[u] = (uint32_t)pos;
    if (u < t.cap) {
        t.row[pos] = (uint32_t)u;
        t.row_key[u] = key;
    } else {
        t.row[pos] = kNoRow;
        t.flags[0] = 1u;
    }
}
// batch-local id of every entry into the slot's fid array (0 for a key without an id: the upload fails then)
__global__ void __launch_bounds__(256) batch_find_kernel(const unsigned long long* __restrict__ keys, int64_t n, KeyView t,
                                                         uint32_t* __restrict__ fid) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    if (i >= n) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const long long pos = tile_find(t, keys[i], sub, gmask);
    if (sub != 0) return;
    const uint32_t u = pos >= 0 ? __ldg(t.row + pos) : kNoRow;
    fid[i] = u == kNoRow ? 0u : u;
}
// the slots the dedupe claimed back to empty
__global__ void __launch_bounds__(256) batch_clear_kernel(KeyView t, const uint32_t* __restrict__ claimed_slots, size_t T) {
    const size_t n = min((size_t)*t.count, T);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t pos = claimed_slots[i];
        t.key[pos] = kEmptyKey;
        t.row[pos] = kNoRow;
    }
}

__device__ __forceinline__ unsigned char* key_region_of(const PeerTable& P, const ArenaLayout& A, int rank, int slot2, int world, int q) {
    return P.p[rank].arena + A.key_inbox + ((size_t)slot2 * world + q) * A.key_region;
}

// owner: every requester's lists of this (slot, generation) have landed, or a bounded wait has run out; a requester that
// refused its batch or overflowed a region fails the translation.  *xstat = first problem in rank order (0: none).
__global__ void xlate_wait_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot2, int flag_slot, unsigned long long gen,
                                  unsigned int* xstat) {
    __shared__ unsigned st[kMaxWorld];
    const int q = threadIdx.x;
    if (q < world) {
        const volatile unsigned long long* f = flag_ptr(P.p[me].arena, A, FLAG_KEYS + flag_slot, q);
        const long long t0 = clock64();
        bool late = false;
        while (*f < gen) {
            if (clock64() - t0 > kXlateWaitCycles) { late = true; break; }
            __nanosleep(256);
        }
        unsigned code = XS_OK;
        if (late) {
            code = XS_TIMEOUT;
        } else {
            __threadfence();
            const unsigned rs = reinterpret_cast<const volatile unsigned int*>(key_region_of(P, A, me, slot2, world, q))[1];
            code = rs == 1u ? XS_REFUSED : (rs == 2u ? XS_INBOX : XS_OK);
        }
        st[q] = code == XS_OK ? 0u : (code << 8 | (unsigned)q);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned first = 0;
        for (int r = world - 1; r >= 0; r--) if (st[r]) first = st[r];
        *xstat = first;
    }
}

// owner: MODE 0 claims a row for every received key (the key table's insert, new rows recorded for key_init_kernel);
// MODE 1 writes the local row of each into pairs[j].x (0 in place of a key left without a row; the upload fails then)
template <int MODE>
__global__ void __launch_bounds__(256) xlate_keys_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot2,
                                                         const unsigned int* __restrict__ xstat, KeyView t) {
    if (*xstat) return;
    const int sub = threadIdx.x & (kGroup - 1);
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const unsigned tile0 = (blockIdx.x * blockDim.x + threadIdx.x) / kGroup, ntiles = gridDim.x * blockDim.x / kGroup;
    for (int q = 0; q < world; q++) {
        unsigned char* region = key_region_of(P, A, me, slot2, world, q);
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(region + A.key_keys);
        uint2* pairs = reinterpret_cast<uint2*>(region + 64);
        for (unsigned j = tile0; j < n; j += ntiles) {  // the 16 lanes of a tile share j
            if (MODE == 0) {
                tile_insert(t, keys[j], sub, gmask);
            } else {
                const long long pos = tile_find(t, keys[j], sub, gmask);
                if (sub == 0) {
                    uint32_t r = pos >= 0 ? __ldg(t.row + pos) : kNoRow;
                    if (r == kNoRow) { t.flags[pos >= 0 ? 0 : 1] = 1u; r = 0; }
                    pairs[j].x = r;
                }
            }
        }
    }
}

// owner: its status (the wait's, else the table's) on every requester as seq << 16 | status; then, as requester, the
// statuses every owner raised for me (bounded wait) into xres[owner]
__global__ void xlate_finish_kernel(PeerTable P, ArenaLayout A, int me, int world, unsigned long long seq,
                                    const unsigned int* __restrict__ xstat, const unsigned int* __restrict__ tflags,
                                    unsigned long long* __restrict__ xres) {
    __shared__ unsigned s_st;
    if (threadIdx.x == 0) {
        unsigned st = *xstat;
        if (!st) st = tflags[1] ? (XS_TABLE_FULL << 8 | (unsigned)me) : (tflags[0] ? (XS_CAPACITY << 8 | (unsigned)me) : 0u);
        s_st = st;
    }
    __syncthreads();
    const int o = threadIdx.x;
    if (o < world) {
        volatile unsigned long long* f = flag_ptr(P.p[o].arena, A, FLAG_XLATED, me);
        *f = seq << 16 | s_st;
        __threadfence_system();
        const volatile unsigned long long* g = flag_ptr(P.p[me].arena, A, FLAG_XLATED, o);
        const long long t0 = clock64();
        unsigned long long v;
        while (((v = *g) >> 16) < seq) {
            if (clock64() - t0 > kXlateWaitCycles) { v = seq << 16 | (XS_TIMEOUT << 8 | (unsigned)o); break; }
            __nanosleep(256);
        }
        xres[o] = v & 0xffffull;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// step 1: owner-driven pull.  Requester r's rows from me land at its cache rows [me * cap_pair, me * cap_pair + n):
// consecutive list positions are consecutive rows, so a warp's stores form long contiguous runs on the wire
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMaxSl = 4;
__global__ void __launch_bounds__(256)
serve_pull_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot, int flag_slot, unsigned long long gen,
                  unsigned long long epoch, int rowlen, unsigned cap_pair, const float* __restrict__ W,
                  const float* __restrict__ V, unsigned int* done_ctr) {
    cudaTriggerProgrammaticLaunchCompletion();  // the compute kernel behind may be scheduled early: it polls the "rows delivered" flags
    wait_flags(P.p[me].arena, A, FLAG_KEYS + flag_slot, world, gen);  // every requester's key list of this upload has landed
    const int lane = threadIdx.x & 31;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    const int vec = (rowlen % 4 == 0) ? 4 : 1;
    const int slices = rowlen / vec;
    int lpr = 1;
    while (lpr < slices && lpr < 32) lpr <<= 1;
    const int G = 32 / lpr, q = lane % lpr, g = lane / lpr;
    for (int r = 0; r < world; r++) {
        if (g_dbg_mode & 1) break;
        const unsigned char* region = P.p[me].arena + A.key_inbox + ((size_t)slot * world + r) * A.key_region;
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const uint2* pairs = reinterpret_cast<const uint2*>(region + 64);
        float* cW = reinterpret_cast<float*>(P.p[r].arena + A.cacheW) + (size_t)me * cap_pair;
        float* cV = reinterpret_cast<float*>(P.p[r].arena + A.cacheV) + (size_t)me * cap_pair * rowlen;
        if (vec == 4 && slices <= lpr * kMaxSl) {
            constexpr int U = 4;  // row groups in flight before the first (posted) store leaves
            for (unsigned b0 = warp * (G * U); b0 < n; b0 += nwarps * (G * U)) {
                unsigned l[U];
                float4 v[U][kMaxSl];
                float w[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const unsigned j = b0 + u * G + g;
                    l[u] = j < n ? pairs[j].x : 0xffffffffu;
                    if (l[u] == 0xffffffffu) continue;
                    const float* src = V + (size_t)l[u] * rowlen;
#pragma unroll
                    for (int i = 0; i < kMaxSl; i++) {
                        const int sl = q + i * lpr;
                        if (sl < slices) v[u][i] = *reinterpret_cast<const float4*>(src + 4 * sl);
                    }
                    if (q == 0) w[u] = W[l[u]];
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (l[u] == 0xffffffffu) continue;
                    const unsigned j = b0 + u * G + g;
                    float* dst = cV + (size_t)j * rowlen;
#pragma unroll
                    for (int i = 0; i < kMaxSl; i++) {
                        const int sl = q + i * lpr;
                        if (sl < slices) *reinterpret_cast<float4*>(dst + 4 * sl) = v[u][i];
                    }
                    if (q == 0) cW[j] = w[u];
                }
            }
        } else {
            for (unsigned j = warp * G + g; j < n; j += nwarps * G) {  // generic fallback (odd row lengths)
                const float* src = V + (size_t)pairs[j].x * rowlen;
                float* dst = cV + (size_t)j * rowlen;
                for (int sl = q * vec; sl < rowlen; sl += lpr * vec)
                    for (int c = 0; c < vec; c++) dst[sl + c] = src[sl + c];
                if (q == 0) cW[j] = W[pairs[j].x];
            }
        }
    }
    raise_flags_last_block(P, A, FLAG_PULLED, me, world, epoch, done_ctr);
}

// stand-alone wait for compute kernels without an in-kernel wait (FFM / non-fused FM and NFM)
__global__ void wait_flags_kernel(PeerTable P, ArenaLayout A, int me, int row, int world, unsigned long long value) {
    wait_flags(P.p[me].arena, A, row, world, value);
}

// end of a pull-only round, launched behind the forward (its reads of my cache are complete): every owner may write my
// cache again
__global__ void release_cache_kernel(PeerTable P, ArenaLayout A, int me, int world, unsigned long long epoch) {
    const int o = threadIdx.x;
    if (o < world) {
        __threadfence_system();
        volatile unsigned long long* f = flag_ptr(P.p[o].arena, A, FLAG_RELEASED, me);
        *f = epoch;
        __threadfence_system();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// step 3: push.  The gradient rows of owner o are rows [o * cap_pair, o * cap_pair + n_o) of my compact buffer, in the
// order of the list o received: one contiguous stream of records [gV (rowlen) | gW | pad] into o's gradient inbox.
// ---------------------------------------------------------------------------------------------------------------
// gv / gw: row p at gv + p * gvs (rowlen floats) and gw + p * gws.  hot_p (fused FM / NFM kernels): rows whose entries were
// accumulated in kHotRep replica rows of Ghot -- folded here.  Local rows (and replicas) are re-zeroed.
__global__ void __launch_bounds__(256)
push_rows_kernel(const unsigned int* __restrict__ seg_cnt, float* __restrict__ gv, int gvs, float* __restrict__ gw, int gws,
                 const uint32_t* __restrict__ hot_p, float* __restrict__ Ghot, int GS, int rowlen, int recw, unsigned cap_pair,
                 PeerTable P, ArenaLayout A, int me, int world, unsigned long long epoch, unsigned int* done_ctr) {
    const int lane = threadIdx.x & 31;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    const int slices = rowlen / 4;  // rowlen % 4 == 0 is required by dist_alloc
    int lpr = 1;
    while (lpr < slices && lpr < 32) lpr <<= 1;
    const int G = 32 / lpr, q = lane % lpr, g = lane / lpr;
    cudaTriggerProgrammaticLaunchCompletion();  // the owner-side kernel behind polls the "pushes landed" flags
    cudaGridDependencySynchronize();            // launched dependent on the gradient kernel: its G / Ghot are complete from here
    for (int o = 0; o < world; o++) {
        const unsigned n = seg_cnt[o];
        float* inbox = reinterpret_cast<float*>(P.p[o].arena + A.grad_inbox + (size_t)me * A.grad_region);
        for (unsigned j = warp * G + g; j < n; j += nwarps * G) {
            const size_t pr = (size_t)o * cap_pair + j;
            float* src = gv + pr * gvs;
            float* dst = inbox + (size_t)j * recw;
            const uint32_t h = hot_p ? __ldg(hot_p + pr) : 0xffffffffu;
            float gwv = q == 0 ? gw[pr * gws] : 0.f;
            for (int sl = q; sl < slices; sl += lpr) {
                float4 v = *reinterpret_cast<const float4*>(src + 4 * sl);
                if (h != 0xffffffffu) {  // fold (and re-zero) the replica rows of a hot slot: column block sl; 16 loads in flight
                    float* tile = Ghot + (size_t)h * kHotRep * GS;
                    for (int r0 = 0; r0 < kHotRep; r0 += 16) {
                        float4 t[16];
#pragma unroll
                        for (int i = 0; i < 16; i++) t[i] = __ldcg(reinterpret_cast<const float4*>(tile + (size_t)(r0 + i) * GS + 4 * sl));
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            v.x += t[i].x; v.y += t[i].y; v.z += t[i].z; v.w += t[i].w;
                            *reinterpret_cast<float4*>(tile + (size_t)(r0 + i) * GS + 4 * sl) = make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                    }
                }
                *reinterpret_cast<float4*>(dst + 4 * sl) = v;
                *reinterpret_cast<float4*>(src + 4 * sl) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if (q == 0) {
                if (h != 0xffffffffu) {
                    float* tile = Ghot + (size_t)h * kHotRep * GS;
                    float t[kHotRep];
#pragma unroll
                    for (int rp = 0; rp < kHotRep; rp++) t[rp] = __ldcg(tile + (size_t)rp * GS + rowlen);
#pragma unroll
                    for (int rp = 0; rp < kHotRep; rp++) { gwv += t[rp]; tile[(size_t)rp * GS + rowlen] = 0.f; }
                }
                *reinterpret_cast<float4*>(dst + rowlen) = make_float4(gwv, 0.f, 0.f, 0.f);  // whole 16 B: the record leaves as full slices
                gw[pr * gws] = 0.f;
            }
        }
    }
    raise_flags_last_block(P, A, FLAG_PUSHED, me, world, epoch, done_ctr);
}

// ---------------------------------------------------------------------------------------------------------------
// step 4: owner folds the R gradient inboxes into its shard's update_g (local REDs) and marks the rows
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
merge_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot, unsigned long long epoch, int rowlen, int recw,
             float* __restrict__ gW, float* __restrict__ gV, uint8_t* __restrict__ touched) {
    wait_flags(P.p[me].arena, A, FLAG_PUSHED, world, epoch);  // every requester's records have landed
    const int lane = threadIdx.x & 31;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    const int slices = rowlen / 4;
    int lpr = 1;
    while (lpr < slices && lpr < 32) lpr <<= 1;
    const int G = 32 / lpr, q = lane % lpr, g = lane / lpr;
    for (int src = 0; src < world; src++) {
        const unsigned char* region = P.p[me].arena + A.key_inbox + ((size_t)slot * world + src) * A.key_region;
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const uint2* pairs = reinterpret_cast<const uint2*>(region + 64);
        const float* recs = reinterpret_cast<const float*>(P.p[me].arena + A.grad_inbox + (size_t)src * A.grad_region);
        for (unsigned j = warp * G + g; j < n; j += nwarps * G) {
            const float* rec = recs + (size_t)j * recw;
            const size_t l = pairs[j].x;
            float* gdst = gV + l * (size_t)rowlen;
            bool any = false;
            for (int sl = q; sl < slices; sl += lpr) {
                const float4 v = __ldcg(reinterpret_cast<const float4*>(rec + 4 * sl));
                if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) { red_add_v4(gdst + 4 * sl, v); any = true; }
            }
            if (q == 0) {
                const float w = __ldcg(rec + rowlen);
                if (w != 0.f) { red_add_f32(gW + l, w); any = true; }
            }
            if (any) touched[l] = 1;  // (idempotent byte store; every lane that added something marks the row)
        }
    }
}

// change tracking (lctr_track_changes): the owner marks every row it served for the step, the rows of the key lists its
// requesters posted for the slot (read after the merge, which waited for them)
__global__ void __launch_bounds__(256)
mark_served_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot2, uint8_t* __restrict__ map, size_t Fl) {
    for (int src = 0; src < world; src++) {
        const unsigned char* region = P.p[me].arena + A.key_inbox + ((size_t)slot2 * world + src) * A.key_region;
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const uint2* pairs = reinterpret_cast<const uint2*>(region + 64);
        for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
            const uint32_t l = pairs[j].x;
            if (l < Fl && !map[l]) map[l] = 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// fused FM / NFM path, owner side.  Once per upload: the union of the requesters' key lists (mark -> compact, the slot-map
// kernels of fm_fused.cuh on the shard) and each union row's position in every list.  Every step: ONE kernel that waits for
// the pushes, sums a row's records over the requesters in rank order (deterministic, no REDs) and applies the updater.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
own_mark_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot2, int flag_slot, unsigned long long gen,
                uint32_t* __restrict__ posmap, size_t Fl, uint8_t* __restrict__ mark, size_t T) {
    wait_flags(P.p[me].arena, A, FLAG_KEYS + flag_slot, world, gen);  // every requester's key list of this upload has landed
    for (int q = 0; q < world; q++) {
        const unsigned char* region = P.p[me].arena + A.key_inbox + ((size_t)slot2 * world + q) * A.key_region;
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const uint2* pairs = reinterpret_cast<const uint2*>(region + 64);
        for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
            const uint32_t l = pairs[j].x;
            posmap[(size_t)q * Fl + l] = j;  // never cleared: an entry counts only if list[entry] == row (own_pos_kernel)
            mark[(size_t)(l & 127u) * T + (l >> 7)] = 1;
        }
    }
}
__global__ void __launch_bounds__(256)
own_pos_kernel(PeerTable P, ArenaLayout A, int me, int world, int slot2, const uint32_t* __restrict__ own_uniq,
               const unsigned int* __restrict__ n_own, const uint32_t* __restrict__ posmap, size_t Fl,
               uint32_t* __restrict__ own_pos, unsigned cap_own) {
    const unsigned total = min(*n_own, cap_own);
    for (int q = 0; q < world; q++) {
        const unsigned char* region = P.p[me].arena + A.key_inbox + ((size_t)slot2 * world + q) * A.key_region;
        const unsigned n = *reinterpret_cast<const volatile unsigned int*>(region);
        const uint2* pairs = reinterpret_cast<const uint2*>(region + 64);
        for (unsigned u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
            const uint32_t l = own_uniq[u];
            const uint32_t j = posmap[(size_t)q * Fl + l];
            own_pos[(size_t)q * cap_own + u] = (j < n && pairs[j].x == l) ? j : 0xffffffffu;
        }
    }
}
template <int K, int OPT>
__global__ void __launch_bounds__(256)
merge_apply_kernel(PeerTable P, ArenaLayout A, int me, int world, unsigned long long epoch, int recw,
                   const uint32_t* __restrict__ own_uniq, const unsigned int* __restrict__ n_own,
                   const uint32_t* __restrict__ own_pos, unsigned cap_own, float* __restrict__ W, float* __restrict__ V,
                   float* __restrict__ s1W, float* __restrict__ s1V, float* __restrict__ s2W, float* __restrict__ s2V, OptParams Pp) {
    wait_flags(P.p[me].arena, A, FLAG_PUSHED, world, epoch);  // every requester's records of this step have landed
    cudaGridDependencySynchronize();  // (launched dependent on my own push kernel; its flag to myself is already in)
    constexpr int LPR = K / 4, GR = 32 / LPR;
    constexpr bool two = OPT == LCTR_OPT_FTRL || OPT == LCTR_OPT_ADAM || OPT == LCTR_OPT_ADADELTA || OPT == LCTR_OPT_PS_DCASGD ||
                         OPT == LCTR_OPT_PS_DCASGDA;
    Pp.opt = OPT;
    const int lane = threadIdx.x & 31, q = lane % LPR, g = lane / LPR;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    const unsigned total = min(*n_own, cap_own);
    for (unsigned b0 = warp * GR; b0 < total; b0 += nwarps * GR) {
        const unsigned idx = b0 + g;
        if (idx >= total) continue;
        const uint32_t l = own_uniq[idx];
        const size_t o = (size_t)l * K + 4 * q;
        float4 v4 = *reinterpret_cast<const float4*>(V + o), a4 = *reinterpret_cast<const float4*>(s1V + o);
        float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (two) b4 = *reinterpret_cast<const float4*>(s2V + o);
        float w = 0.f, a = 0.f, bb = 0.f;
        if (q == 0) { w = W[l]; a = s1W[l]; if (two) bb = s2W[l]; }
        float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float gw = 0.f;
        for (int src = 0; src < world; src++) {  // rank order: the sum is reproducible
            const uint32_t j = own_pos[(size_t)src * cap_own + idx];
            if (j == 0xffffffffu) continue;
            const float* rec = reinterpret_cast<const float*>(P.p[me].arena + A.grad_inbox + (size_t)src * A.grad_region) + (size_t)j * recw;
            const float4 t = __ldcg(reinterpret_cast<const float4*>(rec + 4 * q));
            g4.x += t.x; g4.y += t.y; g4.z += t.z; g4.w += t.w;
            if (q == 0) gw += __ldcg(rec + K);
        }
        update_one(Pp, Pp.corrV, v4.x, g4.x, a4.x, b4.x);
        update_one(Pp, Pp.corrV, v4.y, g4.y, a4.y, b4.y);
        update_one(Pp, Pp.corrV, v4.z, g4.z, a4.z, b4.z);
        update_one(Pp, Pp.corrV, v4.w, g4.w, a4.w, b4.w);
        *reinterpret_cast<float4*>(V + o) = v4;
        *reinterpret_cast<float4*>(s1V + o) = a4;
        if (two) *reinterpret_cast<float4*>(s2V + o) = b4;
        if (q == 0) {
            update_one(Pp, Pp.corrW, w, gw, a, bb);
            W[l] = w; s1W[l] = a;
            if (two) s2W[l] = bb;
        }
    }
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int dist_alloc(lctr_ctx* c) {
    const int R = c->cfg.world;
    LCTR_CHECK(R <= kMaxWorld && (R & (R - 1)) == 0, "world=%d: need a power of two <= %d", R, kMaxWorld);
    c->dist.reset(new DistState());
    DistState* d = c->dist.get();
    d->rank = c->cfg.rank; d->world = R;
    d->keyed = c->cfg.key_mode == LCTR_KEYS_HASHED;
    while ((1 << d->shift) < R) d->shift++;
    if (const char* de = getenv("LCTR_DIST_DEBUG")) {
        const int m = atoi(de);
        LCTR_CUDA(cudaMemcpyToSymbol(g_dbg_mode, &m, sizeof(int)));
    }
    if (const char* fe = getenv("LCTR_DIST_FENCE")) {
        const int sys = strcmp(fe, "gpu") != 0;
        LCTR_CUDA(cudaMemcpyToSymbol(g_block_fence_sys, &sys, sizeof(int)));
    }
    LCTR_CHECK(c->rowlen % 4 == 0, "multi-GPU exchange moves rows in 16 B slices: rowlen %zu must be a multiple of 4", c->rowlen);
    // keys of one batch: at most its entry count (cfg.max_nnz), at most the id space
    d->cap_keys = c->cfg.max_nnz ? std::min<size_t>(c->cfg.max_nnz, c->F) : c->F;
    // keys one requester sends one owner: U / R on average (owner = fid mod R, or the top bits of fmix64(key): binomially
    // tight either way); 1.5x that plus slack
    d->cap_pair = std::min<size_t>(c->Fl, 3 * d->cap_keys / (2 * R) + 4096);
    d->rows_x = (size_t)R * d->cap_pair;
    d->recw = (int)((c->rowlen + 4 + 3) / 4 * 4);
    ArenaLayout& A = d->A;
    size_t off = 0;
    A.flags = off; off = align_up(off + (size_t)(FLAG_KEYS + kNumSlots) * kMaxWorld * sizeof(unsigned long long), 256);
    A.key_keys = 64 + d->cap_pair * sizeof(uint2);
    A.key_region = align_up(A.key_keys + (d->keyed ? d->cap_pair * sizeof(unsigned long long) : 0), 256);
    A.key_inbox = off; off += A.key_region * kNumSlots * 2 * R;
    A.cacheW = off; off = align_up(off + d->rows_x * sizeof(float), 256);
    A.cacheV = off; off = align_up(off + d->rows_x * c->rowlen * sizeof(float), 256);
    A.grad_region = align_up(d->cap_pair * (size_t)d->recw * sizeof(float), 256);
    A.grad_inbox = off; off += A.grad_region * R;
    A.total = off;
    if (d->arena.alloc(A.total)) return 1;
    LCTR_CUDA(cudaMemsetAsync(d->arena, 0, A.total, c->stream));
    d->bytes += A.total;
    if (d->send_cnt.alloc(kMaxWorld)) return 1;
    LCTR_CUDA(cudaMemsetAsync(d->send_cnt, 0, kMaxWorld * sizeof(unsigned int), c->stream));
    if (d->seg_cnt.alloc((size_t)kNumSlots * kMaxWorld)) return 1;
    LCTR_CUDA(cudaMemsetAsync(d->seg_cnt, 0, (size_t)kNumSlots * kMaxWorld * sizeof(unsigned int), c->stream));
    if (d->opos.alloc((size_t)kNumSlots * d->cap_keys)) return 1;
    d->bytes += (size_t)kNumSlots * d->cap_keys * sizeof(uint32_t);
    if (d->done_ctr.alloc(4)) return 1;
    LCTR_CUDA(cudaMemsetAsync(d->done_ctr, 0, 4 * sizeof(unsigned int), c->stream));
    if (d->overflow.alloc(1)) return 1;
    LCTR_CUDA(cudaMemsetAsync(d->overflow, 0, sizeof(int), c->stream));
    if (c->grad_path == GRAD_COMPACT) {  // the fused FM / NFM kernels keep their gradients in fm_fused.cu's G / Ghot (rows p)
        if (d->hot_p.alloc((size_t)kNumSlots * d->rows_x)) return 1;
        LCTR_CUDA(cudaMemsetAsync(d->hot_p, 0xff, (size_t)kNumSlots * d->rows_x * sizeof(uint32_t), c->stream));
        d->bytes += (size_t)kNumSlots * d->rows_x * sizeof(uint32_t);
        d->cap_own = std::min<size_t>(c->Fl, d->rows_x);
        d->own_T = (c->Fl + 127) / 128;  // rows of the permuted byte map (fm_fused.cuh: mark_rows)
        if (d->own_uniq.alloc((size_t)kNumSlots * d->cap_own) || d->own_pos.alloc((size_t)kNumSlots * R * d->cap_own) ||
            d->n_own.alloc(kNumSlots))
            return 1;
        LCTR_CUDA(cudaMemsetAsync(d->n_own, 0, kNumSlots * sizeof(unsigned int), c->stream));
        if (d->posmap.alloc((size_t)R * c->Fl)) return 1;
        LCTR_CUDA(cudaMemsetAsync(d->posmap, 0xff, (size_t)R * c->Fl * sizeof(uint32_t), c->stream));
        if (d->own_mark.alloc(128 * d->own_T)) return 1;
        LCTR_CUDA(cudaMemsetAsync(d->own_mark, 0, 128 * d->own_T, c->stream));
        d->bytes += (size_t)kNumSlots * (R + 1) * d->cap_own * sizeof(uint32_t) + (size_t)R * c->Fl * sizeof(uint32_t) + 128 * d->own_T;
    } else {
        if (d->cgW.alloc(d->rows_x) || d->cgV.alloc(d->rows_x * c->rowlen)) return 1;
        LCTR_CUDA(cudaMemsetAsync(d->cgW, 0, d->rows_x * sizeof(float), c->stream));
        LCTR_CUDA(cudaMemsetAsync(d->cgV, 0, d->rows_x * c->rowlen * sizeof(float), c->stream));
        d->bytes += d->rows_x * (c->rowlen + 1) * sizeof(float);
    }
    if (d->keyed) {  // the requester's batch table (2x the key capacity of a batch, a power of two) and the status words
        size_t T = kGroup;
        while (T < 2 * d->cap_keys) T <<= 1;
        d->bt_T = T;
        if (d->bt_key.alloc(T) || d->bt_row.alloc(T) || d->bt_claimed.alloc(T) || d->bt_cnt.alloc(1) || d->bt_flags.alloc(3) ||
            d->batch_key.alloc(d->cap_keys) || d->xstat.alloc(1) || d->xres.alloc(kMaxWorld))
            return 1;
        LCTR_CUDA(cudaMemsetAsync(d->bt_key, 0xff, T * sizeof(unsigned long long), c->stream));
        LCTR_CUDA(cudaMemsetAsync(d->bt_row, 0xff, T * sizeof(uint32_t), c->stream));
        d->bytes += T * (sizeof(unsigned long long) + 2 * sizeof(uint32_t)) + d->cap_keys * sizeof(unsigned long long);
    }
    c->dist_rows = d->rows_x;
    // compute view: the batch-compact cache and gradient rows (indexed by exchange row p)
    c->cW = reinterpret_cast<float*>(d->arena + A.cacheW);
    c->cV = reinterpret_cast<float*>(d->arena + A.cacheV);
    c->cgW = d->cgW;
    c->cgV = d->cgV;
    memset(&d->peers, 0, sizeof(d->peers));
    d->peers.p[d->rank].arena = d->arena;
    return 0;
}

void dist_close_peers(lctr_ctx* c) {
    DistState* d = c->dist.get();
    for (int r = 0; r < d->world; r++)
        if (d->opened[r]) cudaIpcCloseMemHandle(d->opened[r]);
}

size_t dist_bytes(const lctr_ctx* c) { return c->dist ? c->dist->bytes : 0; }

void dist_wait_info(lctr_ctx* c, const unsigned long long** flags, int* n, unsigned long long* epoch) {
    DistState* d = c->dist.get();
    *flags = reinterpret_cast<const unsigned long long*>(d->arena + d->A.flags) + (size_t)FLAG_PULLED * kMaxWorld;
    *n = d->world;
    *epoch = d->epoch;
}

// key lists of the slot's batch -> the owners' inboxes (after the slot map of fm_fused.cu has been built on `st`)
int dist_send_keys(lctr_ctx* c, Slot& s, int slot, cudaStream_t st) {
    DistState* d = c->dist.get();
    LCTR_CHECK(d->imported, "multi-GPU upload before lctr_ipc_import");
    LCTR_CHECK((size_t)std::min<int64_t>(s.nnz, (int64_t)c->F) <= d->cap_keys,
               "batch of %lld entries exceeds the key capacity %zu of the multi-GPU context (cfg.max_nnz)", (long long)s.nnz, d->cap_keys);
    d->gen[slot]++;
    const int slot2 = slot * 2 + (int)(d->gen[slot] & 1);
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((std::min<int64_t>(s.nnz, (int64_t)c->F) + 255) / 256, (int64_t)c->sm_count * 4));
    uint32_t* opos = d->opos + (size_t)slot * d->cap_keys;
    uint32_t* hot_p = d->hot_p ? d->hot_p + (size_t)slot * d->rows_x : nullptr;
    if (hot_p) LCTR_CUDA(cudaMemsetAsync(hot_p, 0xff, d->rows_x * sizeof(uint32_t), st));  // the previous batch's hot rows
    // keyed: an overflow fails this upload only (reported through the owners' statuses)
    if (d->keyed) LCTR_CUDA(cudaMemsetAsync(d->overflow, 0, sizeof(int), st));
    if (launch(c, {grid, 256, 0, st}, d->keyed ? send_keys_kernel<true> : send_keys_kernel<false>, s.uniq, s.n_uniq, d->peers, d->A,
               d->rank, d->world, slot2, d->shift, (unsigned)d->cap_pair, d->send_cnt, opos, d->overflow,
               d->keyed ? d->batch_key.get() : nullptr) ||
        launch(c, {1, 32, 0, st}, send_keys_finish_kernel, d->peers, d->A, d->rank, d->world, slot2, slot, (unsigned)d->cap_pair,
               d->send_cnt, d->seg_cnt + (size_t)slot * kMaxWorld, d->gen[slot], d->keyed ? d->overflow.get() : nullptr, 0))
        return 1;
    d->posted = d->keyed;
    const unsigned rg = (unsigned)std::max<int64_t>(1, std::min<int64_t>((s.nnz + 255) / 256, (int64_t)c->sm_count * 8));
    return launch(c, {rg, 256, 0, st}, remap_entries_kernel, nullptr, s.nnz, opos, s.ent_pslot, s.ent_slot, hot_p ? s.hot_of.get() : nullptr,
                  s.n_uniq, hot_p);
}

// an empty share (0 rows or 0 entries): empty key lists and the generation flag on every owner, status OK -- the peers'
// serve / translation of this upload then finds my lists like any other
int dist_send_empty(lctr_ctx* c, int slot, cudaStream_t st) {
    DistState* d = c->dist.get();
    LCTR_CHECK(d->imported, "multi-GPU upload before lctr_ipc_import");
    d->gen[slot]++;
    const int slot2 = slot * 2 + (int)(d->gen[slot] & 1);
    if (d->keyed) LCTR_CUDA(cudaMemsetAsync(d->overflow, 0, sizeof(int), st));
    if (launch(c, {1, 32, 0, st}, send_keys_finish_kernel, d->peers, d->A, d->rank, d->world, slot2, slot, (unsigned)d->cap_pair,
               d->send_cnt, d->seg_cnt + (size_t)slot * kMaxWorld, d->gen[slot], d->keyed ? d->overflow.get() : nullptr, 0))
        return 1;
    d->posted = d->keyed;
    return 0;
}

// ---- keyed upload, host side (capi.cu: lctr_upload_batch_keys on world > 1) -------------------------------------------
int dist_keys_begin(lctr_ctx* c) {
    DistState* d = c->dist.get();
    LCTR_CHECK(d->imported, "multi-GPU upload before lctr_ipc_import");
    d->posted = false;
    return 0;
}

// the batch's keys -> batch-local ids in s.fid (device), U of them; fails (nothing sent yet) when U > cap_keys
int dist_keys_dedupe(lctr_ctx* c, Slot& s, const uint64_t* h_keys, int64_t nnz) {
    DistState* d = c->dist.get();
    if ((size_t)nnz > d->bt_stage_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        const size_t cap = (size_t)nnz + (size_t)nnz / 2;
        d->bt_stage_cap = 0;
        if (alloc_group(sized(d->bt_stage, cap))) return 1;
        d->bt_stage_cap = cap;
    }
    LCTR_CUDA(cudaMemcpyAsync(d->bt_stage, h_keys, (size_t)nnz * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream));
    LCTR_CUDA(cudaMemsetAsync(d->bt_cnt, 0, sizeof(unsigned long long), c->stream));
    LCTR_CUDA(cudaMemsetAsync(d->bt_flags, 0, 3 * sizeof(unsigned int), c->stream));
    const KeyView bt{d->bt_key, d->bt_row, d->batch_key, d->bt_cnt, d->bt_flags, nullptr, d->bt_T / kGroup, d->cap_keys};
    const unsigned tg = (unsigned)std::max<int64_t>(1, (nnz * kGroup + 255) / 256);
    const unsigned cg = (unsigned)std::max<int64_t>(1, std::min<int64_t>((std::min<int64_t>(nnz, (int64_t)d->bt_T) + 255) / 256,
                                                                         (int64_t)c->sm_count * 8));
    {
        ProfScope prof(c, PROF_KEYS);
        if (launch(c, {tg, 256, 0, c->stream}, batch_insert_kernel, d->bt_stage, nnz, bt, d->bt_claimed) ||
            launch(c, {tg, 256, 0, c->stream}, batch_find_kernel, d->bt_stage, nnz, bt, s.fid) ||
            launch(c, {cg, 256, 0, c->stream}, batch_clear_kernel, bt, d->bt_claimed, d->bt_T))
            return 1;
    }
    unsigned long long u = 0;
    unsigned int fl[3] = {0, 0, 0};
    LCTR_CUDA(cudaMemcpyAsync(&u, d->bt_cnt, sizeof(u), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaMemcpyAsync(fl, d->bt_flags, sizeof(fl), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    LCTR_CHECK(!fl[1] && u <= d->cap_keys, "lctr_upload_batch_keys: the batch has %llu distinct keys, more than the key capacity "
               "%zu of the multi-GPU context (cfg.max_nnz, at most feature_cnt + 1)", u, d->cap_keys);
    return 0;
}

// a rank that cannot send its batch still posts empty lists, marked refused, so that every peer fails the upload at once
int dist_keys_refuse(lctr_ctx* c, int slot) {
    DistState* d = c->dist.get();
    if (d->posted) return 0;
    d->gen[slot]++;
    const int slot2 = slot * 2 + (int)(d->gen[slot] & 1);
    if (launch(c, {1, 32, 0, c->stream}, send_keys_finish_kernel, d->peers, d->A, d->rank, d->world, slot2, slot,
               (unsigned)d->cap_pair, d->send_cnt, d->seg_cnt + (size_t)slot * kMaxWorld, d->gen[slot], d->overflow, 1))
        return 1;
    d->posted = true;
    return 0;
}

// owner side of the upload: translate what every requester sent me, raise my status on each, collect every owner's
// status for my own lists.  Returns non-zero with the message every rank composes alike when an owner failed.
int dist_keys_translate(lctr_ctx* c, int slot) {
    DistState* d = c->dist.get();
    const int slot2 = slot * 2 + (int)(d->gen[slot] & 1);
    d->posted = false;
    d->xseq++;
    KeyView t = keys_view(c);
    if (scratch_reserve(c, std::min(d->rows_x, keys_capacity(c)))) return 1;
    t = keys_view(c);  // the scratch may have moved
    LCTR_CUDA(cudaMemsetAsync(t.flags, 0, 3 * sizeof(unsigned int), c->stream));
    const unsigned tg = (unsigned)std::max<int64_t>(1, std::min<int64_t>(((int64_t)d->rows_x * kGroup + 255) / 256,
                                                                         (int64_t)c->sm_count * 16));
    {
        ProfScope prof(c, PROF_KEYS);
        if (launch(c, {1, 32, 0, c->stream}, xlate_wait_kernel, d->peers, d->A, d->rank, d->world, slot2, slot, d->gen[slot], d->xstat) ||
            launch(c, {tg, 256, 0, c->stream}, xlate_keys_kernel<0>, d->peers, d->A, d->rank, d->world, slot2, d->xstat, t) ||
            init_new_rows(c, (int64_t)std::min(d->rows_x, keys_capacity(c))) ||
            launch(c, {tg, 256, 0, c->stream}, xlate_keys_kernel<1>, d->peers, d->A, d->rank, d->world, slot2, d->xstat, t) ||
            launch(c, {1, 32, 0, c->stream}, xlate_finish_kernel, d->peers, d->A, d->rank, d->world, d->xseq, d->xstat, t.flags, d->xres))
            return 1;
    }
    unsigned long long res[kMaxWorld] = {0};
    LCTR_CUDA(cudaMemcpyAsync(res, d->xres, (size_t)d->world * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    for (int o = 0; o < d->world; o++) {
        if (!res[o]) continue;
        const unsigned code = (unsigned)(res[o] >> 8), r = (unsigned)(res[o] & 0xff);
        const unsigned long long fc = c->cfg.feature_cnt;
        switch (code) {
            case XS_CAPACITY:
                set_error("lctr_upload_batch_keys: owner rank %u: key shard capacity of %llu rows exhausted; the batch's new keys "
                          "do not fit (cfg.feature_cnt %llu over %d ranks)", r, (fc + d->world - 1 - r) / d->world, fc, d->world);
                break;
            case XS_TABLE_FULL:
                set_error("lctr_upload_batch_keys: owner rank %u: no free slot on a probe path of its key table", r);
                break;
            case XS_REFUSED:
                set_error("lctr_upload_batch_keys: rank %u refused its part of this collective upload (its own error names "
                          "the reason)", r);
                break;
            case XS_INBOX:
                set_error("lctr_upload_batch_keys: rank %u: a per-owner key list outgrew its inbox (%zu records, bounded by "
                          "cfg.max_nnz and by the rows of a shard)", r, d->cap_pair);
                break;
            default:
                set_error("lctr_upload_batch_keys: timed out waiting for rank %u (every rank must make the same collective "
                          "upload calls)", r);
                break;
        }
        return 1;
    }
    return 0;
}

// host-visible check (called where the host synchronises anyway): a key list that outgrew its inbox region is an error,
// never a silent drop
int dist_check_overflow(lctr_ctx* c) {
    DistState* d = c->dist.get();
    int h = 0;
    LCTR_CUDA(cudaMemcpyAsync(&h, d->overflow, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    LCTR_CHECK(h == 0, "multi-GPU: a per-owner key list outgrew its inbox (%zu records); raise cfg.max_nnz", d->cap_pair);
    return 0;
}

// train = false: a pull-only round (no owner-side union: only the merge reads it); end it with dist_release
int dist_pre_step(lctr_ctx* c, Slot& s, int slot, bool in_kernel_wait, bool train) {
    DistState* d = c->dist.get();
    LCTR_CHECK(d->imported, "multi-GPU step before lctr_ipc_import");
    LCTR_CHECK(s.fused_valid, "multi-GPU step on a slot without its key set");
    d->epoch++;
    if (train && c->grad_path == GRAD_COMPACT && d->own_gen[slot] != d->gen[slot]) {  // first step on this upload of the slot: the owner-side union
        const int slot2 = slot * 2 + (int)(d->gen[slot] & 1);
        const unsigned g1 = (unsigned)std::max<int64_t>(8, std::min<int64_t>((int64_t)c->sm_count * 4, ((int64_t)d->cap_pair + 255) / 256));
        LCTR_CUDA(cudaMemsetAsync(d->n_own + slot, 0, sizeof(unsigned int), c->stream));
        if (launch(c, {g1, 256, 0, c->stream}, own_mark_kernel, d->peers, d->A, d->rank, d->world, slot2, slot, d->gen[slot], d->posmap,
                   c->Fl, d->own_mark, d->own_T) ||
            launch_slotmap_compact(c, d->own_mark, d->own_T, d->own_uniq + (size_t)slot * d->cap_own, d->n_own + slot, c->stream) ||
            launch(c, {g1, 256, 0, c->stream}, own_pos_kernel, d->peers, d->A, d->rank, d->world, slot2,
                   d->own_uniq + (size_t)slot * d->cap_own, d->n_own + slot, d->posmap, c->Fl,
                   d->own_pos + (size_t)slot * d->world * d->cap_own, (unsigned)d->cap_own))
            return 1;
        d->own_gen[slot] = d->gen[slot];
    }
    if (d->released) {  // the previous round was pull-only: its requesters' kernels may still read their caches
        if (launch(c, {1, 32, 0, c->stream}, wait_flags_kernel, d->peers, d->A, d->rank, FLAG_RELEASED, d->world, d->released)) return 1;
        d->released = 0;
    }
    { ProfScope prof(c, PROF_DIST_PULL);
    // rows this rank serves ~ the union of what R requesters ask of it ~ (keys of a batch): one warp iteration = 32 rows (FM).
    // A rank with an empty share has no batch of its own to size by: it sizes for a full list (cap_pair)
    const int64_t serve_keys = s.nnz > 0 ? std::min<int64_t>(s.nnz, (int64_t)c->F) : (int64_t)d->cap_pair;
    const unsigned pull_grid = (unsigned)std::max<int64_t>(8, std::min<int64_t>((int64_t)c->sm_count * 4,
        (serve_keys * (int64_t)std::max<size_t>(1, c->rowlen / 16) + 255) / 256));
    if (launch(c, {pull_grid, 256, 0, c->stream}, serve_pull_kernel, d->peers, d->A, d->rank, d->world,
               slot * 2 + (int)(d->gen[slot] & 1), slot, d->gen[slot], d->epoch, (int)c->rowlen, (unsigned)d->cap_pair, c->W, c->V,
               d->done_ctr + 0))
        return 1; }
    if (in_kernel_wait) return 0;
    ProfScope prof(c, PROF_DIST_BAR1);
    return launch(c, {1, 32, 0, c->stream}, wait_flags_kernel, d->peers, d->A, d->rank, FLAG_PULLED, d->world, d->epoch);
}

// end of a pull-only round (behind its forward): my cache is released to every owner for the next round
int dist_release(lctr_ctx* c) {
    DistState* d = c->dist.get();
    if (launch(c, {1, 32, 0, c->stream}, release_cache_kernel, d->peers, d->A, d->rank, d->world, d->epoch)) return 1;
    d->released = d->epoch;
    return 0;
}

int dist_post_step(lctr_ctx* c, Slot& s, int slot, int64_t rows_divisor) {
    DistState* d = c->dist.get();
    const unsigned xgrid = (unsigned)std::max<int64_t>(8, std::min<int64_t>((int64_t)c->sm_count * 4,
        (std::min<int64_t>(s.nnz, (int64_t)c->F) * (int64_t)std::max<size_t>(1, c->rowlen / 16) + 255) / 256));
    const unsigned int* seg = d->seg_cnt + (size_t)slot * kMaxWorld;
    if (c->grad_path == GRAD_COMPACT) {  // push from G / Ghot, then merge + updater in one kernel over the owner-side union
        {
            ProfScope prof(c, PROF_DIST_PUSH);
            FusedState* f = c->fused.get();
            // dependent: behind the gradient kernel
            if (launch(c, {xgrid, 256, 0, c->stream, true}, push_rows_kernel, seg, f->G, f->GS, f->G + c->rowlen, f->GS,
                       d->hot_p + (size_t)slot * d->rows_x, f->Ghot, f->GS, (int)c->rowlen, d->recw, (unsigned)d->cap_pair, d->peers,
                       d->A, d->rank, d->world, d->epoch, d->done_ctr + 1))
                return 1;
        }
        ProfScope prof(c, PROF_DIST_MERGE);
        const OptParams Pp = make_opt_params(c, rows_divisor);
        auto kern = by_value<4, 8, 16, 32>((int)c->cfg.factor_cnt, [&](auto K) {
            return by_opt(Pp.opt, [&](auto o) { return merge_apply_kernel<K, o>; });
        });
        // dependent: behind my push kernel
        if (launch(c, {(unsigned)c->sm_count * 4, 256, 0, c->stream, true}, kern, d->peers, d->A, d->rank, d->world,
                   d->epoch, d->recw, d->own_uniq + (size_t)slot * d->cap_own, d->n_own + slot,
                   d->own_pos + (size_t)slot * d->world * d->cap_own, (unsigned)d->cap_own, c->W, c->V, c->s1W, c->s1V, c->s2W,
                   c->s2V, Pp))
            return 1;
        // change tracking: the owner-side union of the requesters' lists is the set of rows served
        return track_mark_rows(c, d->own_uniq + (size_t)slot * d->cap_own, d->n_own + slot, d->cap_own);
    }
    { ProfScope prof(c, PROF_DIST_PUSH);
    if (launch(c, {xgrid, 256, 0, c->stream}, push_rows_kernel, seg, d->cgV, (int)c->rowlen, d->cgW, 1, nullptr, nullptr, 0,
               (int)c->rowlen, d->recw, (unsigned)d->cap_pair, d->peers, d->A, d->rank, d->world, d->epoch, d->done_ctr + 1))
        return 1; }
    { ProfScope prof(c, PROF_DIST_MERGE);
    if (launch(c, {xgrid, 256, 0, c->stream}, merge_kernel, d->peers, d->A, d->rank, d->world, slot * 2 + (int)(d->gen[slot] & 1),
               d->epoch, (int)c->rowlen, d->recw, c->gW, c->gV, c->touched))
        return 1; }
    if (launch_apply(c, rows_divisor)) return 1;  // sparse updater on the shard (the merge waited for every requester's pushes)
    if (!c->changed) return 0;
    return launch(c, {(unsigned)std::max<int64_t>(8, std::min<int64_t>((int64_t)c->sm_count * 4, ((int64_t)d->cap_pair + 255) / 256)),
                      256, 0, c->stream}, mark_served_kernel, d->peers, d->A, d->rank, d->world,
                  slot * 2 + (int)(d->gen[slot] & 1), c->changed, c->Fl);
}

}  // namespace lctr

using namespace lctr;

extern "C" {

// one handle per rank: its arena, the only buffer a peer reads or writes
int lctr_ipc_export(lctr_ctx* c, void* handles_out, size_t cap, size_t* bytes) {
    LCTR_CHECK(c && bytes, "null argument");
    LCTR_CHECK(c->dist, "lctr_ipc_export: ctx was created with world == 1");
    const size_t need = sizeof(cudaIpcMemHandle_t);
    *bytes = need;
    if (!handles_out) return 0;
    LCTR_CHECK(cap >= need, "lctr_ipc_export: need %zu bytes", need);
    cudaIpcMemHandle_t h;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    LCTR_CUDA(cudaIpcGetMemHandle(&h, c->dist->arena));
    memcpy(handles_out, &h, sizeof(h));
    return 0;
}

int lctr_ipc_import(lctr_ctx* c, const void* all_handles, size_t bytes_per_rank) {
    LCTR_CHECK(c && all_handles, "null argument");
    LCTR_CHECK(c->dist, "lctr_ipc_import: ctx was created with world == 1");
    LCTR_CHECK(bytes_per_rank == sizeof(cudaIpcMemHandle_t),
               "lctr_ipc_import: bytes_per_rank %zu, this build exports %zu (size the blob with lctr_ipc_export(ctx, NULL, 0, &n))",
               bytes_per_rank, sizeof(cudaIpcMemHandle_t));
    DistState* d = c->dist.get();
    const unsigned char* base = reinterpret_cast<const unsigned char*>(all_handles);
    for (int r = 0; r < d->world; r++) {
        if (r == d->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, base + (size_t)r * bytes_per_rank, sizeof(h));
        LCTR_CUDA(cudaIpcOpenMemHandle(&d->opened[r], h, cudaIpcMemLazyEnablePeerAccess));
        d->peers.p[r].arena = (unsigned char*)d->opened[r];
    }
    d->imported = true;
    return 0;
}

/* device memory of this context in bytes: the shard figure is W, V and the updater state (s1, and s2 for two-state
 * updaters), plus update_g (gW / gV, the size of W and V) on the dense path and for the grouped FFM backward, plus the
 * touched map (1 B per row) on the dense path, plus the key table in keyed mode; the exchange figure is the multi-GPU
 * arena, caches and index buffers (DESIGN.md 6) */
int lctr_device_bytes(lctr_ctx* c, uint64_t* shard_bytes, uint64_t* exchange_bytes) {
    LCTR_CHECK(c, "null ctx");
    const size_t tables = 2 + (c->s2W ? 1 : 0) + (c->gW ? 1 : 0);  // [W | V] blocks: parameters, s1, s2, update_g
    if (shard_bytes) *shard_bytes = (uint64_t)(c->Fl * (c->rowlen + 1) * sizeof(float) * tables + (c->touched ? c->Fl : 0) + (c->changed ? c->Fl : 0) + keys_bytes(c));
    if (exchange_bytes) *exchange_bytes = (uint64_t)dist_bytes(c);
    return 0;
}

}  // extern "C"
