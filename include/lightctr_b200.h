/* include/lightctr_b200.h -- the drop-in boundary (C ABI) of the H100-native LightCTR hot path.
 *
 * The reference (cnkuangshi/LightCTR) has no FFI: its "API" is C++ inheritance
 * (FM_Algo_Abst::Train() fm_algo_abst.h:137, Train_FM_Algo/Train_FFM_Algo/Train_NFM_Algo ctors
 * train_fm_algo.h:23, train_ffm_algo.h:25, train_nfm_algo.h:21, Fully_Conn_Layer
 * train/layer/fullyconnLayer.h:80-206, updaters util/gradientUpdater.h:128-278,
 * util/momentumUpdater.h:172-215).  The host shims in lightctr_b200/host/ keep those class
 * surfaces; each of their methods lowers to the entry points below.  Plain pointers and sizes
 * only, no C++/torch types, no exceptions across the boundary.  Every function returns 0 on
 * success, non-zero on failure (lctr_last_error() gives the message; the host shims turn that
 * into the reference's own style: print + exit(1), fm_algo_abst.h:79-82).
 *
 * Threading: one ctx per trainer, driven from one host thread (the reference's Train() is
 * synchronous and single-caller, SURVEY.md 8b).  All device work is issued on the ctx's
 * stream; calls that return host-visible results synchronise that stream only.
 */
#ifndef LIGHTCTR_B200_H
#define LIGHTCTR_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define LCTR_ABI_VERSION 1

typedef struct lctr_ctx lctr_ctx;

/* LCTR_MODEL_WND: Wide&Deep with the per-field concat input of Distributed_Algo_Abst (distributed_algo_abst.h:176-280):
 * factor_cnt = the tensor width d (the reference's factor_dim 4), field_cnt > 0, hidden[] = the dense chain on the
 * field_cnt * d input; single GPU, RED scatter. */
enum { LCTR_MODEL_FM = 1, LCTR_MODEL_FFM = 2, LCTR_MODEL_NFM = 3, LCTR_MODEL_WND = 4 };
/* updater = the reference's `_Num` family member (gradientUpdater.h:128-154 Adagrad, :200-233 RMSprop,
 * :235-278 FTRL; momentumUpdater.h:74-111 Adadelta, :172-215 Adam) */
enum { LCTR_OPT_ADAGRAD = 0, LCTR_OPT_FTRL = 1, LCTR_OPT_ADAM = 2, LCTR_OPT_RMSPROP = 3, LCTR_OPT_ADADELTA = 4,
       /* the parameter server's own update rules (distribut/paramserver.h:232-300), applied by the owner of a row to the
        * step's summed gradient as ONE push of worker 0: SGD (:295-300, the PS default :49; Wide&Deep tensors use the tensor
        * form :232-237), Adagrad (:288-294), DCASGD / DCASGDA (:252-286; shadow copy and accumulator kept per coordinate).
        * The synchronous exchange has no staleness, so the delay-compensation term of DCASGD* sees the parameter change
        * since the previous step. */
       LCTR_OPT_PS_SGD = 5, LCTR_OPT_PS_ADAGRAD = 6, LCTR_OPT_PS_DCASGD = 7, LCTR_OPT_PS_DCASGDA = 8 };
enum { LCTR_ACT_SIGMOID = 0, LCTR_ACT_TANH = 1 };
enum { LCTR_MLP_FP32 = 0, LCTR_MLP_BF16 = 1 };
enum { LCTR_KEYS_DENSE = 0, LCTR_KEYS_HASHED = 1 };

#define LCTR_MAX_LAYERS 8

/* Snapshot of the reference's process-global statics (main.cpp:64-73; SURVEY.md 8b "Hyper-parameter
 * sources") plus the trainer ctor arguments.  Zero-initialise, then fill. */
typedef struct lctr_cfg {
    uint32_t abi_version;     /* LCTR_ABI_VERSION */
    int32_t model;            /* LCTR_MODEL_* */
    int32_t optimizer;        /* LCTR_OPT_* for W and V (and the MLP, which the reference fixes to Adagrad) */
    int32_t device;           /* CUDA device ordinal */
    uint64_t feature_cnt;     /* F = max fid + 1 (fm_algo_abst.h:95) */
    uint32_t field_cnt;       /* Fc; 0 for FM/NFM (fm_algo_abst.h:57-59) */
    uint32_t factor_cnt;      /* k */
    float learning_rate;      /* GradientUpdater::__global_learning_rate */
    float l2_reg;             /* L2Reg_ratio (train_fm_algo.cpp:13) */
    uint64_t minibatch_size;  /* updater divisor; 0 => rows of the step (FM/FFM: train_fm_algo.cpp:38) */
    float momentum;           /* MomentumUpdater::__global_momentum       (Adam beta1 -- used for BOTH moments) */
    float momentum_adam2;     /* MomentumUpdater::__global_momentum_adam2 (Adam bias correction only) */
    float ftrl_alpha, ftrl_beta, ftrl_lambda1, ftrl_lambda2; /* gradientUpdater.h:275; 0 => reference defaults */
    /* MLP (NFM deep part): dims k -> hidden[0] -> ... -> hidden[n_hidden-1] -> 1 */
    int32_t n_hidden;
    uint32_t hidden[LCTR_MAX_LAYERS];
    int32_t activation;       /* LCTR_ACT_* of the hidden layers */
    int32_t mlp_precision;    /* LCTR_MLP_FP32 (parity) or LCTR_MLP_BF16 (tensor-core perf mode) */
    /* capacity hints (0 => grow on demand) */
    uint64_t max_rows, max_nnz;
    /* multi-GPU: this process' rank / world (1 process per GPU); tables are owner-sharded by fid % world */
    int32_t rank, world;
    /* Backward scatter-add strategy (FFM: 0 and 2 only):
     *  0  vector REDs into update_g + sparse apply (sum order arbitrary, like the reference's Hogwild threads);
     *  1  feature-major (CSC) view of the slot built on the HOST at upload: every gradient is summed in ascending
     *     row order -- the order of the reference's canonical single-thread run -- no atomics, updater fused.
     *     csc_row_block = rows per train_step range (0 => whole slot; NFM: the minibatch size);
     *  2  the same view built on the DEVICE at upload (overlaps the previous step); entries of a feature arrive in
     *     arbitrary order and are accumulated in double precision, so the fp32 result is order-independent.
     *     Whole-slot steps only; FM with k in {4, 8, 16, 32}, FFM with k % 4 == 0 and field_cnt * k <= 512. */
    int32_t deterministic;
    /* LCTR_KEYS_DENSE (0): fids index the tables directly, feature_cnt = max fid + 1.
     * LCTR_KEYS_HASHED (1): batches carry uint64_t hashed keys (lctr_upload_batch_keys); the library maps each key to a
     * table row, creating and initialising rows on first sight.  feature_cnt is then the row CAPACITY (< 2^32 - 1, and
     * >= world); deterministic = 0 only.  world > 1: the key table is sharded, see "keyed mode on several GPUs" below. */
    int32_t key_mode;
    uint64_t csc_row_block;
    float ema_rate;           /* GradientUpdater::__global_ema_rate (RMSpropUpdater_Num, gradientUpdater.h:200-233); 0 => 0.99 (main.cpp:66) */
    /* keyed mode only: 1 = every row records the insert-upload that last met it (8 B per row), which lctr_evict_keys
     * needs; 0 = no record (refused on a dense context when non-zero, and with world > 1) */
    int32_t key_evict;
    union {
        /* keyed mode only: capacity in rows of the host tier that keeps evicted rows (see lctr_evict_keys); 0 = no tier.
         * Needs key_mode = LCTR_KEYS_HASHED, key_evict = 1 and world = 1.  Takes (16 + 4 (rowlen + 1) (1 + states)) bytes
         * of pinned host memory per row, states = 2 for the two-state updaters (FTRL, Adam, Adadelta, DCASGD, DCASGDA)
         * and 1 otherwise, and an index of T = 2^m >= 2 key_host_rows slots of 12 B in device memory. */
        uint32_t key_host_rows;
        uint32_t reserved[2]; /* reserved[1] must stay 0 */
    };
} lctr_cfg;

const char* lctr_last_error(void);
int lctr_abi_version(void);

/* ---- lifetime ------------------------------------------------------------------------------- */
int lctr_create(const lctr_cfg* cfg, lctr_ctx** out);
int lctr_destroy(lctr_ctx* ctx);
int lctr_sync(lctr_ctx* ctx);

/* ---- parameters (replaces direct pokes at FM_Algo_Abst::W / V, fm_algo_abst.h:141,145) ------- */
/* V layout == reference: FM/NFM V[fid*k + f] (fm_algo_abst.h:146-148); FFM V[fid*Fc*k + field*k + f] (:149-151) */
int lctr_upload_params(lctr_ctx* ctx, const float* W, const float* V);
int lctr_download_params(lctr_ctx* ctx, float* W, float* V);
/* synthetic initialisation on the device: W = 0, V ~ scale * N(0,1) (hash of the global element index; independent
 * of the sharding).  Used by bench.py for tables too large to stage through host memory. */
int lctr_fill_params(lctr_ctx* ctx, uint64_t seed, float scale);
/* optimizer state: s1 = adagrad accum | ftrl z | adam m ; s2 = ftrl n | adam v ; each F + |V| floats, W part first
 * (same concatenation as update_g, train_fm_algo.h:52-57).  NULL pointers are skipped.  world > 1: full global arrays, as
 * lctr_upload_params / lctr_download_params take them; each rank fills / takes only the rows it owns. */
int lctr_download_opt_state(lctr_ctx* ctx, float* s1, float* s2);
int lctr_upload_opt_state(lctr_ctx* ctx, const float* s1, const float* s2);

/* ---- data: CSR form of FM_Algo_Abst::dataSet / label (fm_algo_abst.h:29-35,156,170) ---------- */
/* Copies one CSR batch (or a whole dataset) host->device into `slot` (0..3), asynchronously on the
 * ctx stream.  row_ptr has rows+1 entries; field may be NULL for FM/NFM; val may be NULL meaning all
 * 1.0f (the shipped data).  Indexing is bit-exact w.r.t. the reference parser. */
int lctr_upload_batch(lctr_ctx* ctx, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr,
                      const uint32_t* fid, const uint16_t* field, const float* val, const int32_t* label);

/* ---- keyed mode (cfg.key_mode = LCTR_KEYS_HASHED) ------------------------------------------- */
/* Replaces the host-side vocabulary a caller would otherwise build to renumber hashed ids into 0..F-1; the reference
 * keeps such a map only on its parameter server (size_t keys, created on first touch, distribut/paramserver.h:315-339).
 * The table rows are what the row-indexed calls see: lctr_upload_params / lctr_download_params and the opt-state
 * transfers take `capacity` rows (rows not allocated yet read as zero); train_step, predict, eval and the MLP calls work
 * unchanged.  lctr_upload_batch, lctr_train_batch and lctr_train_batch_async are refused on a keyed context.
 *
 * Keyed twin of lctr_upload_batch (same validation of row_ptr and field).  insert = 1 (training): a key seen for the first
 * time gets the next free row, initialised as W = 0, V = scale * N(0,1) drawn from a hash of (seed, key, element) -- the
 * values depend on the key only, never on its row or on arrival order; they are NOT the reference's rand() stream -- and
 * the optimizer state lctr_create gives.  insert = 0 (prediction): unseen keys map to a null row of zeros that is never
 * updated, i.e. the feature is dropped (predict/fm_predict.cpp:122); lctr_train_step refuses such a slot.  Wide&Deep reads
 * the first id of each field, which may then be the null row (the reference's server would create a fresh tensor).  A
 * batch whose new keys exceed the capacity fails naming it: keys inserted before keep their rows, the slot is unusable
 * until uploaded again.  The key 0xFFFFFFFFFFFFFFFF is reserved. */
int lctr_upload_batch_keys(lctr_ctx* ctx, int slot, int64_t rows, int64_t nnz, const int64_t* row_ptr,
                           const uint64_t* key, const uint16_t* field, const float* val, const int32_t* label, int insert);
/* row of each key, -1 when absent; never inserts */
int lctr_lookup_keys(lctr_ctx* ctx, int64_t n, const uint64_t* keys, int64_t* rows);
/* row -> key map of rows [0, *n_rows); keys may be NULL to query the count, otherwise it must hold cap >= *n_rows */
int lctr_download_keys(lctr_ctx* ctx, uint64_t* keys, uint64_t cap, uint64_t* n_rows);
/* parameters of the given keys (replaces lctr_upload_params for keyed tables).  Absent keys get consecutive rows in
 * array order (seeding keys[i] in order on a fresh context gives row i) and the optimizer state lctr_create gives; present
 * keys keep their row and state.  W (n) / V (n * rowlen) may be NULL.  A duplicate key is an error. */
int lctr_upload_keyed_params(lctr_ctx* ctx, int64_t n, const uint64_t* keys, const float* W, const float* V);
/* lazy-init parameters of new rows; defaults seed 0, scale 1 / sqrt(k) (the reference's scale, fm_algo_abst.h:62-65) */
int lctr_set_key_init(lctr_ctx* ctx, uint64_t seed, float scale);
/* Eviction of idle rows (cfg.key_evict = 1), so that a drifting key stream can train within a fixed capacity.
 * Clock: every lctr_upload_batch_keys with insert = 1 advances a u64 counter by one, then stamps every row it meets (new or
 * not) with the new value; lctr_upload_keyed_params stamps the rows it names with the current value; lookup-only uploads
 * and lctr_lookup_keys stamp nothing.  The age of a row is clock - stamp (0: met by the latest insert-upload).
 * lctr_evict_keys frees
 *   1. every row older than max_idle;
 *   2. if more than max_rows rows remain, also the oldest: only rows younger than a* stay, a* the largest age for which
 *      that set holds at most max_rows rows (rows that tie at the cutoff leave together).  UINT64_MAX = no limit.
 * keys_out / W_out / V_out (each may be NULL) receive the evicted keys in ascending order of their old row, their W (n)
 * and V (n * rowlen); when any is given, cap_out must be >= the number evicted, else the call fails and nothing changes.
 * *n_evicted receives that number.  Survivors are renumbered by one fixed rule: with n_live survivors, a survivor below
 * row n_live keeps its row; the j-th survivor at or above n_live (ascending) moves into the j-th evicted row below n_live
 * (ascending), carrying W, V, the optimizer state and its stamp bit for bit.  Rows [n_live, rows in use) return to the
 * state lctr_create gives and the table is rebuilt from the survivors, so keys stored without a row after a capacity
 * overflow are forgotten.  When a row was freed, every resident keyed slot becomes stale: train_step and predict refuse
 * it until it is uploaded again.  Without a host tier, an evicted key that comes back is a new key: lazy-init values
 * (which depend on the key only) and fresh optimizer state; re-uploading exported rows with lctr_upload_keyed_params
 * restores W and V, also with fresh optimizer state.  With a host tier (cfg.key_host_rows, below) the evicted rows are
 * kept there and come back whole.  Refused on a dense context and on a keyed context created with key_evict = 0. */
int lctr_evict_keys(lctr_ctx* ctx, uint64_t max_idle, uint64_t max_rows, uint64_t* keys_out, float* W_out, float* V_out,
                    uint64_t cap_out, uint64_t* n_evicted);
/* Host tier (cfg.key_host_rows > 0; keyed, key_evict = 1, one GPU), so that the model can outgrow device memory.
 * THE RULE: on a tiered context the model is the device rows plus the tier rows.  A key lives in at most one of them,
 * and no call except lctr_evict_host_tier loses one.  A tier row holds the key, its stamp, W, V and the optimizer state.
 *   lctr_evict_keys: the same rule, renumbering and export as without a tier, but the evicted rows are appended to the tier
 *     (in export order) instead of being dropped; without room in the tier for all of them the call fails before
 *     anything changes, naming the tier's capacity and its free rows.
 *   lctr_upload_batch_keys, insert = 1: a key absent from the device but held in the tier gets a device row as a new key
 *     does, then its W, V and optimizer state from the tier bit for bit (in place of the lazy init), and the new clock as
 *     any row the upload meets; it leaves the tier.  A key the capacity check refuses stays in the tier unchanged.
 *   lctr_upload_batch_keys, insert = 0: keys held in the tier are brought back the same way and keep their tier stamp;
 *     the clock does not advance; keys in neither table map to the null row.  Restoring past the device capacity fails
 *     with the capacity message, as an insert-upload does.
 *   lctr_upload_keyed_params: a key held in the tier counts as present: it gets its device row by the rule for absent
 *     keys, its optimizer state from the tier, then the call's W / V.
 *   lctr_lookup_keys, lctr_download_keys, the parameter and the opt-state transfers see the device rows only.
 *   Checkpoints carry the tier (a tiered file and an untiered context refuse each other, as files of another key_evict).
 * Cost: restored and spilled rows cross PCIe as zero-copy 16-byte accesses (scalar when rowlen % 4 != 0); keys that miss
 * the tier cost one probe of its device-side index per new row. */
/* the tier's rows in tier order: keys [n], W [n], V [n * rowlen]; keys = W = V = NULL queries *n_rows, otherwise each
 * non-NULL array must hold cap >= *n_rows rows.  The only view of the part of the model held in the tier. */
int lctr_download_host_tier(lctr_ctx* ctx, uint64_t* keys, float* W, float* V, uint64_t cap, uint64_t* n_rows);
/* lctr_evict_keys's rule, tie handling, export order (ascending tier row) and cap_out contract, applied to the tier's
 * stamps against the same clock.  The rows it frees leave the model; the rest are renumbered by the same rule. */
int lctr_evict_host_tier(lctr_ctx* ctx, uint64_t max_idle, uint64_t max_rows, uint64_t* keys_out, float* W_out, float* V_out,
                         uint64_t cap_out, uint64_t* n_evicted);
/* Frequency admission (keyed, world = 1, FM / FFM / NFM), so that keys met once and never again get no row: a new key
 * gets a row only once it has been met min_count times.  The counts live in a count-min sketch in device memory: 4 rows
 * of 2^log2_width u32 counters (16 * 2^log2_width bytes, counted by lctr_device_bytes), log2_width in [10, 28]; counter i
 * (0..3) of key x is
 *     fmix64(x ^ ((i + 1) * 0x9E3779B97F4A7C15)) >> (64 - log2_width)      (arithmetic mod 2^64)
 * with fmix64 the MurmurHash3 finaliser of the owner rule below.  The count of a key is the smallest of its 4 counters.
 * A key is PRESENT when the key table holds it (with a row, or without one after a capacity overflow) or the host tier
 * holds it.  One lctr_upload_batch_keys with insert = 1:
 *   1. every entry whose key is not present adds 1 to the key's 4 counters (entries, not distinct keys: the counts do not
 *      depend on order);
 *   2. then a key that is not present is admitted when its count is >= min_count, and gets a row as a new key does (lazy
 *      init, capacity check and failure message unchanged);
 *   3. every entry of a key that is not admitted is removed from the batch: kept entries keep their order within their
 *      row, with their field / val.  Rows are never removed: labels, the row count and the per-row outputs
 *      (lctr_predict, lctr_download_pred) stay aligned with the caller's rows, and a row that lost every entry trains as
 *      a row without entries does;
 *   4. key_evict = 1: the clock advances as always; only rows that kept entries are stamped.
 * Present keys (tier keys restored by the upload included) are never counted or dropped; insert = 0 uploads count and
 * drop nothing; lctr_upload_keyed_params creates the keys it names whatever their count.  Eviction leaves the counters as
 * they are, so an evicted key is admitted again at its next occurrence unless the sketch was decayed or reset since.
 * Checkpoints carry the settings and the sketch (header flag bit 10): lctr_load_checkpoint requires the same settings on
 * both sides (off = off) and refuses otherwise before writing anything, naming both; lctr_load_checkpoint_shards into a
 * context with admission off ignores the section, into one with other settings it refuses.  Files saved with admission off
 * keep their bytes.
 *
 * lctr_set_key_admission sets min_count and zeroes the sketch, at any time.  min_count <= 1 turns admission off and frees
 * the sketch (log2_width is then ignored): the context behaves, and launches, exactly as one that never called it.
 * Refused on a dense context, with world > 1, on Wide&Deep (it reads the first id of each field, which dropping entries
 * would change) and with log2_width outside [10, 28].
 * lctr_decay_key_admission shifts every counter right by shift, in [1, 32] (32 clears the sketch), so that admission can
 * age with a drifting stream: without it collisions fill a finite sketch and eventually admit everything.
 * lctr_key_admission_stats gives the entries the last insert-upload dropped and the keys it admitted (0 and 0 when
 * admission is off); either pointer may be NULL. */
int lctr_set_key_admission(lctr_ctx* ctx, uint32_t min_count, uint32_t log2_width);
int lctr_decay_key_admission(lctr_ctx* ctx, uint32_t shift);
int lctr_key_admission_stats(lctr_ctx* ctx, uint64_t* dropped_entries, uint64_t* admitted_keys);
/* Keyed mode on several GPUs (world > 1; the reference's parameter servers key by size_t and create on first touch,
 * distribut/paramserver.h:315-339).
 * Owner rule: key k lives on rank fmix64(k) >> (64 - log2 world) (the top bits of MurmurHash3's 64-bit finaliser); the
 * owner's table takes its home slot from the low bits.  Local row l of rank o is global row l * world + o -- the dense
 * convention -- so lctr_upload_params / lctr_download_params with full arrays of feature_cnt rows keep working, and rank o
 * holds at most the number of global rows < feature_cnt it owns.
 * lctr_upload_batch_keys (insert = 1) is COLLECTIVE: every rank calls it for the same slot, in the same order, each with
 * its own batch (steps are collective in the same way).  Each rank dedupes its batch's keys, sends each owner its keys,
 * and as owner creates and initialises the rows of the keys it received (values as on one GPU: they depend on the key
 * only, so a sharded run starts from what a single-GPU keyed run starts from).  Every rank then reads every owner's status
 * and fails the upload with the same message, naming the first failing owner (shard capacity exhausted, key table full);
 * keys inserted before keep their rows, and the slot is unusable until it is uploaded again, as on one GPU.  A rank whose
 * own arguments are refused still takes part with an empty, refused list, so its peers fail the upload at once.  The
 * waits of the upload are bounded (a few seconds): the ranks must enter it about together, else it fails as timed out.
 * cfg.max_nnz must be > 0: it bounds the entries of a batch and its distinct keys, and sizes the per-batch key tables.
 * Per rank, no communication: lctr_download_keys gives the rank's own local row -> key map; lctr_lookup_keys gives the
 * GLOBAL row of the keys this rank holds, -1 otherwise; lctr_upload_keyed_params takes from the arrays only the keys this
 * rank owns, in array order, so the same call on every rank seeds the sharded table; lctr_set_key_init must be called
 * with the same values on every rank.  lctr_device_bytes counts the shard's key table in the shard figure and the batch
 * dedupe table and inbox key arrays in the exchange figure.
 * An empty batch (0 rows or 0 entries) is a valid share of a collective upload: its rank posts empty lists.
 * Refused with world > 1: key_evict = 1 (at lctr_create) and insert = 0 uploads.  lctr_predict covers keyed slots uploaded
 * with insert = 1; a test set with unseen keys (lookup-only, insert = 0) still goes through a world = 1 context loaded with
 * lctr_load_checkpoint_shards. */

/* ---- the hot path --------------------------------------------------------------------------- */
/* One reference "batch": forward (gather + interaction [+ MLP]) -> loss -> backward scatter-add ->
 * per-coordinate update on the rows [row_begin,row_end) of the resident slot.
 *   FM : Train_FM_Algo::batchGradCompute + accumWVGrad + ApplyGrad   (train_fm_algo.cpp:63-126)
 *   FFM: Train_FFM_Algo::...                                         (train_ffm_algo.cpp:51-126)
 *   NFM: Train_NFM_Algo::batchGradCompute + ApplyGrad                (train_nfm_algo.cpp:56-169)
 * loss_sum / acc_cnt (may be NULL: then no host sync happens) receive the summed logloss and the
 * number of correct rows of this step, the quantities the reference prints per epoch. */
int lctr_train_step(lctr_ctx* ctx, int slot, int64_t row_begin, int64_t row_end, float* loss_sum, float* acc_cnt);
/* Per-row weights of the batch resident in `slot`: rows must equal the slot's row count; weight = NULL drops them.
 * Each weight must be finite and >= 0; a refused call writes nothing to the device.  Returns once `weight` may be reused.
 * THE RULE: a train step over rows [rb, re) of a weighted slot trains row r as if its whole per-row objective were
 * multiplied by w_r.
 *   - head: wherever a kernel forms d_r = p_r - y_r it uses fl(w_r (p_r - y_r)) (FM, FFM, the dense layers' output delta,
 *     the NFM and Wide&Deep wide terms);
 *   - L2: every term the reference adds per occurrence inside the row loop uses fl(w_r l2) for l2 (FM's l2 W, also inside
 *     the V multiplier, and l2 V; FFM's per-pair l2 c_ib; NFM's l2 W and l2 V; Wide&Deep's l2 W);
 *   - the dense layers' +-15 clip (fullyconnLayer.h:129-131) applies to the weighted deltas;
 *   - FFM's early return on d == 0 tests the weighted d, so a zero-weight row contributes nothing;
 *   - the updater's divisor stays cfg.minibatch_size, or the rows of the step;
 *   - loss_sum = sum w_r loss_r and acc_cnt = sum w_r [correct_r].
 * So w = 1 everywhere is bit for bit an unweighted step; a row of w = 0 is an absent row, except that its entries still
 * mark rows for change tracking; an integer w equals w copies of the row (fixed minibatch_size) up to re-association and
 * the clip.  Weights change gradients and statistics, not pCTR: lctr_score, lctr_predict, lctr_eval and lctr_eval_pred
 * ignore them; lctr_eval_weighted evaluates the slot with them.  They are batch data: any later upload into
 * the slot (lctr_upload_batch, lctr_upload_batch_keys with insert 0 or 1, lctr_upload_libffm, lctr_train_batch) drops
 * them, and checkpoints do not carry them.  Key admission removes entries, never rows, so weights stay aligned with the
 * rows of a keyed slot.  On several GPUs each rank weights its own rows (no collective).
 * Every model, deterministic mode and world trains weighted slots.  The statistics cost one more launch, and only when
 * loss_sum or acc_cnt is requested.  The streamed pipeline takes weights through lctr_train_batch_weighted_async. */
int lctr_set_row_weights(lctr_ctx* ctx, int slot, int64_t rows, const float* weight);
/* End-to-end convenience: upload_batch(slot 0) + train_step + result readback, host buffers in. */
int lctr_train_batch(lctr_ctx* ctx, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                     const uint16_t* field, const float* val, const int32_t* label, float* loss_sum,
                     float* acc_cnt);
/* Streamed training (host buffers in, results out, every step) with the copy of batch i+1 overlapping the kernels of
 * batch i: the batch is copied on a second stream into one of LCTR_PIPE_DEPTH pipeline slots (its slot map is built on a
 * third stream), the step is enqueued behind it and its (loss, acc) are copied back into a pinned ring; returns immediately
 * with a ticket.  At most LCTR_PIPE_DEPTH tickets may be outstanding; the host buffers must stay valid until the ticket has
 * been waited for.  lctr_wait blocks until that step's results are on the host.  (Depth 3: while step t computes, batch
 * t+1 has its slot map built and batch t+2 is on the copy engine.) */
#define LCTR_PIPE_DEPTH 3
int lctr_train_batch_async(lctr_ctx* ctx, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                           const uint16_t* field, const float* val, const int32_t* label, uint64_t* ticket);
/* lctr_train_batch_async plus one weight per row; weight = NULL is lctr_train_batch_async exactly.  The ticket's step
 * trains exactly as lctr_upload_batch + lctr_set_row_weights + lctr_train_step(0, rows) would (the rule of
 * lctr_set_row_weights), and lctr_wait returns its weighted statistics (sum w loss, sum w [correct]).  The weights are
 * checked on the host as lctr_set_row_weights checks them before anything is enqueued: a refused call issues no ticket and
 * leaves the pipeline usable.  `weight` must stay valid until the ticket has been waited for, like the other buffers.
 * Every model and world (each rank weights its own rows); on the captured-graph path (FM, cfg.deterministic 0 with a
 * compact gradient or 2, one GPU) a pipeline slot captures a weighted variant of its step graph the first time it streams a
 * weighted batch after an unweighted one, and the other way round, so a stream of one kind never recaptures. */
int lctr_train_batch_weighted_async(lctr_ctx* ctx, int64_t rows, int64_t nnz, const int64_t* row_ptr, const uint32_t* fid,
                                    const uint16_t* field, const float* val, const int32_t* label, const float* weight,
                                    uint64_t* ticket);
int lctr_wait(lctr_ctx* ctx, uint64_t ticket, float* loss_sum, float* acc_cnt);
/* Forward only on a resident slot; pctr (rows floats, host; may be NULL) receives sigmoid(pred).
 * quirk_sumvx_slot >= 0 reproduces FM_Predict's use of the TRAINING sumVX of the same row index
 * (predict/fm_predict.cpp:27-32); -1 computes the proper FM prediction.
 * Without the quirk, FM and Wide&Deep run the forward of lctr_score, so their pCTR equals lctr_score(ctx, slot, 0, rows)
 * bit for bit; Wide&Deep runs the rows in blocks as lctr_score does (a bounded dense scratch), and is refused with bf16
 * dense layers (cfg.mlp_precision = LCTR_MLP_BF16).  FFM predicts with the plain CTA-per-sample forward, or in the
 * reference's own pair loop order under cfg.deterministic = 1.
 * world > 1 (FM, FFM, Wide&Deep): a COLLECTIVE call, like a train step: every rank calls it for the same slot, in the same
 * order relative to the other collective calls, and receives the pCTR of its own rows.  The owners serve the rows from
 * their shards as they stand after every step issued before the call; no gradient moves and the step counter does not
 * advance.  FM and FFM run the single-GPU forward kernels on the pulled rows, in the same entry order, so the pCTR equals
 * that of a single-GPU context holding the merged parameters bit for bit.  A rank whose share of the test set is empty
 * takes part and receives 0 rows.  Dense slots and keyed slots uploaded with insert = 1 are supported.  A per-owner key
 * list that outgrew its inbox (cfg.max_nnz) fails the call with the overflow message.  Refused with world > 1:
 * quirk_sumvx_slot >= 0, and NFM (no NFM predictor exists on any world). */
int lctr_predict(lctr_ctx* ctx, int slot, int quirk_sumvx_slot, float* pctr);
/* The forward half of lctr_train_step(ctx, slot, row_begin, row_end, ...) alone: pctr[i] (row_end - row_begin floats,
 * host; may be NULL: then no copy and no synchronisation) is, bit for bit, the pCTR that train step would compute for row
 * row_begin + i from the current state -- for every model (FM, FFM, NFM, Wide&Deep), every gradient path the context
 * chose and both dense-layer precisions.  The same values are left in the slot's pred array, so lctr_eval,
 * lctr_download_pred and the global metrics of several GPUs work after a score as after a predict.
 * No side effects: no parameter, optimizer state, dense layer, bf16 weight copy, step counter or statistics entry changes
 * and no gradient is written; a train step after a score runs exactly as it would have without it.
 * Dropout masks apply as they stand, because that is the step's forward; a caller who wants a mask-free forward sets
 * all-ones masks with lctr_mlp_set_mask first.
 * NFM and Wide&Deep score the rows in blocks of at most max(65536, the largest dense batch the context has run) rows, so
 * the dense scratch stays bounded whatever the slot's size.
 * Slots as for lctr_predict: an invalid or stale keyed slot is refused; a lookup-only keyed slot (insert = 0, one GPU) is
 * scored with its unseen keys on the null row.  world > 1: a COLLECTIVE call like a train step (one pull-only round; every
 * rank calls it for the same slot in the same order and receives the pCTR of its own rows; an empty share takes part and
 * receives 0 rows).  NFM's replicated dense layers make each rank's pCTR that of one GPU holding the merged parameters;
 * Wide&Deep without a dense all-reduce uses the rank's own layers. */
int lctr_score(lctr_ctx* ctx, int slot, int64_t row_begin, int64_t row_end, float* pctr);
/* sumVX[rows*k] of a slot as left by the last forward over it (FM_Algo_Abst::sumVX, fm_algo_abst.h:145). */
int lctr_download_sumvx(lctr_ctx* ctx, int slot, float* sumVX);
/* per-row sigmoid(pred) of the last forward over the slot */
int lctr_download_pred(lctr_ctx* ctx, int slot, float* pred);

/* ---- MLP (Fully_Conn_Layer chain, fullyconnLayer.h) ------------------------------------------ */
/* The chain as a stand-alone operator -- what a DL_Algo_Abst subclass calls per minibatch (dl_algo_abst.h:46-49:
 * Predict / BP / applyBP) and what Layer_Base::forward / backward / applyBatchGradient do per sample
 * (layer_abst.h:45-67, fullyconnLayer.h:80-206), batched over `rows` samples, fp32 reference-order arithmetic:
 *   forward   x [rows][in0] (in0 = factor_cnt, or field_cnt * factor_cnt for Wide&Deep) -> out [rows] = the last layer's
 *             linear output (:116); hidden activations stay on the device for the backward.  out may be NULL.
 *   backward  dout [rows] = outputDelta of the last layer; clips to +-15 (:129-131), accumulates weightDelta / biasDelta
 *             (:165-179) in the fused dense-gradient buffer, returns the first layer's inputDelta in dx [rows][in0]
 *             (NULL to skip the copy).  Must follow a forward of the same row count.
 *   apply     applyBatchGradient (:194-197): Adagrad on bias then weights with divisor `minibatch`, deltas zeroed.
 *             With world > 1 the registered dense all-reduce runs first.  (Dropout masks: lctr_mlp_set_mask.) */
int lctr_mlp_forward(lctr_ctx* ctx, int64_t rows, const float* x, float* out);
int lctr_mlp_backward(lctr_ctx* ctx, int64_t rows, const float* dout, float* dx);
int lctr_mlp_apply(lctr_ctx* ctx, uint64_t minibatch);
/* layer l: weight [out][in] row-major (fullyconnLayer.h:211-216), bias[out], dropout mask[out] (1/0). */
int lctr_mlp_upload(lctr_ctx* ctx, int layer, const float* weight, const float* bias);
int lctr_mlp_download(lctr_ctx* ctx, int layer, float* weight, float* bias);
int lctr_mlp_set_mask(lctr_ctx* ctx, int layer, const float* mask);
/* Fully_Conn_Layer::weightDelta / biasDelta (fullyconnLayer.h:165-179) as they stand in the fused dense-gradient
 * buffer; zero after a step unless the process runs with LCTR_MLP_SKIP_UPDATE=1 (test hook: gradients are left in
 * place and the Adagrad update of the dense layers is skipped). */
int lctr_mlp_download_grad(lctr_ctx* ctx, int layer, float* dweight, float* dbias);

/* ---- multi-GPU (replaces distribut/ring_collect.h + pull.h/push.h; see DESIGN.md) ------------ */
/* Exchange of CUDA IPC handles is done by the caller's process group (torch.distributed / MPI):
 * export this rank's handle, gather them, import all peers'.  A rank shares one buffer, its exchange arena (flags, key
 * inboxes, parameter cache, gradient inboxes), so the blob is one cudaIpcMemHandle_t (64 B); size it with
 * lctr_ipc_export(ctx, NULL, 0, &n).  Import refuses a bytes_per_rank other than that size. */
int lctr_ipc_export(lctr_ctx* ctx, void* handles_out, size_t cap, size_t* bytes);
int lctr_ipc_import(lctr_ctx* ctx, const void* all_handles, size_t bytes_per_rank);
/* device memory of the context in bytes.  shard_bytes: the table shard W, V and the updater state s1 (+ s2 for the
 * two-state updaters), Fl (k + 1) floats each for FM / NFM, Fl (Fc k + 1) for FFM; + update_g of the same size on the
 * dense gradient path (FFM with deterministic 0 or 1, Wide&Deep, FM / NFM with deterministic = 0 and k outside
 * {4, 8, 16, 32}, NFM with deterministic = 2) and for the grouped FFM backward (deterministic = 2); + the touched map,
 * 1 B per row, on the dense path only; + the key table in keyed mode and 8 B per row of stamps with key_evict = 1; + the
 * host tier's index (12 B per slot) with cfg.key_host_rows > 0 (its rows are in host memory and not counted); + the key
 * admission sketch (16 * 2^log2_width B) while admission is on (lctr_set_key_admission); + the change map, 1 B per
 * row, while change tracking is on (lctr_track_changes).  The
 * compact (FM / NFM, deterministic = 0, k in {4, 8, 16, 32}) and the other feature-major paths hold no gradient per row.
 * Per-call scratch is not counted.  exchange_bytes (world > 1): the exchange arena, caches and inboxes -- owner-sharding
 * keeps it O(keys of a batch), not O(feature_cnt) */
int lctr_device_bytes(lctr_ctx* ctx, uint64_t* shard_bytes, uint64_t* exchange_bytes);
/* Data-parallel dense layers (world > 1, NFM): the per-rank weightDelta / biasDelta of the batch must be summed over
 * the ranks before the updater runs -- Worker_RingReduce::syncGradient (distribut/ring_collect.h:48-72) on the
 * BufferFusion of Fully_Conn_Layer::registerGradient (fullyconnLayer.h:69-75).  The library calls `fn` once per train
 * step, between the MLP backward and the dense Adagrad, with the fused gradient buffer and the CUDA stream the step
 * runs on; `fn` must enqueue an in-place SUM all-reduce on that stream (ncclAllReduce(buf, buf, n, ncclFloat, ncclSum,
 * comm, stream), or torch.distributed.all_reduce under that stream) and return 0.  Required when world > 1. */
typedef int (*lctr_allreduce_fn)(void* user, float* dev_buf, size_t n_floats, void* cuda_stream);
int lctr_set_dense_allreduce(lctr_ctx* ctx, lctr_allreduce_fn fn, void* user);
/* device pointer + element count of the fused dense-gradient buffer (the BufferFusion of
 * fullyconnLayer.h:69-75) for an external ncclAllReduce; 0 elements when the model has no MLP */
int lctr_dense_grad_buffer(lctr_ctx* ctx, void** dev_ptr, size_t* n_floats);

/* ---- host-side ingest (fm_algo_abst.h:70-107), bit-exact indexing ----------------------------- */
typedef struct lctr_dataset {
    int64_t rows, nnz, label_cnt;
    uint64_t feature_cnt, field_cnt;
    int64_t* row_ptr;
    uint32_t* fid;
    uint16_t* field;
    float* val;
    int32_t* label;
} lctr_dataset;
int lctr_load_libffm(const char* path, uint64_t field_cnt_in, uint64_t feature_cnt_in, lctr_dataset** out);
int lctr_free_dataset(lctr_dataset* d);
/* the same parser for keyed contexts: ids keep their full %zu width as uint64_t keys (no >= 2^32 rejection) */
typedef struct lctr_keyed_dataset {
    int64_t rows, nnz, label_cnt;
    uint64_t field_cnt;
    int64_t* row_ptr;
    uint64_t* key;
    uint16_t* field;
    float* val;
    int32_t* label;
} lctr_keyed_dataset;
int lctr_load_libffm_keys(const char* path, uint64_t field_cnt_in, lctr_keyed_dataset** out);
int lctr_free_keyed_dataset(lctr_keyed_dataset* d);
/* ---- libffm text parsed on the device ------------------------------------------------------------ */
/* Parses libffm text into `slot` on the GPU.  Split a text T at line boundaries into calls, LCTR_TEXT_BEGIN on the first
 * and LCTR_TEXT_END on the last: the slots of the calls, concatenated in call order, hold bit for bit what
 * lctr_load_libffm(T) + lctr_upload_batch give (row_ptr rebased per slot, ids, fields, value bits, the first `rows`
 * labels); keyed contexts: lctr_load_libffm_keys(T) + lctr_upload_batch_keys.  The reference parser's quirks carry across
 * calls: a line with a label but no features is dropped while its label is kept, shifting every later row's label; a
 * two-field token keeps the value of the token before it, also from an earlier line or call.  Lines that a token outside
 * the fast grammar (`digits:digits:plain-decimal`, <= 18 digits per id, label <= 9 digits) makes the device decline
 * are parsed by the host parser, in order (info->host_lines counts them).  A slot whose values are all exactly 1.0f
 * stores no val array, as lctr_upload_batch(val = NULL).
 * Errors name the line (counted from 1 at LCTR_TEXT_BEGIN): those lctr_load_libffm raises (an id >= 2^32 on a dense
 * context, a field >= 2^16), then those of the upload (field >= field_cnt for FFM / Wide&Deep, fid >= feature_cnt, the
 * reserved key).  After a failed call the parser state is unchanged and the slot holds no usable batch; keys inserted
 * before the failure keep their rows.  Text after the last '\n' is not consumed unless LCTR_TEXT_END is set.  The call
 * ends in a stream synchronise, so `text` (pinned memory copies fastest) may be reused when it returns.
 * Refused: world > 1, deterministic = 1 (its feature-major view is built on the host from host arrays), a slot out of
 * range, LCTR_TEXT_LOOKUP on a dense context.  Not covered: multi-GPU text uploads, the exact-order mode
 * (deterministic = 1), overlapping text uploads with steps (lctr_train_batch_async takes host CSR), FM_Predict's own
 * test-set loader quirks (its first feature dropped); the host shims keep lctr_load_libffm. */
#define LCTR_TEXT_BEGIN 1  /* this text starts a file: reset the state the reference's loop carries across lines */
#define LCTR_TEXT_END 2    /* this text ends the file: a last line without '\n' is parsed too */
#define LCTR_TEXT_LOOKUP 4 /* keyed contexts: insert = 0 (unseen keys -> the null row), as lctr_upload_batch_keys */
typedef struct lctr_text_info {
    int64_t rows, nnz;               /* what the slot now holds */
    int64_t lines, labels;           /* lines consumed; labels parsed from them */
    uint64_t feature_cnt, field_cnt; /* max id + 1, max field + 1 over the consumed lines (0 without entries) */
    int64_t host_lines;              /* lines the device grammar declined, parsed by the host parser */
    size_t consumed;                 /* bytes consumed: whole lines only */
} lctr_text_info;
int lctr_upload_libffm(lctr_ctx* ctx, int slot, const char* text, size_t bytes, int flags, lctr_text_info* info);
/* a slot read back: *rows / *nnz, row_ptr [rows + 1], fid [nnz] (rows of the key table on keyed contexts), field [nnz]
 * (zeros when the slot has none), val [nnz] (1.0f when it has no val array), label [rows] as the floats the slot holds.
 * Any pointer may be NULL; query the sizes first. */
int lctr_download_batch(lctr_ctx* ctx, int slot, int64_t* rows, int64_t* nnz, int64_t* row_ptr, uint32_t* fid,
                        uint16_t* field, float* val, float* label);
/* binary CSR cache of a parsed file: the sscanf-per-token parse is paid once (SURVEY.md 8f-2) */
int lctr_save_dataset_bin(const lctr_dataset* d, const char* path);
int lctr_load_dataset_bin(const char* path, lctr_dataset** out);

/* ---- test-set metrics on the device (SURVEY.md 8f-1) ----------------------------------------- */
/* Summed logloss and correct count of FM_Predict::Predict (predict/fm_predict.cpp:63-72) and AucEvaluator's AUC
 * (util/evaluator.h:51-104, 2^24 - 1 buckets, fp32 trapezoid walk from the top bucket) over the pCTR / label arrays
 * that lctr_predict left in `slot`.  The AUC is bit-identical to the reference's for the same pCTR values. */
int lctr_eval(lctr_ctx* ctx, int slot, float* loss_sum, int64_t* correct, float* auc);
/* The same three numbers, by the same kernels, over n host (pCTR, label) pairs in row order, on any context and any world:
 * the metrics of a whole test set gathered from the ranks of a sharded trainer (lightctr_b200.dist.eval_global) equal
 * lctr_eval on one GPU holding the concatenated batch, bit for bit.  lctr_eval keeps its meaning: the rows of this rank's
 * slot. */
int lctr_eval_pred(lctr_ctx* ctx, int64_t n, const float* pctr, const int32_t* label, float* loss_sum, int64_t* correct,
                   float* auc);
/* Weighted test-set metrics: lctr_eval over the slot's row weights (lctr_set_row_weights); refused when the slot has none
 * or no rows.  THE RULE, deterministic, and lctr_eval bit for bit when every w = 1:
 *   - loss: in row order, loss = (float)((double)loss + (double)w_i * term_i) over the rows with w_i != 0 (so no 0 * inf at
 *     p in {0, 1}), term_i being lctr_eval's term;
 *   - correct: sum w_i [correct_i] in double, in row order;
 *   - AUC: lctr_eval's bucket, (p * (2^24 - 1)) truncated.  With M = max w_i and 2^(E-1) <= M < 2^E, row i adds the
 *     integer q_i = rint(w_i 2^(32-E)) in [0, 2^32] to its bucket's u64 sum P_b (label 1) or N_b (otherwise), exact and
 *     independent of row order for n < 2^31; the fp32 trapezoid walk then runs over (fl32(P_b), fl32(N_b)) in place of the
 *     counts.  The walk runs in units of 2^(E-32), a power-of-two scale that commutes with each of its fp32 operations and
 *     that auc / totPos / totNeg divides out.  So integer weights give the AUC of the rows duplicated w times bit for bit,
 *     scaling every weight by 2^k changes no bit, and weights below 2^(E-33) round to q = 0 and leave the AUC alone (they
 *     still count in loss and correct).  M = 0 gives AUC 0.
 * The first weighted evaluation allocates 256 MB of histograms (not counted by lctr_device_bytes, like lctr_eval's 128 MB). */
int lctr_eval_weighted(lctr_ctx* ctx, int slot, float* loss_sum, double* correct, float* auc);
/* the same over n host (pCTR, label, weight) triples in row order, on any context and any world; each weight must be finite
 * and >= 0 (checked before anything is launched) */
int lctr_eval_pred_weighted(lctr_ctx* ctx, int64_t n, const float* pctr, const int32_t* label, const float* weight,
                            float* loss_sum, double* correct, float* auc);
/* test hook: overwrite the slot's pCTR array with host values */
int lctr_upload_pred(lctr_ctx* ctx, int slot, const float* pctr);

/* ---- checkpoint / resume (SURVEY.md 8f-3) ---------------------------------------------------- */
/* FM_Algo_Abst::saveModel (fm_algo_abst.h:109-135) writes W and V as text (kept in the host shims); these dump and
 * restore the complete trainer state in binary -- W, V, updater state (Adagrad accumulators | FTRL z, n | Adam m, v and
 * its call counter), dense layers with their Adagrad state and dropout masks, step counter -- so that a restored
 * trainer continues exactly where the saved one stopped.  The restoring ctx must have been created with the same cfg.
 * world > 1: every rank saves its own shard to its own path (no communication: the call synchronises the ctx stream, on
 * which every update of the shard runs), in a shard format of its own -- the rows it owns (local row l = global row
 * l * world + rank), its copy of the dense layers, and (keyed) its local row -> key map.  lctr_load_checkpoint loads the
 * file the same rank of the same world wrote (a single-GPU file is rank 0 of world 1) and refuses any other, naming both
 * ranks and worlds.  On any world, one GPU included: the file is checked (cfg, length, key section) before anything is
 * written, so a refused load changes nothing; keyed loads rebuild the key table, and every resident keyed slot becomes
 * stale (train_step refuses it until it is uploaded again), as after lctr_evict_keys; dense slots stay valid. */
int lctr_save_checkpoint(lctr_ctx* ctx, const char* path);
int lctr_load_checkpoint(lctr_ctx* ctx, const char* path);
/* The files of ONE save -- ranks 0..n-1 of a world-n run, or n = 1 and a single-GPU file -- into this context, whatever
 * its world (1 included).  Every rank takes the rows it owns under its own world; per rank, no communication.
 * Everything is checked before anything is written, and on failure the context is unchanged: every file has this cfg,
 * the set holds each rank 0..n-1 once, all files carry the same step and adam_iter, and when the world changes (n > 1)
 * the dense layers are bit-identical across the files (Wide&Deep without a dense all-reduce trains per-rank layers, which
 * no rule merges).  With the world unchanged it loads this rank's file as lctr_load_checkpoint does.
 * Dense tables: the row sections stream through a bounded device staging buffer.  Keyed tables: this rank's keys under
 * its world take rows 0..m-1 in source order (rank 0's rows ascending, then rank 1's, ...); m above the shard's capacity
 * fails naming the rank; rows past m return to the state lctr_create gives. */
int lctr_load_checkpoint_shards(lctr_ctx* ctx, int n, const char* const* paths);
/* Incremental checkpoints.  Change tracking for incremental saves: enable = 1 allocates a per-row change map over the
 * shard (1 B per local row, counted in shard_bytes while on) and clears it; enable = 0 frees it, and the context launches
 * exactly as before; either call forgets the parent.  A row's byte is set when a train step's entries name the row (on
 * several GPUs: when its owner serves it for a step), when lctr_upload_params / lctr_upload_opt_state / lctr_fill_params
 * write every row, and on keyed tables when a row is given a key (insert-upload, an owner's translation, restore from the
 * host tier, lctr_upload_keyed_params), is named by lctr_upload_keyed_params, or receives a row in lctr_evict_keys's move;
 * score, predict, eval and lookup-only uploads mark nothing.  With tracking on a train step costs one more launch (the
 * streamed pipeline's captured graphs are captured again with it).  The parent of a delta is the last file this context
 * saved or loaded while tracking was on (a full save, a delta, the last file of a chain, or an in-place
 * lctr_load_checkpoint); that save or load clears the map. */
int lctr_track_changes(lctr_ctx* ctx, int enable);
/* The rows changed since the parent save, plus the small state (dense layers, counters, and for keyed tables the key map,
 * stamps, host tier and admission sketch, whole), into `path` (layout: csrc/checkpoint.cu).  *rows_written may be NULL.
 * Refused, naming the reason, while tracking is off, before any parent exists, and after a resharding
 * lctr_load_checkpoint_shards until a full save. */
int lctr_save_checkpoint_delta(lctr_ctx* ctx, const char* path, uint64_t* rows_written);
/* paths[0]: a full file that lctr_load_checkpoint would accept on this context.  paths[1..n-1]: its deltas, in order.
 * Every file is checked first (cfg, rank and world, each delta's parent hash against the file before it, steps that never
 * decrease), so a refused chain changes nothing; then the full file loads in place and each delta's rows are applied.
 * Keyed slots become stale as after any keyed load.  A chain loads on the world that wrote it. */
int lctr_load_checkpoint_chain(lctr_ctx* ctx, int n, const char* const* paths);
/* the 64-bit hash that links a delta to its parent, of any file (host only, no device needed) */
int lctr_checkpoint_hash(const char* path, uint64_t* hash);

/* per-kernel device timing for bench.py's roofline: when enabled, every launch on the ctx stream is bracketed by
 * CUDA events; lctr_profile_read sums the elapsed ms and launch counts per kernel class
 * (0 fm_forward, 1 fm_backward(RED), 2 sparse apply, 3 ffm_fused, 4 fm_backward(CSC)+update, 5 mlp). */
int lctr_profile(lctr_ctx* ctx, int enable);
int lctr_profile_read(lctr_ctx* ctx, double* ms, int64_t* counts, int n, int reset);

/* introspection for tests / bench: number of kernels this library has launched on ctx so far */
int64_t lctr_launch_count(const lctr_ctx* ctx);
/* raw CUDA stream handle (cudaStream_t) of the ctx, for event timing on the launching stream */
void* lctr_stream(lctr_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* LIGHTCTR_B200_H */
