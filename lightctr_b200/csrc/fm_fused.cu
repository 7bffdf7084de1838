// lightctr_b200/csrc/fm_fused.cu -- host side of the order-free FM step (kernels: fm_fused.cuh).
//
// Train_FM_Algo::Train() per batch (train/train_fm_algo.cpp:44-57) for cfg.deterministic == 0 on one GPU:
//   upload   slot map of the batch (5 integer kernels on the upload stream: mark, compact, sample, hot, assign)
//   step     fm_fused_kernel (gather + interaction + loss + RED scatter into the batch-compact buffer)
//            apply_compact_kernel (updater over the compact buffer; re-zeroes it)
#include <algorithm>

#include "fm_fused.cuh"

namespace lctr {

static int fused_init(lctr_ctx* c) {
    if (c->fused) return 0;
    auto f = std::make_unique<FusedState>();  // the context's only once complete
    const bool compact = c->grad_path == GRAD_COMPACT;
    f->T = mark_rows(c->F);
    f->GS = compact ? grad_stride((int)c->cfg.factor_cnt) : 0;
    const size_t n_hot = (size_t)kHotMax * kHotRep * f->GS;
    if (f->mark.alloc(128 * f->T + 512) || f->slot_of.alloc(c->F) || f->Ghot.alloc(n_hot) || f->d_opt.alloc(1)) return 1;
    LCTR_CUDA(cudaMemsetAsync(f->mark, 0, 128 * f->T + 512, c->stream));
    if (compact) LCTR_CUDA(cudaMemsetAsync(f->Ghot, 0, n_hot * sizeof(float), c->stream));
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    c->fused = std::move(f);
    return 0;
}

// capacity for a batch of `nnz` entries in slot s (per-slot key set + per-context gradient buffer)
int fused_reserve(lctr_ctx* c, Slot& s, int64_t nnz) {
    if (fused_init(c)) return 1;
    FusedState* f = c->fused.get();
    const int64_t need_u = std::min<int64_t>(std::max<int64_t>(nnz, 1), (int64_t)c->F);
    if (nnz > s.cap_ent_slot) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        const int64_t cap = std::max<int64_t>(nnz, s.cap_ent_slot + s.cap_ent_slot / 2);
        s.cap_ent_slot = 0;
        if (alloc_group(sized(s.ent_slot, (size_t)(cap + 64)), sized(s.ent_pslot, c->cfg.world > 1 ? (size_t)(cap + 64) : 0)))
            return 1;
        s.cap_ent_slot = cap;
    }
    if (need_u > s.cap_uniq || !s.hot_of) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        const int64_t cap = std::min<int64_t>(std::max<int64_t>(need_u, s.cap_uniq + s.cap_uniq / 2), (int64_t)c->F);
        s.cap_uniq = 0;
        if (alloc_group(sized(s.uniq, (size_t)(cap + 64)), sized(s.hot_of, (size_t)(cap + 64)))) return 1;
        if ((!s.n_uniq && s.n_uniq.alloc(1)) || (!s.n_hot && s.n_hot.alloc(1)) || (!s.hot_slot && s.hot_slot.alloc(kHotMax)))
            return 1;
        s.cap_uniq = cap;
    }
    if ((size_t)s.cap_uniq > f->cnt_cap) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        if (c->copy_stream) LCTR_CUDA(cudaStreamSynchronize(c->copy_stream));
        f->cnt_cap = 0;
        if (alloc_group(sized(f->cnt, (size_t)(s.cap_uniq + 64)))) return 1;
        LCTR_CUDA(cudaMemset(f->cnt, 0, (size_t)(s.cap_uniq + 64) * sizeof(unsigned int)));
        f->cnt_cap = (size_t)s.cap_uniq;
    }
    // gradient rows: one per slot; on several GPUs one per exchange row (dist.cu re-indexes the entries)
    const size_t g_rows = c->cfg.world > 1 ? c->dist_rows : (size_t)s.cap_uniq;
    if (c->grad_path == GRAD_COMPACT && g_rows > f->G_rows) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        f->G_rows = 0;
        if (alloc_group(sized(f->G, (g_rows + 64) * f->GS))) return 1;
        LCTR_CUDA(cudaMemset(f->G, 0, (g_rows + 64) * f->GS * sizeof(float)));
        f->G_rows = g_rows;
    }
    return 0;
}

// slot map of the batch held by slot s, on stream st.  hdr != nullptr (graph capture): {rows, nnz} are read from device
// memory and the grids are sized for the slot's capacities.  An empty batch (0 rows or 0 entries) gets an empty map and no
// kernel.
int fused_build_slot(lctr_ctx* c, Slot& s, cudaStream_t st, const int64_t* hdr, int64_t rows_cap, int64_t nnz_cap) {
    FusedState* f = c->fused.get();
    s.fused_valid = false;
    const int SM = c->sm_count;
    LCTR_CUDA(cudaMemsetAsync(s.n_uniq, 0, sizeof(unsigned int), st));
    LCTR_CUDA(cudaMemsetAsync(s.n_hot, 0, sizeof(unsigned int), st));
    if (rows_cap <= 0 || nnz_cap <= 0) {
        s.fused_valid = true;
        return 0;
    }
    const unsigned mkg = (unsigned)std::max<int64_t>(1, std::min<int64_t>((nnz_cap + 2047) / 2048, (int64_t)SM * 4));
    if (launch(c, {mkg, 256, 0, st}, slotmap_mark_kernel, s.fid, hdr, nnz_cap, f->mark, f->T)) return 1;
    const size_t ntiles = (128 * f->T + 511) / 512;
    const unsigned cg = (unsigned)std::max<size_t>(1, std::min<size_t>((ntiles + 7) / 8, (size_t)SM * 8));
    if (launch(c, {cg, 256, 0, st}, slotmap_compact_kernel, f->mark, f->T, s.uniq, s.n_uniq, f->slot_of)) return 1;
    const bool hot = c->grad_path == GRAD_COMPACT;  // replica rows only exist for the fused FM / NFM kernels
    if (hot) {
        const unsigned sg = (unsigned)std::min<int64_t>(((int64_t)kHotSampleRows * 128 + 255) / 256, (int64_t)SM * 8);
        if (launch(c, {sg, 256, 0, st}, slotmap_sample_kernel, s.row_ptr, s.fid, hdr, rows_cap, f->slot_of, f->cnt) ||
            launch(c, {(unsigned)SM * 2, 256, 0, st}, slotmap_hot_kernel, f->cnt, s.n_uniq, hdr, rows_cap, s.hot_of, s.hot_slot,
                   s.n_hot))
            return 1;
    }
    const unsigned ag = (unsigned)std::max<int64_t>(1, std::min<int64_t>((nnz_cap + 255) / 256, (int64_t)SM * 8));
    if (launch(c, {ag, 256, 0, st}, slotmap_assign_kernel, s.fid, hdr, nnz_cap, f->slot_of, hot ? s.hot_of.get() : nullptr, s.ent_slot,
               c->cfg.world > 1 ? s.ent_pslot.get() : nullptr))
        return 1;
    s.fused_valid = true;
    return 0;
}

int launch_slotmap_compact(lctr_ctx* c, uint8_t* mark, size_t T, uint32_t* uniq, unsigned int* n_uniq, cudaStream_t st) {
    const size_t ntiles = (128 * T + 511) / 512;
    const unsigned cg = (unsigned)std::max<size_t>(1, std::min<size_t>((ntiles + 7) / 8, (size_t)c->sm_count * 8));
    return launch(c, {cg, 256, 0, st}, slotmap_compact_kernel, mark, T, uniq, n_uniq, nullptr);
}

template <int K>
static int fused_go(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int stats, double* out_slot, const int64_t* hdr, int mode) {
    FusedState* f = c->fused.get();
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((re - rb + 3) / 4, (int64_t)c->sm_count * 4));
    // one GPU: parameters straight from the tables (index = fid); several: from the batch-compact cache the owners filled
    // (index = plain slot), after the owners' "rows delivered" flags of this step (dist.cu)
    const bool multi = c->cfg.world > 1;
    const unsigned long long* wf = nullptr;
    int nw = 0;
    unsigned long long ep = 0;
    if (multi && mode != 3) dist_wait_info(c, &wf, &nw, &ep);
    // dependent launches: MODE 1 on several GPUs behind my own serve kernel (it polls the owners' flags at its head); the NFM
    // backward on one GPU behind the dense kernels in front of it (it requests its batch data before their end)
    const bool dependent = mode == 1 ? multi : mode == 3 && !multi;
    // mode 1: FM forward + backward;  2: NFM forward (z, wide part);  3: NFM backward from dz.  Weighted rows: the weighted
    // instances of the modes that form a head (the NFM forward has none)
    auto kern = by_value<1, 2, 3>(mode, [&](auto m) {
        return by_flags([&](auto hv, auto rw) { return fm_fused_kernel<K, hv, m, false, 4, rw && m != 2>; }, s.has_val, s.has_rw);
    });
    return launch(c, {grid, 128, 0, c->stream, dependent}, kern, s.row_ptr, multi ? s.ent_pslot : s.fid, s.ent_slot, s.val, s.label, c->cW, c->cV, s.pred, s.sumvx, nullptr, f->G,
                  f->Ghot, f->GS, c->cfg.l2_reg, rb, re, hdr, c->stat_partial, c->stat_done, out_slot, stats, wf, nw, ep,
                  mode == 2 ? c->z : mode == 3 ? c->dz.get() : nullptr, mode == 2 ? s.wide.get() : nullptr, row_weights(s));
}

// the launchers below are built for FM k in {4, 8, 16, 32} and take 32 for any other k
static int launch_fused_mode(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats, const int64_t* hdr, double* out_slot_override,
                             int mode, int prof_id) {
    if (re - rb <= 0) return 0;
    LCTR_CHECK(s.fused_valid, "fused FM step on a slot without its slot map (uploaded before the context supported it?)");
    double* out_slot = out_slot_override ? out_slot_override : c->stats + 2 * (c->step % kStatRing);
    ProfScope prof(c, prof_id);
    return by_value<4, 8, 16, 32>((int)c->cfg.factor_cnt,
                                  [&](auto K) { return fused_go<K>(c, s, rb, re, stats ? 1 : 0, out_slot, hdr, mode); });
}

// forward + RED backward of rows [rb, re) of the slot.  hdr != nullptr: `re` only sizes the grid, the row count comes
// from hdr[0].
int launch_fm_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats, const int64_t* hdr, double* out_slot_override) {
    return launch_fused_mode(c, s, rb, re, stats, hdr, out_slot_override, 1, PROF_FM_FUSED);
}
// NFM embedding side around the dense layers: forward fills c->z (bi-interaction) and the slot's wide part; backward reads
// c->dz (the first dense layer's input delta) and the predictions the loss kernel left in the slot
int launch_nfm_forward_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    return launch_fused_mode(c, s, rb, re, false, nullptr, nullptr, 2, PROF_FM_FWD);
}
int launch_nfm_backward_fused(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    return launch_fused_mode(c, s, rb, re, false, nullptr, nullptr, 3, PROF_FM_FUSED);
}

// order-free forward alone (predictions, sumVX, statistics): the throughput predictor of cfg.deterministic == 0 contexts and
// the kernel bench.py times for the gather roofline.  Needs no slot map on one GPU.  Several GPUs (a pull-only round of
// lctr_predict): the same kernel on the batch-compact cache (index = plain slot, read in the same entry order, so the
// pCTR equals a single-GPU context's bit for bit), launched dependent on my serve kernel like the MODE 1 step, polling
// the owners' "rows delivered" flags at its head.
template <int K>
static int fwd_tree_go(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, int stats, double* out_slot) {
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((re - rb + 3) / 4, (int64_t)c->sm_count * 4));
    const bool multi = c->cfg.world > 1;
    const unsigned long long* wf = nullptr;
    int nw = 0;
    unsigned long long ep = 0;
    if (multi) dist_wait_info(c, &wf, &nw, &ep);
    const uint32_t* fid = multi ? s.ent_pslot : s.fid;
    return launch(c, {grid, 128, 0, c->stream, multi}, s.has_val ? fm_fused_kernel<K, true, 0, true> : fm_fused_kernel<K, false, 0, true>,
                  s.row_ptr, fid, fid, s.val, s.label, multi ? c->cW : c->W, multi ? c->cV : c->V, s.pred, s.sumvx, nullptr, nullptr,
                  nullptr, grad_stride(K), c->cfg.l2_reg, rb, re, nullptr, c->stat_partial, c->stat_done, out_slot, stats, wf, nw, ep,
                  nullptr, nullptr, nullptr);
}
int launch_fm_forward_tree(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, bool stats) {
    if (re - rb <= 0) return 0;
    double* out_slot = c->stats + 2 * (c->step % kStatRing);
    ProfScope prof(c, PROF_FM_FWD);
    return by_value<4, 8, 16, 32>((int)c->cfg.factor_cnt,
                                  [&](auto K) { return fwd_tree_go<K>(c, s, rb, re, stats ? 1 : 0, out_slot); });
}

template <int K>
static int apply_go(lctr_ctx* c, Slot& s, const OptParams& P, const OptParams* P_dev) {
    FusedState* f = c->fused.get();
    const int main_blocks = c->sm_count * 3;
    const unsigned grid = (unsigned)(main_blocks + kHotMax / 8);  // + one warp per possible hot slot
    // Programmatic dependent launch behind the gradient kernel (one GPU): the updater's CTAs start as the gradient kernel's
    // retire, request their ids, parameter and state rows, and only then wait for its completion.
    return launch(c, {grid, 256, 0, c->stream, c->cfg.world == 1}, by_opt(P.opt, [](auto o) { return apply_compact_kernel<K, o.value>; }), s.uniq, s.n_uniq, f->G,
                  s.hot_of, s.hot_slot, s.n_hot, f->Ghot, f->GS, main_blocks, c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V, P, P_dev);
}

// updater over the slot's key set.  P_host (optional) / dP: parameters already staged in device memory (graph launches).
int launch_apply_compact(lctr_ctx* c, Slot& s, int64_t rows_in_step, const OptParams* P_host, const OptParams* dP) {
    const OptParams P = P_host ? *P_host : make_opt_params(c, rows_in_step);
    ProfScope prof(c, PROF_APPLY_COMPACT);
    return by_value<4, 8, 16, 32>((int)c->cfg.factor_cnt, [&](auto K) { return apply_go<K>(c, s, P, dP); });
}

void fused_opt_params(lctr_ctx* c, int64_t rows, void* out) { *reinterpret_cast<OptParams*>(out) = make_opt_params(c, rows); }
void* fused_dev_opt(lctr_ctx* c) { return c->fused ? c->fused->d_opt.get() : nullptr; }

}  // namespace lctr
