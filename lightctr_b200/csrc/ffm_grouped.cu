// lightctr_b200/csrc/ffm_grouped.cu -- feature-grouped (atomic-free) FFM backward with the updater fused in.
//
// Why: the fused kernel of ffm.cu scatters every entry's Fc*k-float gradient row with REDs and is bound by the L2
// reduction rate of fp32 adds.  The gradient row of an
// entry i of sample s (field a = fld_i) is
//     g_i[b] = d_s x_i ( T_s[a][b] - [b == a] x_i R_i[a] ) + l2 c_{i,b} R_i[b]        (ffm.cu header; reference
//     train_ffm_algo.cpp:81-118), c_{i,b} = cnt_s[b] - [b == a],
// i.e. a function of the sample's field-pair tile T_s and of the feature's OWN row R_i only.  So the forward kernel
// stores T_s once per sample (as [a][b][k]: the slice an entry needs is one contiguous Fc*k row), and this kernel
// walks the batch feature-major (the device-built view of csc.cu): one warp per feature segment sums its entries'
// rows in registers -- plain coalesced 16 B loads, no atomics -- and applies the updater on the spot (no update_g
// traffic, no touched map, no apply pass).  Segments longer than kTaskLen are cut into tasks that meet in update_g with
// a handful of REDs; the last task to arrive applies the update.
// Sums are carried in double so that the fp32-rounded result does not depend on the (arbitrary) order of the entries
// inside a segment.
#include <algorithm>

#include "opt.cuh"

namespace lctr {

constexpr int kFfmTaskLen = 256;  // must equal csc.cu's kTaskLen (the long work list is cut with it)
constexpr int kFfmU = 8;          // entries in flight per warp

struct FfmView {
    const int64_t* seg_ptr;
    const uint32_t* seg_fid;
    const uint32_t* ent_row;
    const float* ent_x;
    const uint16_t* ent_field;
    const float* label;
    const float* pred;
    const float* Tbuf;
    const uint16_t* cntbuf;
    const uint32_t* short_list;
    const uint2* long_list;
    const unsigned int* totals;  // [2] = n_short, [3] = n_long
};
struct FfmParams {
    float *W, *V, *s1W, *s1V, *s2W, *s2V;  // FUSE: the tables and updater state; else W / V are the read-only row cache
    float *gW, *gV;                        // update_g (meeting point of multi-task segments; the output when !FUSE)
    unsigned int* arrived;
};

// Work item = (task, slot block i): warp (task, i) owns float4 slots [32 i, 32 i + 32) of the feature's row and walks
// the task's entries on its own -- the NS = ceil(A/32) warps of a task never synchronise (the entry metadata they all
// read is 10 B per entry against a 16 B x 32 lane tile slice).  One float4 slot per lane keeps the register count low
// enough for 16 warps per SM with kFfmU = 8 entries (8 x 512 B per warp) in flight.
// RW: the slot's row weights rw scale each entry's head d and its per-pair L2 coefficient by its row's weight
template <bool HAS_VAL, bool FUSE, bool RW = false>
__global__ void __launch_bounds__(128, 4)
ffm_backward_grouped_kernel(FfmView C, FfmParams T, int Fc, int k, int NS, float l2, OptParams P, const float* __restrict__ rw) {
    const int lane = threadIdx.x & 31;
    const int A = Fc * k / 4, PPF = k / 4;
    const size_t rowlen = (size_t)Fc * k;
    const unsigned n_long = C.totals[3], n_short = C.totals[2];
    const unsigned ntask = n_long + n_short;
    const unsigned nitem = ntask * (unsigned)NS;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);

    // the work item, its segment bounds and feature id of the NEXT item are fetched while the current one is reduced:
    // two of the four dependent round trips of a (typically 1-8 entry) task leave the critical path
    auto fetch = [&](unsigned it, uint32_t& seg, int& t0, int64_t& eb0, int& ntot, uint32_t& f) {
        if (it >= nitem) { seg = 0; t0 = 0; eb0 = 0; ntot = 0; f = 0; return; }
        const unsigned wi = it / (unsigned)NS;
        if (wi < n_long) { const uint2 task = C.long_list[wi]; seg = task.x; t0 = (int)task.y; }
        else { seg = C.short_list[wi - n_long]; t0 = 0; }
        eb0 = C.seg_ptr[seg];
        ntot = (int)(C.seg_ptr[seg + 1] - eb0);
        f = C.seg_fid[seg];
    };
    uint32_t nseg, nf; int nt0, nntot; int64_t neb0;
    fetch(warp, nseg, nt0, neb0, nntot, nf);
    for (unsigned it = warp; it < nitem; it += nwarps) {
        const uint32_t seg = nseg, f = nf;
        const int t0 = nt0, ntot = nntot;
        const int64_t eb0 = neb0;
        fetch(it + nwarps, nseg, nt0, neb0, nntot, nf);
        const int blk = (int)(it % (unsigned)NS);
        const int q = lane + 32 * blk;  // my float4 slot of the row
        const bool own = q < A;
        const int fq = own ? q / PPF : 0;
        const int64_t eb = eb0 + t0;
        const int n = min(kFfmTaskLen, ntot - t0);
        const bool single = ntot <= kFfmTaskLen;
        const size_t o = (size_t)f * rowlen + 4 * q;
        const float w = T.W[f];
        const float4 v = own ? *reinterpret_cast<const float4*>(T.V + o) : make_float4(0.f, 0.f, 0.f, 0.f);
        // updater state of a single-task row is needed at the end: issue its loads now
        const bool two = opt_two_states(P.opt);
        float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), b2 = a1;
        if (FUSE && single && own) {
            a1 = *reinterpret_cast<const float4*>(T.s1V + o);
            if (two) b2 = *reinterpret_cast<const float4*>(T.s2V + o);
        }
        double u0 = 0.0, u1 = 0.0, u2 = 0.0, u3 = 0.0, gws = 0.0;
        int nvalid = 0;
        // entry metadata of up to 32 entries, one per lane; the next chunk is prefetched
        auto meta = [&](int base, uint32_t& r, int& a, float& x) {
            const bool has = base + lane < n;
            r = has ? __ldg(C.ent_row + eb + base + lane) : 0u;
            a = has ? (int)__ldg(C.ent_field + eb + base + lane) : 0;
            x = HAS_VAL ? (has ? __ldg(C.ent_x + eb + base + lane) : 0.f) : 1.f;
        };
        uint32_t r_n; int a_n; float x_n;
        meta(0, r_n, a_n, x_n);
        for (int base = 0; base < n; base += 32) {
            const uint32_t my_r = r_n;
            const int my_a = a_n;
            const float my_x = x_n;
            if (base + 32 < n) meta(base + 32, r_n, a_n, x_n);
            const float my_d = base + lane < n ? row_head<RW>(__ldg(C.pred + my_r), __ldg(C.label + my_r), rw, my_r) : 0.f;
            const float my_l2 = RW && base + lane < n ? row_l2<RW>(l2, rw, my_r) : l2;
            const int m = min(32, n - base);
            for (int j0 = 0; j0 < m; j0 += kFfmU) {
                float4 tt[kFfmU];
                int cb[kFfmU], a[kFfmU];
                float x[kFfmU], d[kFfmU], l2e[kFfmU];
#pragma unroll
                for (int uu = 0; uu < kFfmU; uu++) {
                    const int j = min(j0 + uu, 31);
                    const uint32_t r = __shfl_sync(kFull, my_r, j);
                    a[uu] = __shfl_sync(kFull, my_a, j);
                    x[uu] = HAS_VAL ? __shfl_sync(kFull, my_x, j) : 1.f;
                    d[uu] = __shfl_sync(kFull, my_d, j);
                    if (RW) l2e[uu] = __shfl_sync(kFull, my_l2, j);
                    if (j0 + uu >= m) d[uu] = 0.f;  // train_ffm_algo.cpp:81-83: d == 0 contributes nothing at all
                    // unconditional loads (row 0 / stale tiles are valid addresses): not behind the pred/label gather
                    if (own) {
                        tt[uu] = ldg_f4(C.Tbuf + ((size_t)r * Fc + a[uu]) * rowlen + 4 * q);
                        cb[uu] = (int)__ldg(C.cntbuf + (size_t)r * Fc + fq);
                    } else {
                        tt[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
                        cb[uu] = 0;
                    }
                }
#pragma unroll
                for (int uu = 0; uu < kFfmU; uu++) {
                    if (d[uu] == 0.f) continue;
                    nvalid++;
                    const float sx = d[uu] * x[uu];
                    const float l2u = RW ? l2e[uu] : l2;
                    gws += (double)(sx + l2u * w);  // train_ffm_algo.cpp:98
                    const bool self = fq == a[uu];
                    const int c_ib = cb[uu] - (self ? 1 : 0);
                    if (c_ib <= 0) continue;
                    const float lc = l2u * (float)c_ib;
                    float4 tv = tt[uu];
                    if (self) { tv.x -= x[uu] * v.x; tv.y -= x[uu] * v.y; tv.z -= x[uu] * v.z; tv.w -= x[uu] * v.w; }
                    u0 += (double)(sx * tv.x + lc * v.x);
                    u1 += (double)(sx * tv.y + lc * v.y);
                    u2 += (double)(sx * tv.z + lc * v.z);
                    u3 += (double)(sx * tv.w + lc * v.w);
                }
            }
        }
        if (single && FUSE) {
            if (!nvalid) continue;
            if (blk == 0 && lane == 0) {
                float ww = w, aw = T.s1W[f], bw = two ? T.s2W[f] : 0.f;
                update_one(P, P.corrW, ww, (float)gws, aw, bw);
                T.W[f] = ww; T.s1W[f] = aw;
                if (two) T.s2W[f] = bw;
            }
            if (own) {
                float4 vv = v;
                update_one(P, P.corrV, vv.x, (float)u0, a1.x, b2.x);
                update_one(P, P.corrV, vv.y, (float)u1, a1.y, b2.y);
                update_one(P, P.corrV, vv.z, (float)u2, a1.z, b2.z);
                update_one(P, P.corrV, vv.w, (float)u3, a1.w, b2.w);
                *reinterpret_cast<float4*>(T.V + o) = vv;
                *reinterpret_cast<float4*>(T.s1V + o) = a1;
                if (two) *reinterpret_cast<float4*>(T.s2V + o) = b2;
            }
            continue;
        }
        // partial sums meet in update_g (the only output when !FUSE: the multi-GPU push reads it)
        if (nvalid) {
            if (own) red_add_v4(T.gV + o, make_float4((float)u0, (float)u1, (float)u2, (float)u3));
            if (blk == 0 && lane == 0) red_add_f32(T.gW + f, (float)gws);
        }
        if (!FUSE) continue;
        __threadfence();
        unsigned last = 0;
        if (lane == 0) {
            const unsigned narr = (unsigned)((ntot + kFfmTaskLen - 1) / kFfmTaskLen) * (unsigned)NS;
            last = atomicAdd(&T.arrived[seg], 1u) == narr - 1 ? 1u : 0u;
        }
        last = __shfl_sync(kFull, last, 0);
        if (!last) continue;
        // the last of the segment's (task, block) items applies the update to the whole row and re-arms the meeting point
        __threadfence();
        if (lane == 0) {
            const float g = __ldcg(T.gW + f);
            __stcg(T.gW + f, 0.f);
            T.arrived[seg] = 0u;
            float ww = w, aw = T.s1W[f], bw = two ? T.s2W[f] : 0.f;
            update_one(P, P.corrW, ww, g, aw, bw);
            T.W[f] = ww; T.s1W[f] = aw;
            if (two) T.s2W[f] = bw;
        }
        for (int qq = lane; qq < A; qq += 32) {
            const size_t oo = (size_t)f * rowlen + 4 * qq;
            const float4 g = __ldcg(reinterpret_cast<const float4*>(T.gV + oo));
            __stcg(reinterpret_cast<float4*>(T.gV + oo), make_float4(0.f, 0.f, 0.f, 0.f));
            float4 vv = *reinterpret_cast<const float4*>(T.V + oo);
            float4 s1 = *reinterpret_cast<const float4*>(T.s1V + oo);
            float4 s2 = two ? *reinterpret_cast<const float4*>(T.s2V + oo) : make_float4(0.f, 0.f, 0.f, 0.f);
            update_one(P, P.corrV, vv.x, g.x, s1.x, s2.x);
            update_one(P, P.corrV, vv.y, g.y, s1.y, s2.y);
            update_one(P, P.corrV, vv.z, g.z, s1.z, s2.z);
            update_one(P, P.corrV, vv.w, g.w, s1.w, s2.w);
            *reinterpret_cast<float4*>(T.V + oo) = vv;
            *reinterpret_cast<float4*>(T.s1V + oo) = s1;
            if (two) *reinterpret_cast<float4*>(T.s2V + oo) = s2;
        }
    }
}

bool ffm_grouped_supported(const lctr_ctx* c) {
    const int k = (int)c->cfg.factor_cnt, Fc = (int)c->cfg.field_cnt;
    return c->cfg.model == LCTR_MODEL_FFM && k % 4 == 0 && Fc * k / 4 <= 128;
}

// tile buffer for `rows` samples: rows * Fc * Fc * k floats (C5: 3.2 GB at 65536 rows) + the per-field counts
int ffm_grouped_reserve(lctr_ctx* c, int64_t rows) {
    if ((size_t)rows <= c->ffm_T_rows) return 0;
    LCTR_CUDA(cudaStreamSynchronize(c->stream));
    c->ffm_T_rows = 0;
    const size_t Fc = c->cfg.field_cnt, k = c->cfg.factor_cnt;
    if (alloc_group(sized(c->ffm_T, (size_t)rows * Fc * Fc * k), sized(c->ffm_cnt, (size_t)rows * Fc))) return 1;
    c->ffm_T_rows = (size_t)rows;
    return 0;
}

int launch_ffm_backward_grouped(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    LCTR_CHECK(s.dev_csc && s.ent_field, "slot has no device-built feature-major view with fields");
    LCTR_CHECK(rb == 0 && re == s.rows, "the device-built view covers whole slots only (rows [%lld,%lld) of %lld)",
               (long long)rb, (long long)re, (long long)s.rows);
    const int k = (int)c->cfg.factor_cnt, Fc = (int)c->cfg.field_cnt;
    const int A = Fc * k / 4, NS = (A + 31) / 32;
    const OptParams P = make_opt_params(c, re - rb);
    const FfmView C{s.seg_ptr, s.seg_fid, s.ent_row, s.ent_x, s.ent_field, s.label, s.pred, c->ffm_T, c->ffm_cnt,
                    s.short_list, s.long_list, s.csc_totals};
    const bool fuse = c->cfg.world == 1;
    const FfmParams T{fuse ? c->W : c->cW, fuse ? c->V : c->cV, c->s1W, c->s1V, c->s2W, c->s2V, c->cgW, c->cgV, s.csc_arrived};
    const unsigned grid = (unsigned)c->sm_count * 8;
    ProfScope prof(c, PROF_FM_BWD_CSC);
    LCTR_CHECK(NS >= 1 && NS <= 4, "grouped FFM backward: row of %d floats exceeds 512", Fc * k);
    auto kern = by_flags([](auto hv, auto fu, auto rw) { return ffm_backward_grouped_kernel<hv, fu, rw>; }, s.has_val, fuse, s.has_rw);
    return launch(c, {grid, 128, 0, c->stream}, kern, C, T, Fc, k, NS, c->cfg.l2_reg, P, row_weights(s));
}

}  // namespace lctr
