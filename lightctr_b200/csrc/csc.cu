// lightctr_b200/csrc/csc.cu -- feature-major view of a batch built ON THE DEVICE at upload, and the
// atomic-free backward + fused updater that consumes it (cfg.deterministic == 2, the streamed-batch default).
//
// Why: the RED scatter of fm.cu issues 17 fp32 atomic adds per nnz and is bound by the L2 atomic units.  Grouping the entries by feature id turns the scatter
// into a segmented reduction: each unique fid's gradient is summed in registers by one lane group and the
// updater is applied on the spot -- no update_g traffic, no atomics on floats, no touched map, no apply pass.
// The grouping depends only on the batch (not on the parameters), so it runs on the upload stream and overlaps
// the previous step's kernels.
//
// Build (5 small kernels, integer work only):
//   count      cnt[fid] += 1 for every entry                                  (RED.ADD.U32)
//   tile_reduce / tile_scan / tile_write: exclusive scan of cnt over the id space in 512-id tiles -> entry
//              offset of every present fid, the segment list (seg_fid, seg_ptr) in ascending fid order, and two
//              work lists: short segments (<= 8 entries) and long ones
//   fill       every entry takes a slot of its fid's segment with an atomic cursor (cnt counts back down to 0)
// The order of the entries INSIDE a segment is therefore arbitrary; the backward accumulates each segment in
// double precision, so the fp32-rounded gradient does not depend on that order (the sum of <= 2^16 fp32 terms is
// carried with 2^-53 relative error per add; a different order changes the fp32 result only if the exact sum lies
// within ~1e-12 ulp of a rounding boundary).  Reference semantics of the accumulated expression:
// train_fm_algo.cpp:101-116 (see fm.cu); the host-built view of cfg.deterministic == 1 keeps the reference's exact
// ascending-row fp32 order instead.
#include <string.h>

#include <algorithm>
#include <vector>

#include "opt.cuh"

namespace lctr {

constexpr int kShortMax = 8;     // segments up to this many entries: one lane group each
constexpr int kTaskLen = 256;    // longer segments are cut into warp tasks of this many entries

// also widens the int32 labels that were copied into `label_i32` (the reference compares a float target)
__global__ void csc_count_kernel(const uint32_t* __restrict__ fid, int64_t nnz_arg, unsigned int* __restrict__ cnt,
                                 const int32_t* __restrict__ label_i32, float* __restrict__ label, int64_t rows_arg,
                                 const int64_t* __restrict__ hdr) {
    const int64_t nnz = hdr ? hdr[1] : nnz_arg, rows = hdr ? hdr[0] : rows_arg;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i < nnz; i += nt) atomicAdd(&cnt[fid[i]], 1u);
    if (label_i32)
        for (int64_t i = t0; i < rows; i += nt) label[i] = (float)label_i32[i];
}

// per 512-id tile: (sum of counts, number of present ids)
__global__ void __launch_bounds__(256)
csc_tile_reduce_kernel(const unsigned int* __restrict__ cnt, size_t F, uint2* __restrict__ tile_sum) {
    const int lane = threadIdx.x & 31;
    const size_t warp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
    const size_t ntiles = (F + 511) / 512;
    for (size_t tile = warp; tile < ntiles; tile += nwarps) {
        const size_t base = tile * 512 + (size_t)lane * 16;
        unsigned s = 0, p = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const unsigned v = base + i < F ? cnt[base + i] : 0u;
            s += v;
            p += v != 0u;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(kFull, s, o);
            p += __shfl_xor_sync(kFull, p, o);
        }
        if (lane == 0) tile_sum[tile] = make_uint2(s, p);
    }
}

// exclusive scan of the tile sums by ONE block; also publishes the totals, the sentinel seg_ptr[nseg] and re-arms
// the work-list counters
__global__ void __launch_bounds__(1024)
csc_tile_scan_kernel(const uint2* __restrict__ tile_sum, size_t ntiles, uint2* __restrict__ tile_off,
                     unsigned int* __restrict__ totals /* [0]=nnz [1]=nseg [2]=n_short [3]=n_long */,
                     int64_t* __restrict__ seg_ptr) {
    __shared__ uint2 sh[1024];
    __shared__ uint2 carry;
    if (threadIdx.x == 0) carry = make_uint2(0, 0);
    __syncthreads();
    for (size_t b = 0; b < ntiles; b += 1024) {
        const size_t i = b + threadIdx.x;
        uint2 v = i < ntiles ? tile_sum[i] : make_uint2(0, 0);
        sh[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {  // Hillis-Steele inclusive scan
            uint2 t = make_uint2(0, 0);
            if ((int)threadIdx.x >= o) t = sh[threadIdx.x - o];
            __syncthreads();
            sh[threadIdx.x].x += t.x;
            sh[threadIdx.x].y += t.y;
            __syncthreads();
        }
        const uint2 incl = sh[threadIdx.x];
        const uint2 c = carry;
        if (i < ntiles) tile_off[i] = make_uint2(c.x + incl.x - v.x, c.y + incl.y - v.y);
        __syncthreads();
        if (threadIdx.x == 1023) carry = make_uint2(c.x + incl.x, c.y + incl.y);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        totals[0] = carry.x;
        totals[1] = carry.y;
        totals[2] = 0;
        totals[3] = 0;
        seg_ptr[carry.y] = (int64_t)carry.x;  // sentinel: seg_ptr[n_segs] = nnz
    }
}

// per tile: offsets of the present ids, segment list, work lists
__global__ void __launch_bounds__(256)
csc_tile_write_kernel(const unsigned int* __restrict__ cnt, size_t F, const uint2* __restrict__ tile_off,
                      unsigned int* __restrict__ off, uint32_t* __restrict__ seg_fid, int64_t* __restrict__ seg_ptr,
                      uint32_t* __restrict__ short_list, uint2* __restrict__ long_list,
                      unsigned int* __restrict__ totals) {
    const int lane = threadIdx.x & 31;
    const size_t warp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
    const size_t ntiles = (F + 511) / 512;
    for (size_t tile = warp; tile < ntiles; tile += nwarps) {
        const size_t base = tile * 512 + (size_t)lane * 16;
        unsigned v[16];
        unsigned s = 0, p = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            v[i] = base + i < F ? cnt[base + i] : 0u;
            s += v[i];
            p += v[i] != 0u;
        }
        unsigned is = s, ip = p;  // inclusive warp scans
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned ts = __shfl_up_sync(kFull, is, o), tp = __shfl_up_sync(kFull, ip, o);
            if (lane >= o) { is += ts; ip += tp; }
        }
        const unsigned tot_p = __shfl_sync(kFull, ip, 31);
        if (tot_p == 0) continue;
        const uint2 to = tile_off[tile];
        unsigned eoff = to.x + is - s, sidx = to.y + ip - p;
        unsigned nshort = 0, nlong = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (v[i]) { nshort += v[i] <= kShortMax; nlong += v[i] > kShortMax ? (v[i] + kTaskLen - 1) / kTaskLen : 0; }
        }
        // work-list slots: warp-aggregated reservation
        unsigned ish = nshort, ilo = nlong;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned a = __shfl_up_sync(kFull, ish, o), b = __shfl_up_sync(kFull, ilo, o);
            if (lane >= o) { ish += a; ilo += b; }
        }
        unsigned bs = 0, bl = 0;
        if (lane == 31) {
            if (ish) bs = atomicAdd(&totals[2], ish);
            if (ilo) bl = atomicAdd(&totals[3], ilo);
        }
        bs = __shfl_sync(kFull, bs, 31) + ish - nshort;
        bl = __shfl_sync(kFull, bl, 31) + ilo - nlong;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (!v[i]) continue;
            const size_t f = base + i;
            off[f] = eoff;
            seg_fid[sidx] = (uint32_t)f;
            seg_ptr[sidx] = (int64_t)eoff;
            if (v[i] <= kShortMax) short_list[bs++] = sidx;
            else for (unsigned t0 = 0; t0 < v[i]; t0 += kTaskLen) long_list[bl++] = make_uint2(sidx, t0);
            eoff += v[i];
            sidx++;
        }
    }
}

// every entry claims a slot of its fid's segment; cnt returns to zero (ready for the next upload)
__global__ void __launch_bounds__(256)
csc_fill_kernel(const int64_t* __restrict__ row_ptr, const uint32_t* __restrict__ fid, const float* __restrict__ val,
                int64_t rows_arg, const unsigned int* __restrict__ off, unsigned int* __restrict__ cnt,
                uint32_t* __restrict__ ent_row, float* __restrict__ ent_x, const int64_t* __restrict__ hdr,
                const uint16_t* __restrict__ field, uint16_t* __restrict__ ent_field) {
    const int64_t rows = hdr ? hdr[0] : rows_arg;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = warp; r < rows; r += nwarps) {
        const int64_t b = row_ptr[r], e = row_ptr[r + 1];
        for (int64_t i = b + lane; i < e; i += 32) {
            const uint32_t f = fid[i];
            const unsigned left = atomicSub(&cnt[f], 1u);
            const unsigned pos = off[f] + left - 1u;
            ent_row[pos] = (uint32_t)r;
            if (val) ent_x[pos] = val[i];
            if (field) ent_field[pos] = field[i];  // FFM: the entry's field travels with it
        }
    }
}

// ------------------------------------------------------------------------------------------------
// backward + fused updater, K % 4 == 0: a V row is LPR = K/4 lanes x float4
// ------------------------------------------------------------------------------------------------
struct CscView {
    const int64_t* seg_ptr;
    const uint32_t* seg_fid;
    const uint32_t* ent_row;
    const float* ent_x;
    const float* label;
    const float* pred;
    const float* sumvx;
};
struct ParamView {
    float *W, *V, *s1W, *s1V, *s2W, *s2V;
};

template <int K>
__device__ __forceinline__ void accumulate(double (&u)[4], double& gws, const float4& s, float d, float x, float w,
                                           const float4& v, float l2) {
    const float gw = d * x + l2 * w;      // train_fm_algo.cpp:108
    gws += (double)gw;                    // :109
    // (sumVX - x*V) * gradW  and  + L2 * V   (:112-115); each product is rounded to fp32 like the reference's
    u[0] += (double)((s.x + v.x * (-x)) * gw) + (double)(v.x * l2);
    u[1] += (double)((s.y + v.y * (-x)) * gw) + (double)(v.y * l2);
    u[2] += (double)((s.z + v.z * (-x)) * gw) + (double)(v.z * l2);
    u[3] += (double)((s.w + v.w * (-x)) * gw) + (double)(v.w * l2);
}

template <int K>
__device__ __forceinline__ void apply_update(const ParamView& T, const OptParams& P, uint32_t f, int q, float w, float4 v,
                                             const double (&u)[4], double gws) {
    const bool two = opt_two_states(P.opt);
    if (q == 0) {
        float ww = w, a = T.s1W[f], b2 = two ? T.s2W[f] : 0.f;
        update_one(P, P.corrW, ww, (float)gws, a, b2);
        T.W[f] = ww; T.s1W[f] = a;
        if (two) T.s2W[f] = b2;
    }
    const size_t o = (size_t)f * K + 4 * q;
    float4 a = *reinterpret_cast<const float4*>(T.s1V + o);
    float4 b2 = two ? *reinterpret_cast<const float4*>(T.s2V + o) : make_float4(0.f, 0.f, 0.f, 0.f);
    update_one(P, P.corrV, v.x, (float)u[0], a.x, b2.x);
    update_one(P, P.corrV, v.y, (float)u[1], a.y, b2.y);
    update_one(P, P.corrV, v.z, (float)u[2], a.z, b2.z);
    update_one(P, P.corrV, v.w, (float)u[3], a.w, b2.w);
    *reinterpret_cast<float4*>(T.V + o) = v;
    *reinterpret_cast<float4*>(T.s1V + o) = a;
    if (two) *reinterpret_cast<float4*>(T.s2V + o) = b2;
}

// SHORT segments (<= 8 entries): one LPR-lane group per segment.  The <= 8 row indices are fetched with one load
// per lane, then all <= 8 sumVX / pred / label gathers are in flight together: two memory round trips per segment.
template <int K, bool HAS_VAL>
__global__ void __launch_bounds__(256)
csc_backward_short_kernel(const uint32_t* __restrict__ work, const unsigned int* __restrict__ totals, CscView C,
                          ParamView T, float l2, OptParams P_arg, const OptParams* __restrict__ dP) {
    const OptParams P = dP ? *dP : P_arg;
    constexpr int LPR = K / 4;
    constexpr int G = 32 / LPR;
    constexpr int PER = kShortMax / LPR;  // row indices fetched per lane
    const int lane = threadIdx.x & 31;
    const int q = lane % LPR, g = lane / LPR;
    const unsigned nwork = totals[2];
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    for (unsigned w0 = warp * G; w0 < nwork; w0 += nwarps * G) {
        const unsigned wi = w0 + g;
        const bool sv = wi < nwork;
        const uint32_t seg = sv ? work[wi] : 0u;
        const int64_t eb = sv ? C.seg_ptr[seg] : 0;
        const int n = sv ? (int)(C.seg_ptr[seg + 1] - eb) : 0;
        const uint32_t f = sv ? C.seg_fid[seg] : 0u;
        uint32_t rows[PER];
        float xs[PER];
#pragma unroll
        for (int p = 0; p < PER; p++) {
            const int e = p * LPR + q;
            rows[p] = e < n ? __ldg(C.ent_row + eb + e) : 0u;
            xs[p] = HAS_VAL ? (e < n ? __ldg(C.ent_x + eb + e) : 0.f) : 1.f;
        }
        const float w = sv ? T.W[f] : 0.f;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (sv) v = *reinterpret_cast<const float4*>(T.V + (size_t)f * K + 4 * q);
        float4 s[kShortMax];
        float d[kShortMax], x[kShortMax];
#pragma unroll
        for (int e = 0; e < kShortMax; e++) {
            const uint32_t r = __shfl_sync(kFull, rows[e / LPR], (e % LPR), LPR);
            x[e] = HAS_VAL ? __shfl_sync(kFull, xs[e / LPR], (e % LPR), LPR) : 1.f;
            s[e] = ldg_f4(C.sumvx + (size_t)r * K + 4 * q);       // row 0 for e >= n: valid address, masked below
            d[e] = __ldg(C.pred + r) - __ldg(C.label + r);
        }
        double u[4] = {0.0, 0.0, 0.0, 0.0}, gws = 0.0;
#pragma unroll
        for (int e = 0; e < kShortMax; e++)
            if (e < n) accumulate<K>(u, gws, s[e], d[e], x[e], w, v, l2);
        if (sv) apply_update<K>(T, P, f, q, w, v, u, gws);
    }
}

// LONG segments: warp tasks of <= kTaskLen entries; 32/LPR entry slots work in parallel, 32 row indices per chunk are
// fetched with one coalesced load, the next chunk's indices are prefetched while the current one is reduced.
// Segments of more than kTaskLen entries are covered by several tasks whose partial sums meet in acc[seg] (double
// atomics); the task that arrives last applies the update and re-arms the accumulator.
template <int K, bool HAS_VAL>
__global__ void __launch_bounds__(256)
csc_backward_long_kernel(const uint2* __restrict__ work, const unsigned int* __restrict__ totals, CscView C, ParamView T,
                         double* __restrict__ acc, unsigned int* __restrict__ arrived, float l2, OptParams P_arg,
                         const OptParams* __restrict__ dP) {
    const OptParams P = dP ? *dP : P_arg;
    constexpr int LPR = K / 4;
    constexpr int G = 32 / LPR;
    const int lane = threadIdx.x & 31;
    const int q = lane % LPR, g = lane / LPR;
    const unsigned nwork = totals[3];
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    for (unsigned wi = warp; wi < nwork; wi += nwarps) {
        const uint2 task = work[wi];
        const uint32_t seg = task.x;
        const int64_t eb0 = C.seg_ptr[seg];
        const int ntot = (int)(C.seg_ptr[seg + 1] - eb0);
        const int64_t eb = eb0 + task.y;
        const int n = min(kTaskLen, ntot - (int)task.y);
        const uint32_t f = C.seg_fid[seg];
        const float w = T.W[f];
        const float4 v = *reinterpret_cast<const float4*>(T.V + (size_t)f * K + 4 * q);
        double u[4] = {0.0, 0.0, 0.0, 0.0}, gws = 0.0;
        uint32_t rows_n = lane < n ? __ldg(C.ent_row + eb + lane) : 0u;
        float xs_n = HAS_VAL ? (lane < n ? __ldg(C.ent_x + eb + lane) : 0.f) : 1.f;
        for (int base = 0; base < n; base += 32) {
            const uint32_t rows = rows_n;
            const float xs = xs_n;
            const int nb = base + 32 + lane;
            rows_n = nb < n ? __ldg(C.ent_row + eb + nb) : 0u;
            if (HAS_VAL) xs_n = nb < n ? __ldg(C.ent_x + eb + nb) : 0.f;
            float4 s[LPR];
            float d[LPR], x[LPR];
#pragma unroll
            for (int j = 0; j < LPR; j++) {
                const int e = j * G + g;
                const uint32_t r = __shfl_sync(kFull, rows, e);
                x[j] = HAS_VAL ? __shfl_sync(kFull, xs, e) : 1.f;
                s[j] = ldg_f4(C.sumvx + (size_t)r * K + 4 * q);
                d[j] = __ldg(C.pred + r) - __ldg(C.label + r);
            }
#pragma unroll
            for (int j = 0; j < LPR; j++)
                if (base + j * G + g < n) accumulate<K>(u, gws, s[j], d[j], x[j], w, v, l2);
        }
        // fold the G entry slots (lanes with the same q) in a fixed tree
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < 4; c++) u[c] += __shfl_xor_sync(kFull, u[c], o);
            gws += __shfl_xor_sync(kFull, gws, o);
        }
        if (ntot <= kTaskLen) {
            if (g == 0) apply_update<K>(T, P, f, q, w, v, u, gws);
            continue;
        }
        // multi-task segment: meet in the accumulator
        double* a = acc + (size_t)seg * (K + 1);
        if (g == 0) {
#pragma unroll
            for (int c = 0; c < 4; c++) atomicAdd(a + 4 * q + c, u[c]);
            if (q == 0) atomicAdd(a + K, gws);
        }
        __threadfence();
        unsigned last = 0;
        if (lane == 0) {
            const unsigned ntasks = (unsigned)((ntot + kTaskLen - 1) / kTaskLen);
            last = atomicAdd(&arrived[seg], 1u) == ntasks - 1 ? 1u : 0u;
        }
        last = __shfl_sync(kFull, last, 0);
        if (last) {
            __threadfence();
            if (g == 0) {
                double uu[4];
#pragma unroll
                for (int c = 0; c < 4; c++) { uu[c] = atomicAdd(a + 4 * q + c, 0.0); }
                const double gg = atomicAdd(a + K, 0.0);
                apply_update<K>(T, P, f, q, w, v, uu, gg);
#pragma unroll
                for (int c = 0; c < 4; c++) a[4 * q + c] = 0.0;
                if (q == 0) { a[K] = 0.0; arrived[seg] = 0u; }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct CscScratch {
    Buf<unsigned int> cnt;   // F, all zero between builds
    Buf<unsigned int> off;   // F
    Buf<uint2> tile_sum;
    Buf<uint2> tile_off;
    size_t ntiles = 0;
};
void drop(CscScratch* p) { delete p; }

static int scratch_get(lctr_ctx* c, CscScratch** out) {
    if (!c->csc_scratch) {
        Owned<CscScratch> s(new CscScratch());  // the context's only once complete
        s->ntiles = (c->F + 511) / 512;
        if (s->cnt.alloc(c->F + 512) || s->off.alloc(c->F + 512) || s->tile_sum.alloc(s->ntiles + 1) ||
            s->tile_off.alloc(s->ntiles + 1))
            return 1;
        LCTR_CUDA(cudaMemset(s->cnt, 0, (c->F + 512) * sizeof(unsigned int)));
        c->csc_scratch = std::move(s);
    }
    *out = c->csc_scratch.get();
    return 0;
}

// (re)allocate the per-slot arrays of the view for up to `max_nnz` entries
int csc_reserve(lctr_ctx* c, Slot& s, int64_t max_nnz) {
    CscScratch* sc0;
    if (scratch_get(c, &sc0)) return 1;  // never allocate inside a stream capture
    const int64_t max_segs = std::min<int64_t>(max_nnz, (int64_t)c->F);
    if (max_segs > s.cap_segs || !s.short_list) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        const int64_t cap = std::max<int64_t>(max_segs, s.cap_segs + s.cap_segs / 2);
        const size_t n = (size_t)(cap + 1);
        // FM: per-segment double accumulators; FFM meets in update_g instead (ffm_grouped.cu)
        const size_t na = c->cfg.model == LCTR_MODEL_FFM ? 8 : n * (c->cfg.factor_cnt + 1);
        s.cap_segs = 0; s.cap_long = 0;
        if (alloc_group(sized(s.seg_ptr, n), sized(s.seg_fid, n), sized(s.short_list, n), sized(s.long_list, (size_t)max_nnz / 8 + n),
                        sized(s.csc_acc, na), sized(s.csc_arrived, n)) ||
            (!s.csc_totals && s.csc_totals.alloc(4)))
            return 1;
        LCTR_CUDA(cudaMemset(s.csc_acc, 0, na * sizeof(double)));
        LCTR_CUDA(cudaMemset(s.csc_arrived, 0, n * sizeof(unsigned int)));
        s.cap_segs = cap;
        s.cap_long = max_nnz;
    } else if (max_nnz > s.cap_long) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        s.cap_long = 0;
        if (alloc_group(sized(s.long_list, (size_t)(max_nnz / 8 + s.cap_segs + 1)))) return 1;
        s.cap_long = max_nnz;
    }
    if (max_nnz > s.cap_ent) {
        LCTR_CUDA(cudaStreamSynchronize(c->stream));
        const int64_t cap = std::max<int64_t>(max_nnz, s.cap_ent + s.cap_ent / 2);
        const size_t n = (size_t)(cap + 32);
        s.cap_ent = 0;
        if (alloc_group(sized(s.ent_row, n), sized(s.ent_x, n), sized(s.ent_field, c->cfg.model == LCTR_MODEL_FFM ? n : 0))) return 1;
        s.cap_ent = cap;
    }
    return 0;
}

// build the feature-major view of the whole slot on stream `st`.  label_i32 != nullptr: the int32 labels just
// copied there are widened into s.label by the first kernel.  hdr != nullptr (graph capture): sizes come from the
// device header {rows, nnz}; `rows_cap` / `nnz_cap` then only size the grids.
int csc_build_device(lctr_ctx* c, Slot& s, cudaStream_t st, const int32_t* label_i32, const int64_t* hdr,
                     int64_t rows_cap, int64_t nnz_cap) {
    s.dev_csc = false;
    const int64_t nnz = hdr ? nnz_cap : s.nnz, rows = hdr ? rows_cap : s.rows;
    if (nnz == 0) return 0;
    CscScratch* sc;
    if (scratch_get(c, &sc)) return 1;
    if (!hdr && csc_reserve(c, s, nnz)) return 1;
    const unsigned g1 = (unsigned)std::min<int64_t>((nnz + 255) / 256, (int64_t)c->sm_count * 8);
    const unsigned gt = (unsigned)std::min<size_t>((sc->ntiles + 7) / 8, (size_t)c->sm_count * 8);
    const unsigned gf = (unsigned)std::min<int64_t>((rows + 7) / 8, (int64_t)c->sm_count * 8);
    if (launch(c, {std::max(g1, 1u), 256, 0, st}, csc_count_kernel, s.fid, s.nnz, sc->cnt, label_i32, s.label, s.rows, hdr) ||
        launch(c, {std::max(gt, 1u), 256, 0, st}, csc_tile_reduce_kernel, sc->cnt, c->F, sc->tile_sum) ||
        launch(c, {1, 1024, 0, st}, csc_tile_scan_kernel, sc->tile_sum, sc->ntiles, sc->tile_off, s.csc_totals, s.seg_ptr) ||
        launch(c, {std::max(gt, 1u), 256, 0, st}, csc_tile_write_kernel, sc->cnt, c->F, sc->tile_off, sc->off, s.seg_fid, s.seg_ptr,
               s.short_list, s.long_list, s.csc_totals) ||
        launch(c, {std::max(gf, 1u), 256, 0, st}, csc_fill_kernel, s.row_ptr, s.fid, s.has_val ? s.val.get() : nullptr, s.rows, sc->off,
               sc->cnt, s.ent_row, s.ent_x, hdr, s.has_field && s.ent_field ? s.field.get() : nullptr, s.ent_field))  // FFM only
        return 1;
    s.dev_csc = true;
    s.csc_block = 0;
    return 0;
}

template <int K>
static int bwd_go(lctr_ctx* c, Slot& s, const OptParams& P, const OptParams* dP) {
    const unsigned grid = (unsigned)c->sm_count * 4;
    const CscView C{s.seg_ptr, s.seg_fid, s.ent_row, s.ent_x, s.label, s.pred, s.sumvx};
    const ParamView T{c->W, c->V, c->s1W, c->s1V, c->s2W, c->s2V};
    const uint2* longs = s.long_list;
    return launch(c, {grid, 256, 0, c->stream}, s.has_val ? csc_backward_long_kernel<K, true> : csc_backward_long_kernel<K, false>,
                  longs, s.csc_totals, C, T, s.csc_acc, s.csc_arrived, c->cfg.l2_reg, P, dP) ||
           launch(c, {grid, 256, 0, c->stream}, s.has_val ? csc_backward_short_kernel<K, true> : csc_backward_short_kernel<K, false>,
                  s.short_list, s.csc_totals, C, T, c->cfg.l2_reg, P, dP);
}

// dP != nullptr (graph capture): the updater parameters are read from device memory at run time
int launch_fm_backward_devcsc_ex(lctr_ctx* c, Slot& s, int64_t rb, int64_t re, const OptParams* P_host, const void* dP) {
    LCTR_CHECK(s.dev_csc, "slot has no device-built feature-major view");
    LCTR_CHECK(rb == 0 && (dP || re == s.rows), "the device-built view covers whole slots only (rows [%lld,%lld) of %lld)",
               (long long)rb, (long long)re, (long long)s.rows);
    const int k = (int)c->cfg.factor_cnt;
    OptParams P;
    if (P_host) P = *P_host; else P = make_opt_params(c, re - rb);
    ProfScope prof(c, PROF_FM_BWD_CSC);
    const OptParams* d = reinterpret_cast<const OptParams*>(dP);
    switch (k) {
        case 4: return bwd_go<4>(c, s, P, d);
        case 8: return bwd_go<8>(c, s, P, d);
        case 16: return bwd_go<16>(c, s, P, d);
        case 32: return bwd_go<32>(c, s, P, d);
        default:
            set_error("device feature-major backward is built for k in {4, 8, 16, 32} (k=%d)", k);
            return 1;
    }
}

int launch_fm_backward_devcsc(lctr_ctx* c, Slot& s, int64_t rb, int64_t re) {
    return launch_fm_backward_devcsc_ex(c, s, rb, re, nullptr, nullptr);
}

// host-side snapshot of the updater parameters for a step of `rows` rows (advances the Adam call counter)
void csc_opt_params(lctr_ctx* c, int64_t rows, void* out) {
    const OptParams P = make_opt_params(c, rows);
    memcpy(out, &P, sizeof(P));
}

bool csc_device_supported(const lctr_ctx* c) {
    const int k = (int)c->cfg.factor_cnt;
    if (c->cfg.model == LCTR_MODEL_FFM) return ffm_grouped_supported(c);
    return c->cfg.model == LCTR_MODEL_FM && (k == 4 || k == 8 || k == 16 || k == 32);
}

}  // namespace lctr
