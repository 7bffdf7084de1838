// lightctr_b200/csrc/opt.cu -- sparse per-coordinate updaters (Adagrad / FTRL / Adam), sm_90a.
//
// Reference: AdagradUpdater_Num::update (util/gradientUpdater.h:139-150), FTRLUpdater::update
// (:252-273), AdamUpdater_Num::update (util/momentumUpdater.h:187-210), applied by
// Train_*_Algo::ApplyGrad as a DENSE sweep over all F*(rowlen+1) coordinates.  Every updater
// skips coordinates whose batch gradient is exactly 0, and a gradient is only ever produced
// for the fids present in the batch (L2 terms are added inside the nnz loops), so visiting only
// the touched fids is exactly equivalent (SURVEY.md 8a-7).  The backward kernels mark
// touched[fid] = 1 (plain byte store, idempotent); this kernel scans the byte map 16 B per lane,
// pops set entries 32 at a time and updates G = 32/LPR rows concurrently, LPR lanes per row,
// each lane owning VEC-float slices q, q+LPR, ...  It also zeroes the gradient and the mark, which
// replaces the reference's memset(grad) (gradientUpdater.h:149).
#include <algorithm>
#include <vector>

#include "opt.cuh"

namespace lctr {

// Stage A: scan the touched byte map (16 marks per lane, 512 per warp tile), clear it, and append the set
// positions to a global list of fids (one warp-aggregated atomicAdd per non-empty tile).  Decoupling the
// scan from the update balances the update work: the small-vocabulary fields at the low end of the id
// space are dense (every mark set) while the tail is ~5 % dense.
__global__ void __launch_bounds__(256)
compact_touched_kernel(uint8_t* __restrict__ touched, size_t F, uint32_t* __restrict__ list,
                       unsigned int* __restrict__ n_list) {
    const int lane = threadIdx.x & 31;
    const size_t warp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
    const size_t ntiles = (F + 511) / 512;
    for (size_t tile = warp; tile < ntiles; tile += nwarps) {
        const size_t base = tile * 512 + (size_t)lane * 16;
        uint4 m = make_uint4(0, 0, 0, 0);
        if (base + 16 <= F) {
            m = *reinterpret_cast<const uint4*>(touched + base);
        } else if (base < F) {
            unsigned char tmp[16];
            for (int i = 0; i < 16; i++) tmp[i] = base + i < F ? touched[base + i] : 0;
            m = *reinterpret_cast<uint4*>(tmp);
        }
        const bool any = (m.x | m.y | m.z | m.w) != 0;
        if (!__any_sync(kFull, any)) continue;
        unsigned bits = 0;
        {
            const unsigned wv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int b = 0; b < 4; b++)
                    if ((wv[i] >> (8 * b)) & 0xffu) bits |= 1u << (i * 4 + b);
        }
        if (any) {  // clear the marks (memset(grad) analogue, gradientUpdater.h:149)
            if (base + 16 <= F) *reinterpret_cast<uint4*>(touched + base) = make_uint4(0, 0, 0, 0);
            else for (int i = 0; i < 16 && base + i < F; i++) touched[base + i] = 0;
        }
        const int mycnt = __popc(bits);
        int incl = mycnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += t;
        }
        const int total = __shfl_sync(kFull, incl, 31);
        unsigned int gbase = 0;
        if (lane == 31) gbase = atomicAdd(n_list, (unsigned int)total);
        gbase = __shfl_sync(kFull, gbase, 31);
        unsigned int pos = gbase + (unsigned int)(incl - mycnt);
        while (bits) {
            const int bit = __ffs(bits) - 1;
            bits &= bits - 1;
            list[pos++] = (uint32_t)(base + bit);
        }
    }
}

// Stage B: walk the list G*U rows at a time.  Slice = VEC contiguous floats of a row; a row has rowlen/VEC
// slices spread over LPR lanes, SPL slices per lane (slice index = q + i*LPR).  ALL loads of a batch
// (gradient, weight, state of U rows per lane group) are issued before the first update is computed, so one
// HBM/L2 round trip covers 32/LPR*U rows.  The last block re-arms the list counter.
// OPT: the updater as a compile-time constant (-1 = decide at run time).  With the five updaters' double-precision
// divisions and square roots inlined U * (SPL * VEC + 1) times the run-time version is a very long kernel with
// one resident CTA per SM whose top stall is instruction-cache misses.  The VEC = 4 instances are therefore specialised per updater.
template <int LPR, int VEC, int SPL, int U, int OPT>
__global__ void __launch_bounds__(256, (OPT >= 0 ? 2 : 1))
apply_kernel(const uint32_t* __restrict__ list, unsigned int* __restrict__ n_list, unsigned int* __restrict__ done,
             int rowlen, float* __restrict__ W, float* __restrict__ V,
             float* __restrict__ gW, float* __restrict__ gV, float* __restrict__ s1W, float* __restrict__ s1V,
             float* __restrict__ s2W, float* __restrict__ s2V, OptParams P_in) {
    OptParams P = P_in;
    if (OPT >= 0) P.opt = OPT;  // folds every `P.opt ==` test of update_one
    constexpr int G = 32 / LPR;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int q = lane % LPR, g = lane / LPR;
    const unsigned warp = blockIdx.x * (blockDim.x >> 5) + wid;
    const unsigned nwarps = gridDim.x * (blockDim.x >> 5);
    const bool two_state = opt_two_states(P.opt);
    const int slices = rowlen / VEC;
    const unsigned total = *reinterpret_cast<volatile unsigned int*>(n_list);
    {
        for (unsigned b0 = warp * (G * U); b0 < total; b0 += nwarps * (G * U)) {
            size_t f[U];
            bool ok[U];
            float gw_[U], w_[U], a_[U], b_[U];
            float gv[U][SPL][VEC], wv[U][SPL][VEC], s1[U][SPL][VEC], s2[U][SPL][VEC];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const unsigned idx = b0 + u * G + g;
                ok[u] = idx < total;
                f[u] = ok[u] ? __ldg(list + idx) : 0;
                if (ok[u] && q == 0) {
                    gw_[u] = gW[f[u]]; w_[u] = W[f[u]]; a_[u] = s1W[f[u]];
                    b_[u] = two_state ? s2W[f[u]] : 0.f;
                }
                const size_t ro = f[u] * (size_t)rowlen;
#pragma unroll
                for (int i = 0; i < SPL; i++) {
                    const int sl = q + i * LPR;
                    const bool on = ok[u] && sl < slices;
                    const size_t o = ro + (size_t)sl * VEC;
                    if (VEC == 4) {
                        float4 t0 = make_float4(0, 0, 0, 0), t1 = t0, t2 = t0, t3 = t0;
                        if (on) {
                            t0 = *reinterpret_cast<const float4*>(gV + o);
                            t1 = *reinterpret_cast<const float4*>(V + o);
                            t2 = *reinterpret_cast<const float4*>(s1V + o);
                            if (two_state) t3 = *reinterpret_cast<const float4*>(s2V + o);
                        }
                        gv[u][i][0] = t0.x; gv[u][i][1 % VEC] = t0.y; gv[u][i][2 % VEC] = t0.z; gv[u][i][3 % VEC] = t0.w;
                        wv[u][i][0] = t1.x; wv[u][i][1 % VEC] = t1.y; wv[u][i][2 % VEC] = t1.z; wv[u][i][3 % VEC] = t1.w;
                        s1[u][i][0] = t2.x; s1[u][i][1 % VEC] = t2.y; s1[u][i][2 % VEC] = t2.z; s1[u][i][3 % VEC] = t2.w;
                        s2[u][i][0] = t3.x; s2[u][i][1 % VEC] = t3.y; s2[u][i][2 % VEC] = t3.z; s2[u][i][3 % VEC] = t3.w;
                    } else {
                        gv[u][i][0] = on ? gV[o] : 0.f;
                        wv[u][i][0] = on ? V[o] : 0.f;
                        s1[u][i][0] = on ? s1V[o] : 0.f;
                        s2[u][i][0] = (on && two_state) ? s2V[o] : 0.f;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (!ok[u]) continue;
                if (q == 0) {
                    float w = w_[u], a = a_[u], b2 = b_[u];
                    update_one(P, P.corrW, w, gw_[u], a, b2);
                    W[f[u]] = w; s1W[f[u]] = a; gW[f[u]] = 0.f;
                    if (two_state) s2W[f[u]] = b2;
                }
                const size_t ro = f[u] * (size_t)rowlen;
#pragma unroll
                for (int i = 0; i < SPL; i++) {
                    const int sl = q + i * LPR;
                    if (sl >= slices) continue;
                    bool nz = false;
#pragma unroll
                    for (int cc = 0; cc < VEC; cc++) nz |= gv[u][i][cc] != 0.f;
                    if (!nz) continue;  // untouched slice (FFM: field absent from every row of the batch)
#pragma unroll
                    for (int cc = 0; cc < VEC; cc++) update_one(P, P.corrV, wv[u][i][cc], gv[u][i][cc], s1[u][i][cc], s2[u][i][cc]);
                    const size_t o = ro + (size_t)sl * VEC;
                    if (VEC == 4) {
                        *reinterpret_cast<float4*>(V + o) = make_float4(wv[u][i][0], wv[u][i][1 % VEC], wv[u][i][2 % VEC], wv[u][i][3 % VEC]);
                        *reinterpret_cast<float4*>(s1V + o) = make_float4(s1[u][i][0], s1[u][i][1 % VEC], s1[u][i][2 % VEC], s1[u][i][3 % VEC]);
                        if (two_state) *reinterpret_cast<float4*>(s2V + o) = make_float4(s2[u][i][0], s2[u][i][1 % VEC], s2[u][i][2 % VEC], s2[u][i][3 % VEC]);
                        *reinterpret_cast<float4*>(gV + o) = make_float4(0, 0, 0, 0);
                    } else {
                        V[o] = wv[u][i][0]; s1V[o] = s1[u][i][0]; gV[o] = 0.f;
                        if (two_state) s2V[o] = s2[u][i][0];
                    }
                }
            }
        }
    }
    // re-arm the list for the next step once every block has consumed it
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(done, 1u) == gridDim.x - 1) { *n_list = 0u; *done = 0u; __threadfence(); }
    }
}

// the sparse apply's instance: Adagrad, FTRL, Adam, RMSprop and Adadelta are specialised on 4-wide rows, every other
// updater and row shape takes OPT = -1
template <int LPR, int VEC, int SPL, int U>
static auto apply_instance(int opt) {
    if (VEC != 4) return apply_kernel<LPR, VEC, SPL, U, -1>;
    switch (opt) {
        case LCTR_OPT_ADAGRAD: return apply_kernel<LPR, VEC, SPL, U, LCTR_OPT_ADAGRAD>;
        case LCTR_OPT_FTRL: return apply_kernel<LPR, VEC, SPL, U, LCTR_OPT_FTRL>;
        case LCTR_OPT_ADAM: return apply_kernel<LPR, VEC, SPL, U, LCTR_OPT_ADAM>;
        case LCTR_OPT_RMSPROP: return apply_kernel<LPR, VEC, SPL, U, LCTR_OPT_RMSPROP>;
        case LCTR_OPT_ADADELTA: return apply_kernel<LPR, VEC, SPL, U, LCTR_OPT_ADADELTA>;
        default: return apply_kernel<LPR, VEC, SPL, U, -1>;
    }
}
template <int VEC>
static auto apply_pick(int lpr, int spl, int opt) {
    switch (lpr) {
        case 1: return apply_instance<1, VEC, 1, 4>(opt);
        case 2: return apply_instance<2, VEC, 1, 4>(opt);
        case 4: return apply_instance<4, VEC, 1, 4>(opt);
        case 8: return apply_instance<8, VEC, 1, 4>(opt);
        case 16: return apply_instance<16, VEC, 1, 4>(opt);
        default:
            return spl == 1 ? apply_instance<32, VEC, 1, 4>(opt) : spl == 2 ? apply_instance<32, VEC, 2, 2>(opt)
                 : spl == 3 ? apply_instance<32, VEC, 3, 1>(opt) : apply_instance<32, VEC, 4, 1>(opt);
    }
}

int launch_apply(lctr_ctx* c, int64_t rows_in_step) {
    OptParams P = make_opt_params(c, rows_in_step);
    const int rowlen = (int)c->rowlen;
    const int vec = (rowlen % 4 == 0) ? 4 : 1;
    const int slices = rowlen / vec;
    int lpr = 1;
    while (lpr < slices && lpr < 32) lpr <<= 1;
    const int spl = (slices + lpr - 1) / lpr;
    LCTR_CHECK(spl <= 4, "row of %d floats is too long for the sparse apply kernel (max %d)", rowlen, 4 * 32 * vec);
    const size_t ntiles = (c->Fl + 511) / 512;
    unsigned grid_a = (unsigned)std::min<size_t>((ntiles + 7) / 8, (size_t)c->sm_count * 8);
    if (grid_a == 0) grid_a = 1;
    const unsigned grid = (unsigned)c->sm_count * 2;
    ProfScope prof(c, PROF_APPLY);
    if (launch(c, {grid_a, 256, 0, c->stream}, compact_touched_kernel, c->touched, c->Fl, c->touch_list, c->n_touch)) return 1;
    return launch(c, {grid, 256, 0, c->stream}, vec == 4 ? apply_pick<4>(lpr, spl, P.opt) : apply_pick<1>(lpr, spl, P.opt),
                  c->touch_list, c->n_touch, c->apply_done, rowlen, c->W, c->V, c->gW, c->gV, c->s1W, c->s1V, c->s2W, c->s2V, P);
}

}  // namespace lctr
