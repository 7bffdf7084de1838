// scripts/lab/fm_lab.cu -- kernel lab for the FM step: times the candidate kernels of
// lightctr_b200/csrc/fm_fused.cuh and a family of RED micro-benchmarks on a dumped synthetic batch
// (scripts/lab/dump_batch.py), with the L2 flushed before every timed launch.  Not part of the product.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -lineinfo -o scripts/lab/fm_lab scripts/lab/fm_lab.cu
//   scripts/lab/fm_lab /tmp/lab_F1000000_B4096.bin [K=16]
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../lightctr_b200/csrc/fm_fused.cuh"

namespace lctr {
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
}
}  // namespace lctr
using namespace lctr;

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } \
    } while (0)

static void* g_flush = nullptr;
static const size_t kFlushBytes = 256u << 20;
static cudaStream_t st;

template <class F>
static float time_us(F&& launch, int reps = 9, bool flush = true) {
    std::vector<float> t;
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    for (int i = 0; i < reps + 2; i++) {
        if (flush) CK(cudaMemsetAsync(g_flush, i, kFlushBytes, st));
        CK(cudaEventRecord(a, st));
        launch();
        CK(cudaEventRecord(b, st));
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        float ms;
        CK(cudaEventElapsedTime(&ms, a, b));
        if (i >= 2) t.push_back(ms * 1e3f);
    }
    std::sort(t.begin(), t.end());
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    return t[t.size() / 2];
}

__global__ void fill_v_kernel(float* V, size_t n, float scale) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        unsigned long long h = i * 0x9E3779B97F4A7C15ull + 1234;
        h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
        const float u1 = ((unsigned)(h & 0xffffffu) + 1u) * (1.0f / 16777217.0f);
        const float u2 = (unsigned)((h >> 24) & 0xffffffu) * (1.0f / 16777216.0f);
        V[i] = scale * sqrtf(-2.0f * logf(u1)) * cosf(6.2831853f * u2);
    }
}

// naive per-sample reference (thread = sample): pred, and gradients into a compact buffer with plain atomics
__global__ void ref_step_kernel(const int64_t* row_ptr, const uint32_t* fid, const uint32_t* ent_slot, const float* label,
                                const float* W, const float* V, int K, float* pred, float* G, int GS, float l2, int64_t rows) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    float s[32];
    for (int c = 0; c < K; c++) s[c] = 0.f;
    float fm = 0.f;
    for (int64_t e = row_ptr[r]; e < row_ptr[r + 1]; e++) {
        const uint32_t f = fid[e];
        fm += W[f];
        float dot = 0.f;
        for (int c = 0; c < K; c++) { const float t = V[(size_t)f * K + c]; s[c] += t; dot += t * t; }
        fm -= 0.5f * dot;
    }
    float dot = 0.f;
    for (int c = 0; c < K; c++) dot += s[c] * s[c];
    fm += 0.5f * dot;
    const float p = 1.f / (1.f + expf(-fm));
    pred[r] = p;
    const float d = p - label[r];
    for (int64_t e = row_ptr[r]; e < row_ptr[r + 1]; e++) {
        const uint32_t f = fid[e];
        const float gw = d + l2 * W[f];
        float* dst = G + (size_t)ent_slot[e] * GS;
        for (int c = 0; c < K; c++) {
            const float v = V[(size_t)f * K + c];
            atomicAdd(dst + c, (s[c] - v) * gw + l2 * v);
        }
        atomicAdd(dst + K, gw);
    }
}

// ---- RED micro-benchmarks: entry e -> row idx[e]; LPR lanes x (16 B vector RED | 4 B scalar RED) per row ------------
template <int LPR, bool VEC4, bool WITH_W>
__global__ void __launch_bounds__(256)
red_bench_kernel(const uint32_t* __restrict__ idx, int64_t n, float* __restrict__ Gv, int strideV, float* __restrict__ Gw,
                 int strideW, int woff) {
    constexpr int GR = 32 / LPR;
    const int lane = threadIdx.x & 31, q = lane % LPR, g = lane / LPR;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t b0 = warp * 32; b0 < n; b0 += nwarps * 32) {
        const uint32_t mine = b0 + lane < n ? __ldg(idx + b0 + lane) : 0u;
#pragma unroll
        for (int it = 0; it < LPR; it++) {
            const int j = it * GR + g;
            const uint32_t s = __shfl_sync(kFull, mine, j);
            if (b0 + j < n) {
                if (LPR > 0 && Gv) {
                    if (VEC4) red_add_v4(Gv + (size_t)s * strideV + 4 * q, make_float4(1.f, 2.f, 3.f, 4.f));
                    else red_add_f32(Gv + (size_t)s * strideV + q, 1.f);
                }
                if (WITH_W && q == 0) red_add_f32(Gw + (size_t)s * strideW + woff, 1.f);
            }
        }
    }
}

// gather micro-benchmark: same mapping, loads instead of REDs (sum kept live)
template <int LPR>
__global__ void __launch_bounds__(256)
gather_bench_kernel(const uint32_t* __restrict__ idx, int64_t n, const float* __restrict__ T, int stride, float* out) {
    constexpr int GR = 32 / LPR;
    const int lane = threadIdx.x & 31, q = lane % LPR, g = lane / LPR;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    float4 acc = make_float4(0, 0, 0, 0);
    for (int64_t b0 = warp * 64; b0 < n; b0 += nwarps * 64) {
        const uint32_t m0 = b0 + lane < n ? __ldg(idx + b0 + lane) : 0u;
        const uint32_t m1 = b0 + 32 + lane < n ? __ldg(idx + b0 + 32 + lane) : 0u;
        float4 v[2 * LPR];
#pragma unroll
        for (int it = 0; it < 2 * LPR; it++) {
            const int j = it * GR + g;
            const uint32_t s = __shfl_sync(kFull, j < 32 ? m0 : m1, j & 31);
            v[it] = ldg_f4_pinned(T + (size_t)s * stride + 4 * q);
        }
#pragma unroll
        for (int it = 0; it < 2 * LPR; it++) { acc.x += v[it].x; acc.y += v[it].y; acc.z += v[it].z; acc.w += v[it].w; }
    }
    if (acc.x + acc.y + acc.z + acc.w == 123.456f) out[0] = acc.x;
}

__global__ void empty_kernel(int* p) { if (p && threadIdx.x == 12345) *p = 1; }

struct Batch {
    int64_t rows, nnz, F, nf;
    std::vector<int64_t> row_ptr;
    std::vector<uint32_t> fid;
    std::vector<int32_t> label;
};

static Batch load_batch(const char* path) {
    Batch b;
    FILE* f = fopen(path, "rb");
    if (!f) { perror(path); exit(1); }
    int64_t h[4];
    if (fread(h, 8, 4, f) != 4) exit(1);
    b.rows = h[0]; b.nnz = h[1]; b.F = h[2]; b.nf = h[3];
    b.row_ptr.resize(b.rows + 1);
    b.fid.resize(b.nnz);
    b.label.resize(b.rows);
    if (fread(b.row_ptr.data(), 8, b.rows + 1, f) != (size_t)b.rows + 1) exit(1);
    if (fread(b.fid.data(), 4, b.nnz, f) != (size_t)b.nnz) exit(1);
    fseek(f, (long)((b.nnz + (b.nnz & 1)) * 2), SEEK_CUR);
    if (fread(b.label.data(), 4, b.rows, f) != (size_t)b.rows) exit(1);
    fclose(f);
    return b;
}

template <class T>
static T* dmalloc(size_t n) {
    T* p;
    CK(cudaMalloc((void**)&p, std::max<size_t>(n, 1) * sizeof(T)));
    CK(cudaMemset(p, 0, std::max<size_t>(n, 1) * sizeof(T)));
    return p;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: fm_lab batch.bin\n"); return 2; }
    constexpr int K = 16;
    Batch hb = load_batch(argv[1]);
    const int64_t B = hb.rows, nnz = hb.nnz;
    const size_t F = (size_t)hb.F;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CK(cudaMalloc(&g_flush, kFlushBytes));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int SM = prop.multiProcessorCount;
    printf("# device %s, %d SMs; batch rows=%lld nnz=%lld F=%zu K=%d\n", prop.name, SM, (long long)B, (long long)nnz, F, K);

    int64_t* d_rp = dmalloc<int64_t>(B + 1);
    uint32_t* d_fid = dmalloc<uint32_t>(nnz + 64);
    float* d_label = dmalloc<float>(B);
    {
        std::vector<float> lf(B);
        for (int64_t i = 0; i < B; i++) lf[i] = (float)hb.label[i];
        CK(cudaMemcpy(d_rp, hb.row_ptr.data(), (B + 1) * 8, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_fid, hb.fid.data(), nnz * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_label, lf.data(), B * 4, cudaMemcpyHostToDevice));
    }
    float* W = dmalloc<float>(F);
    float* V = dmalloc<float>(F * K);
    float* s1W = dmalloc<float>(F);
    float* s1V = dmalloc<float>(F * K);
    fill_v_kernel<<<SM * 8, 256, 0, st>>>(V, F * K, 0.25f);
    fill_v_kernel<<<SM * 8, 256, 0, st>>>(W, F, 0.01f);
    const size_t MT = mark_rows(F);
    uint8_t* mark = dmalloc<uint8_t>(128 * MT + 512);
    uint32_t* slot_of = dmalloc<uint32_t>(F);
    uint32_t* uniq = dmalloc<uint32_t>(nnz + 64);
    unsigned* n_uniq = dmalloc<unsigned>(1);
    uint32_t* ent_slot = dmalloc<uint32_t>(nnz + 64);
    unsigned* cnt = dmalloc<unsigned>(nnz + 64);
    uint32_t* hot_of = dmalloc<uint32_t>(nnz + 64);
    unsigned* n_hot = dmalloc<unsigned>(1);
    uint32_t* hot_slot = dmalloc<uint32_t>(kHotMax);
    uint32_t* ent_slot_nohot = dmalloc<uint32_t>(nnz + 64);
    float* pred = dmalloc<float>(B);
    float* pred_ref = dmalloc<float>(B);
    float* sumvx = dmalloc<float>(B * K);
    float* dvec = dmalloc<float>(B);
    double* partial = dmalloc<double>(2);
    unsigned* done = dmalloc<unsigned>(1);
    double* out_slot = dmalloc<double>(2);
    const int GSmax = 32;
    float* G = nullptr;  // compact gradient buffer, allocated once U is known
    CK(cudaStreamSynchronize(st));

    // ------------------------------------------------------------------ prep: slot map
    const unsigned mg = (unsigned)std::min<int64_t>((nnz + 255) / 256, (int64_t)SM * 8);
    const unsigned mkg = (unsigned)std::min<int64_t>((nnz + 2047) / 2048, (int64_t)SM * 4);
    const size_t ntiles = (128 * mark_rows(F) + 511) / 512;
    const unsigned cg = (unsigned)std::min<size_t>((ntiles + 7) / 8, (size_t)SM * 8);
    const unsigned sg = (unsigned)std::min<int64_t>(((int64_t)kHotSampleRows * 128 + 255) / 256, (int64_t)SM * 8);
    auto prep_slotmap = [&]() {
        CK(cudaMemsetAsync(n_uniq, 0, 4, st));
        CK(cudaMemsetAsync(n_hot, 0, 4, st));
        slotmap_mark_kernel<<<mkg, 256, 0, st>>>(d_fid, nullptr, nnz, mark, MT);
        slotmap_compact_kernel<<<cg, 256, 0, st>>>(mark, MT, uniq, n_uniq, slot_of);
        slotmap_sample_kernel<<<sg, 256, 0, st>>>(d_rp, d_fid, nullptr, B, slot_of, cnt);
        slotmap_hot_kernel<<<SM * 2, 256, 0, st>>>(cnt, n_uniq, nullptr, B, hot_of, hot_slot, n_hot);
        slotmap_assign_kernel<<<mg, 256, 0, st>>>(d_fid, nullptr, nnz, slot_of, hot_of, ent_slot, nullptr);
    };
    prep_slotmap();
    CK(cudaStreamSynchronize(st));
    unsigned U = 0;
    CK(cudaMemcpy(&U, n_uniq, 4, cudaMemcpyDeviceToHost));
    unsigned NH = 0;
    CK(cudaMemcpy(&NH, n_hot, 4, cudaMemcpyDeviceToHost));
    printf("# unique features U=%u (%.2f entries per unique), hot slots %u (cap %d)\n", U, (double)nnz / U, NH, kHotMax);
    printf("prep_slotmap(mark+compact+sample+hot+assign)_us,%.2f\n", time_us(prep_slotmap));
    printf("prep_sample_us,%.2f\n", time_us([&]() { slotmap_sample_kernel<<<sg, 256, 0, st>>>(d_rp, d_fid, nullptr, B, slot_of, cnt); }));
    CK(cudaMemsetAsync(cnt, 0, (size_t)(nnz + 64) * 4, st));
    printf("prep_assign_us,%.2f\n", time_us([&]() { slotmap_assign_kernel<<<mg, 256, 0, st>>>(d_fid, nullptr, nnz, slot_of, hot_of, ent_slot, nullptr); }));
    printf("prep_mark_us,%.2f\n", time_us([&]() { slotmap_mark_kernel<<<mkg, 256, 0, st>>>(d_fid, nullptr, nnz, mark, MT); }));
    printf("prep_compact(empty map)_us,%.2f\n", time_us([&]() { CK(cudaMemsetAsync(n_uniq, 0, 4, st)); slotmap_compact_kernel<<<cg, 256, 0, st>>>(mark, MT, uniq, n_uniq, slot_of); }));
    {   // the five kernels of the build, timed one by one inside the sequence (L2 flushed first)
        cudaEvent_t ev[8];
        for (auto& e : ev) CK(cudaEventCreate(&e));
        CK(cudaMemsetAsync(g_flush, 1, kFlushBytes, st));
        CK(cudaMemsetAsync(n_uniq, 0, 4, st));
        CK(cudaMemsetAsync(n_hot, 0, 4, st));
        CK(cudaEventRecord(ev[0], st));
        slotmap_mark_kernel<<<mkg, 256, 0, st>>>(d_fid, nullptr, nnz, mark, MT);
        CK(cudaEventRecord(ev[1], st));
        slotmap_compact_kernel<<<cg, 256, 0, st>>>(mark, MT, uniq, n_uniq, slot_of);
        CK(cudaEventRecord(ev[2], st));
        slotmap_sample_kernel<<<sg, 256, 0, st>>>(d_rp, d_fid, nullptr, B, slot_of, cnt);
        CK(cudaEventRecord(ev[3], st));
        slotmap_hot_kernel<<<SM * 2, 256, 0, st>>>(cnt, n_uniq, nullptr, B, hot_of, hot_slot, n_hot);
        CK(cudaEventRecord(ev[4], st));
        slotmap_assign_kernel<<<mg, 256, 0, st>>>(d_fid, nullptr, nnz, slot_of, hot_of, ent_slot, nullptr);
        CK(cudaEventRecord(ev[5], st));
        CK(cudaStreamSynchronize(st));
        const char* nm[5] = {"mark", "compact", "sample", "hot", "assign"};
        for (int i = 0; i < 5; i++) { float ms; CK(cudaEventElapsedTime(&ms, ev[i], ev[i + 1])); printf("prep_seq_%s_us,%.2f\n", nm[i], ms * 1e3f); }
    }
    slotmap_assign_kernel<<<mg, 256, 0, st>>>(d_fid, nullptr, nnz, slot_of, nullptr, ent_slot_nohot, nullptr);
    CK(cudaStreamSynchronize(st));
    G = dmalloc<float>((size_t)(U + 64) * GSmax);
    float* Gref = dmalloc<float>((size_t)(U + 64) * GSmax);
    float* G2 = dmalloc<float>((size_t)(U + 64) * GSmax);
    float* Ghot = dmalloc<float>((size_t)kHotMax * kHotRep * GSmax);

    // ------------------------------------------------------------------ step kernels
    const float l2 = 0.001f;
    const unsigned fgrid = (unsigned)std::min<int64_t>((B + 3) / 4, (int64_t)SM * 4);
    OptParams P;
    memset(&P, 0, sizeof(P));
    P.opt = LCTR_OPT_ADAGRAD; P.invB = (float)(1.0 / (double)B); P.mb = (float)B; P.lr = 0.1f; P.corrW = P.corrV = 1.f;
    for (int GS : {32}) {
        auto fused = [&]() {
            fm_fused_kernel<K, false, 1, false><<<fgrid, 128, 0, st>>>(d_rp, d_fid, ent_slot, nullptr, d_label, W, V, pred, sumvx, dvec, G, Ghot, GS, l2,
                                                                         0, B, nullptr, partial, done, out_slot, 1);
        };
        auto fused3 = [&]() {
            fm_fused_kernel<K, false, 1, false, 3><<<std::min<unsigned>(fgrid, SM * 3), 128, 0, st>>>(d_rp, d_fid, ent_slot, nullptr, d_label, W, V, pred, sumvx, dvec, G, Ghot, GS, l2,
                                                                         0, B, nullptr, partial, done, out_slot, 1);
        };
        auto fused_nohot = [&]() {
            fm_fused_kernel<K, false, 1, false><<<fgrid, 128, 0, st>>>(d_rp, d_fid, ent_slot_nohot, nullptr, d_label, W, V, pred, sumvx, dvec, G, Ghot, GS, l2,
                                                                         0, B, nullptr, partial, done, out_slot, 1);
        };
        auto fwd = [&]() {
            fm_fused_kernel<K, false, 0, true><<<fgrid, 128, 0, st>>>(d_rp, d_fid, d_fid, nullptr, d_label, W, V, pred, sumvx, dvec, nullptr, nullptr, GS, l2,
                                                                        0, B, nullptr, partial, done, out_slot, 1);
        };
        auto apply = [&]() {
            apply_compact_kernel<K, LCTR_OPT_ADAGRAD><<<SM * 3 + kHotMax / 8, 256, 0, st>>>(uniq, n_uniq, G, hot_of, hot_slot, n_hot, Ghot, GS, SM * 3, W, V, s1W, s1V, nullptr, nullptr, P, nullptr);
        };
        // validation against the naive kernel (gradients only; apply is skipped so that parameters stay put)
        CK(cudaMemsetAsync(G, 0, (size_t)(U + 64) * GSmax * 4, st));
        CK(cudaMemsetAsync(Gref, 0, (size_t)(U + 64) * GSmax * 4, st));
        CK(cudaMemsetAsync(G2, 0, (size_t)(U + 64) * GSmax * 4, st));
        CK(cudaMemsetAsync(Ghot, 0, (size_t)kHotMax * kHotRep * GSmax * 4, st));
        ref_step_kernel<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(d_rp, d_fid, ent_slot_nohot, d_label, W, V, K, pred_ref, Gref, GS, l2, B);
        fused();
        CK(cudaStreamSynchronize(st));
        CK(cudaGetLastError());
        {
            std::vector<float> a((size_t)U * GS), b((size_t)U * GS), pa(B), pb(B);
            CK(cudaMemcpy(a.data(), G, a.size() * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(b.data(), Gref, b.size() * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(pa.data(), pred, B * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(pb.data(), pred_ref, B * 4, cudaMemcpyDeviceToHost));
            {   // fold the hot replicas into their slots
                std::vector<float> hh((size_t)kHotMax * kHotRep * GS);
                std::vector<uint32_t> ho(U);
                CK(cudaMemcpy(hh.data(), Ghot, hh.size() * 4, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(ho.data(), hot_of, (size_t)U * 4, cudaMemcpyDeviceToHost));
                for (unsigned sl = 0; sl < U; sl++)
                    if (ho[sl] != 0xffffffffu)
                        for (int rp = 0; rp < kHotRep; rp++)
                            for (int c = 0; c < GS; c++) a[(size_t)sl * GS + c] += hh[((size_t)ho[sl] * kHotRep + rp) * GS + c];
            }
            double mg_ = 0, mp = 0, mx = 0;
            for (size_t i = 0; i < a.size(); i++) { mg_ = std::max(mg_, (double)fabsf(a[i] - b[i])); mx = std::max(mx, (double)fabsf(b[i])); }
            for (int64_t i = 0; i < B; i++) mp = std::max(mp, (double)fabsf(pa[i] - pb[i]));
            printf("# GS=%d fused vs naive: max|dG|=%.3g (max|G|=%.3g) max|dpred|=%.3g\n", GS, mg_, mx, mp);
        }
        CK(cudaMemsetAsync(G, 0, (size_t)(U + 64) * GSmax * 4, st));
        CK(cudaMemsetAsync(Ghot, 0, (size_t)kHotMax * kHotRep * GSmax * 4, st));
        const double gather_bytes = ((double)nnz / B * (4 * K + 12) + 8) * B;
        float t;
        t = time_us(fwd);
        printf("GS=%d,fwd_only_us,%.2f,gather_GBps,%.1f\n", GS, t, gather_bytes / t * 1e-3);
        t = time_us(fused);
        printf("GS=%d,fused_fwd_bwd_red_us,%.2f,gather_GBps,%.1f\n", GS, t, gather_bytes / t * 1e-3);
        t = time_us(fused3);
        printf("GS=%d,fused_minb3_us,%.2f,gather_GBps,%.1f\n", GS, t, gather_bytes / t * 1e-3);
        t = time_us(fused_nohot);
        printf("GS=%d,fused_nohot_us,%.2f,gather_GBps,%.1f\n", GS, t, gather_bytes / t * 1e-3);
        t = time_us([&]() { fused(); apply(); });
        printf("GS=%d,step_red(fused+apply)_us,%.2f\n", GS, t);
        {   // apply alone, right after a fused launch (G hot in L2 as in the real step)
            std::vector<float> ts;
            cudaEvent_t ea, eb;
            cudaEventCreate(&ea); cudaEventCreate(&eb);
            for (int i = 0; i < 7; i++) {
                CK(cudaMemsetAsync(g_flush, i, kFlushBytes, st));
                fused();
                CK(cudaEventRecord(ea, st));
                apply();
                CK(cudaEventRecord(eb, st));
                CK(cudaStreamSynchronize(st));
                float ms; CK(cudaEventElapsedTime(&ms, ea, eb));
                ts.push_back(ms * 1e3f);
            }
            std::sort(ts.begin(), ts.end());
            printf("GS=%d,apply_after_fused_us,%.2f\n", GS, ts[ts.size() / 2]);
        }
        t = time_us([&]() { fused(); apply(); }, 9, false);
        printf("GS=%d,step_red_noflush_us,%.2f\n", GS, t);
        // re-zero state touched by apply so both layouts start alike
        CK(cudaMemsetAsync(s1V, 0, F * K * 4, st));
        CK(cudaMemsetAsync(s1W, 0, F * 4, st));
        fill_v_kernel<<<SM * 8, 256, 0, st>>>(V, F * K, 0.25f);
        fill_v_kernel<<<SM * 8, 256, 0, st>>>(W, F, 0.01f);
        CK(cudaMemsetAsync(G, 0, (size_t)(U + 64) * GSmax * 4, st));
    }
    printf("empty_kernel_pair_us,%.2f\n", time_us([&]() { empty_kernel<<<1, 32, 0, st>>>(nullptr); empty_kernel<<<1, 32, 0, st>>>(nullptr); }, 9, false));
    printf("empty_kernel_x1_us,%.2f\n", time_us([&]() { empty_kernel<<<1, 32, 0, st>>>(nullptr); }, 9, false));

    // ------------------------------------------------------------------ RED micro-benchmarks
    float* gVs = dmalloc<float>(F * K);  // fid-indexed (sparse) target, the r01 layout
    float* gWs = dmalloc<float>(F);
    std::vector<uint32_t> h_rand_u(nnz), h_rand_f(nnz);
    {
        unsigned long long sd = 88172645463325252ull;
        for (int64_t i = 0; i < nnz; i++) {
            sd ^= sd << 13; sd ^= sd >> 7; sd ^= sd << 17;
            h_rand_u[i] = (uint32_t)(sd % U);
            h_rand_f[i] = (uint32_t)((sd >> 20) % F);
        }
    }
    uint32_t* rand_u = dmalloc<uint32_t>(nnz + 64);
    uint32_t* rand_f = dmalloc<uint32_t>(nnz + 64);
    CK(cudaMemcpy(rand_u, h_rand_u.data(), nnz * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(rand_f, h_rand_f.data(), nnz * 4, cudaMemcpyHostToDevice));
    const unsigned rgrid = SM * 8;
    auto report = [&](const char* name, float us, double adds_per_entry, double lines_per_entry) {
        printf("red,%s,us,%.2f,Gadds_s,%.1f,Glines_s,%.2f\n", name, us, nnz * adds_per_entry / us * 1e-3, nnz * lines_per_entry / us * 1e-3);
    };
    report("compact_zipf_v64B+w_merged_stride20", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 20, G, 20, 16); }), 17, 1);
    report("compact_zipf_v64B+w_merged_stride32", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 32, G, 32, 16); }), 17, 1);
    report("compact_zipf_v64B_only_stride16", time_us([&]() { red_bench_kernel<4, true, false><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 16, nullptr, 0, 0); }), 16, 1);
    report("compact_zipf_v64B+w_separate", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 16, Gref, 1, 0); }), 17, 2);
    report("compact_zipf_w_only", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, nullptr, 16, Gref, 1, 0); }), 1, 1);
    report("sparse_fid_zipf_v64B+w_separate(r01 layout)", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(d_fid, nnz, gVs, 16, gWs, 1, 0); }), 17, 2);
    report("sparse_fid_zipf_v64B_only", time_us([&]() { red_bench_kernel<4, true, false><<<rgrid, 256, 0, st>>>(d_fid, nnz, gVs, 16, nullptr, 0, 0); }), 16, 1);
    report("compact_uniform_v64B+w_merged_stride20", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(rand_u, nnz, G, 20, G, 20, 16); }), 17, 1);
    report("sparse_uniform_v64B+w_separate", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(rand_f, nnz, gVs, 16, gWs, 1, 0); }), 17, 2);
    report("compact_zipf_scalar16x4B_stride20", time_us([&]() { red_bench_kernel<16, false, false><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 20, nullptr, 0, 0); }), 16, 1);
    report("compact_zipf_v128B_stride32", time_us([&]() { red_bench_kernel<8, true, false><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 32, nullptr, 0, 0); }), 32, 1);
    report("compact_zipf_v64B+w_merged_stride20_noflush", time_us([&]() { red_bench_kernel<4, true, true><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 20, G, 20, 16); }, 9, false), 17, 1);
    // gathers with the same mapping
    {
        float t = time_us([&]() { gather_bench_kernel<4><<<rgrid, 256, 0, st>>>(d_fid, nnz, V, 16, dvec); });
        printf("gather,table_V_fid_zipf_64B,us,%.2f,GBps,%.1f\n", t, nnz * 64.0 / t * 1e-3);
        t = time_us([&]() { gather_bench_kernel<4><<<rgrid, 256, 0, st>>>(ent_slot_nohot, nnz, G, 32, dvec); });
        printf("gather,compact_rows_64B,us,%.2f,GBps,%.1f\n", t, nnz * 64.0 / t * 1e-3);
        t = time_us([&]() { gather_bench_kernel<4><<<rgrid, 256, 0, st>>>(rand_f, nnz, V, 16, dvec); });
        printf("gather,table_V_uniform_64B,us,%.2f,GBps,%.1f\n", t, nnz * 64.0 / t * 1e-3);
    }
    printf("# done\n");
    return 0;
}
