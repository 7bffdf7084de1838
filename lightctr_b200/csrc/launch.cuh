// lightctr_b200/csrc/launch.cuh -- the one way this library launches a kernel.
#pragma once
#include <map>
#include <mutex>
#include <stdlib.h>
#include <type_traits>
#include <utility>

#include "common.cuh"

namespace lctr {

// Run-time values to kernel template instances.  pick names the instance (or runs the launch) for compile-time constants;
// every branch returns the same type, a kernel pointer or a launch's status.  A combination that is not built is folded
// into the template arguments inside pick, so that it names an instance that is.

// pick(std::bool_constant<b0>(), std::bool_constant<b1>(), ...) for the run-time flags b0, b1, ...
template <typename Pick>
auto by_flags(Pick&& pick) {
    return pick();
}
template <typename Pick, typename... B>
auto by_flags(Pick&& pick, bool b, B... rest) {
    return b ? by_flags([&](auto... f) { return pick(std::true_type(), f...); }, rest...)
             : by_flags([&](auto... f) { return pick(std::false_type(), f...); }, rest...);
}

// pick(std::integral_constant<int, v>()) for v in V0, V1, ..., Vn; any other v takes Vn
template <int V, int... Vs, typename Pick>
auto by_value(int v, Pick&& pick) {
    if constexpr (sizeof...(Vs) == 0) return pick(std::integral_constant<int, V>());
    else return v == V ? pick(std::integral_constant<int, V>()) : by_value<Vs...>(v, pick);
}

// the values a kernel is built for, written once for the check that refuses the others and the dispatch among them
template <int... V>
struct Built {
    static bool has(int v) { return ((v == V) || ...); }
    template <typename Pick>
    static auto pick(int v, Pick&& p) { return by_value<V...>(v, p); }
};

// programmatic dependent launches (updater behind the gradient kernel; dense kernels and the NFM backward behind their
// predecessors): LCTR_PDL=0 turns them off; read per launch, the tests toggle it
inline bool pdl_on() {
    const char* e = getenv("LCTR_PDL");
    return !(e && atoi(e) == 0);
}

// opts kernel in to `smem` bytes of dynamic shared memory on the current device when its static shared memory plus smem
// passes 48 KB; the static size is read once per kernel
inline int smem_opt_in(const void* kernel, size_t smem) {
    static std::mutex mu;
    static std::map<const void*, size_t> static_smem;
    static std::map<std::pair<const void*, int>, size_t> opted;  // (kernel, device) -> bytes already allowed
    int dev = 0;
    LCTR_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    auto it = static_smem.find(kernel);
    if (it == static_smem.end()) {
        cudaFuncAttributes fa;
        LCTR_CUDA(cudaFuncGetAttributes(&fa, kernel));
        it = static_smem.emplace(kernel, fa.sharedSizeBytes).first;
    }
    if (it->second + smem <= 48 * 1024) return 0;
    size_t& allowed = opted[{kernel, dev}];
    if (smem > allowed) {
        LCTR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        allowed = smem;
    }
    return 0;
}

inline int launch_failed(const void* kernel, cudaError_t e) {
    cudaGetLastError();  // the error is reported here; later calls must not see it again
    const char* name = nullptr;
    if (cudaFuncGetName(&name, kernel) != cudaSuccess) name = "?";
    set_error("launch of %s failed: %s", name, cudaGetErrorString(e));
    return 1;
}

struct Launch {
    dim3 grid, block;
    size_t smem = 0;
    cudaStream_t st = nullptr;
    bool dependent = false;  // may start before the kernel in front of it ends (while LCTR_PDL != 0)
};

// Launches kernel(args...) as l describes.  0: launched and counted in c->launches (lctr_launch_count); 1: failed, with the
// CUDA error in set_error.  The arguments convert to the kernel's parameter types.
template <typename... P, typename... A>
int launch(lctr_ctx* c, const Launch& l, void (*kernel)(P...), A&&... args) {
    if (l.smem && smem_opt_in((const void*)kernel, l.smem)) return 1;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = l.grid; cfg.blockDim = l.block; cfg.dynamicSmemBytes = l.smem; cfg.stream = l.st;
    cfg.attrs = at; cfg.numAttrs = l.dependent && pdl_on() ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
    if (e != cudaSuccess) return launch_failed((const void*)kernel, e);
    c->launches++;
    return 0;
}

// Replays a captured graph holding `kernels` kernel nodes, counted like their launches.
inline int launch_graph(lctr_ctx* c, cudaGraphExec_t graph, int kernels, cudaStream_t st) {
    LCTR_CUDA(cudaGraphLaunch(graph, st));
    c->launches += kernels;
    return 0;
}

}  // namespace lctr
