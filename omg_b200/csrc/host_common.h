// Host-side helpers shared by the C-ABI entry points: error string, launch counter, TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <functional>
#include <initializer_list>
#include <utility>

namespace omg {

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

inline int fail(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}

#define OMG_CHECK(cond, ...) \
    do {                     \
        if (!(cond)) return ::omg::fail(__VA_ARGS__); \
    } while (0)

// Attention descriptors (omg_attention, omg_attention_small): the head window [col0, col0 + heads * head_dim) of q, k, v
// and out must lie inside a row of ld elements, else the kernels read or write the next row, or past the buffer's end.
inline int check_head_windows(const char* who, int heads, int head_dim, const int (&col0)[4], const int (&ld)[4]) {
    const char* names[4] = {"q", "k", "v", "out"};
    const long long width = (long long)heads * head_dim;
    for (int i = 0; i < 4; ++i)
        if (col0[i] < 0 || col0[i] + width > ld[i])
            return fail("%s: %s head window [%d, %lld) does not fit its row of %d elements", who, names[i], col0[i],
                        col0[i] + width, ld[i]);
    return 0;
}

// Kernels that move 4 / 8 / 16 B vectors through a caller's pointer need it aligned to that width: a misaligned vector
// access is a sticky fault that takes down the CUDA context of the whole process, so the entry point rejects it first.
// NULL (an absent optional operand) passes.
inline int check_aligned(const char* who, int bytes, std::initializer_list<std::pair<const char*, const void*>> ptrs) {
    for (const auto& p : ptrs)
        if (reinterpret_cast<uintptr_t>(p.second) % (uintptr_t)bytes != 0)
            return fail("%s: %s must be %d B aligned", who, p.first, bytes);
    return 0;
}

#define OMG_CUDA(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) return ::omg::fail("%s failed: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail("launch of %s failed: %s", what, cudaGetErrorString(e));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return 0;
}

// Launch plans (omg_plan_*, include/omg_b200.h): while a thread records, every entry point that launched successfully also
// appends a replayable copy of its call (descriptors by value) to the plan; omg_plan_run re-issues them on a stream.
bool plan_recording();
void plan_note(std::function<int(void*)> step);

// Every kernel of this library can be launched with programmatic dependent launch (PDL): the next kernel's CTAs may
// become resident and run their prologue (barrier init, descriptor prefetch) while the previous kernel drains; each
// kernel executes griddepcontrol.wait before its first dependent global access.  Opt-in (OMG_PDL=1): the one-CTA-per-SM
// GEMM cannot co-reside with its predecessor anyway.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  int cluster_x, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster_x;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
    return launch_cluster(kernel, grid, block, smem, stream, 1, args...);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// libcuda is resolved at run time through the runtime (the build box has no driver library to link against).
PFN_encodeTiled get_encode_tiled();

// Tensor map of rank `rank` (<=5) over 2-byte elements of type `dt` (FLOAT16 | BFLOAT16). dims[0] is the contiguous
// dimension. strides are in ELEMENTS for dims[1..rank-1].  Out-of-bounds box elements read as zero / are clipped on store.
int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, const void* ptr, int rank, const uint64_t* dims,
              const uint64_t* strides_elems, const uint32_t* box, CUtensorMapSwizzle swizzle);

}  // namespace omg
