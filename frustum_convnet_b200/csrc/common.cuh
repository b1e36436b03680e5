// Shared helpers for libfrustum_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <utility>

#include "../../include/frustum_b200.h"

namespace fcn {

extern thread_local char g_err[512];

inline int invalid(const char *fn, const char *msg) {
    snprintf(g_err, sizeof(g_err), "%s: invalid argument: %s", fn, msg);
    return FCN_ERR_INVALID;
}
inline int cuda_fail(const char *fn, cudaError_t e) {
    snprintf(g_err, sizeof(g_err), "%s: CUDA error: %s", fn, cudaGetErrorString(e));
    return FCN_ERR_CUDA;
}

#define FCN_REQUIRE(cond, msg)                                  \
    do {                                                        \
        if (!(cond)) return fcn::invalid(__func__, msg);        \
    } while (0)

#define FCN_CUDA(call)                                              \
    do {                                                            \
        cudaError_t e__ = (call);                                   \
        if (e__ != cudaSuccess) return fcn::cuda_fail(__func__, e__); \
    } while (0)

#define FCN_LAUNCH_CHECK()                                          \
    do {                                                            \
        cudaError_t e__ = cudaGetLastError();                       \
        if (e__ != cudaSuccess) return fcn::cuda_fail(__func__, e__); \
    } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Host copy of CSR offsets o[0..n] (records split per image, class or frame): they start at 0, never decrease and
// end at total.
inline bool offsets_ok(const int32_t *o, int n, int total) {
    if (o[0] != 0 || o[n] != total) return false;
    for (int i = 0; i < n; ++i)
        if (o[i + 1] < o[i]) return false;
    return true;
}

// Workspace of a two-phase entry family (fcn_*_workspace_bytes, then entries that share the caller's workspace).
// The family's layout function takes pieces in a fixed order from a Carve: with a null base it only sizes them, so
// the size query and every entry read one layout.  Each piece is rounded up to 256 bytes.
struct Carve {
    char *base;
    size_t off;
    char *take(size_t bytes) {
        char *p = base ? base + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    }
};

// fcn_<family>_workspace_bytes: the bytes `layout(Carve &)` takes, or -1 when a cub size query in it fails.
template <typename Layout>
inline long long workspace_size(const char *fn, Layout &&layout) {
    Carve c{nullptr, 0};
    const cudaError_t e = layout(c);
    if (e != cudaSuccess) {
        cuda_fail(fn, e);
        return -1;
    }
    return (long long)c.off;
}

// The prepare step of every entry of a family: size the layout, check the caller's workspace against it, carve it.
template <typename Layout>
inline int carve_workspace(const char *fn, const char *family, void *workspace, long long workspace_bytes,
                           Layout &&layout) {
    const long long need = workspace_size(fn, layout);
    if (need < 0) return FCN_ERR_CUDA;
    if (workspace_bytes < need) {
        char msg[96];
        snprintf(msg, sizeof(msg), "workspace smaller than fcn_%s_workspace_bytes()", family);
        return invalid(fn, msg);
    }
    Carve c{(char *)workspace, 0};
    const cudaError_t e = layout(c);
    return e != cudaSuccess ? cuda_fail(fn, e) : FCN_OK;
}

int sm_count();

// Programmatic dependent launch (PDL): every kernel of the forward chain is launched with the
// programmatic-stream-serialization attribute, executes `griddepcontrol.wait` before its first
// global-memory access (full completion + memory flush of the previous grid) and releases its own
// dependents right after, so launch latency / CTA rasterisation / barrier prologues of kernel
// N+1 overlap the tail of kernel N.  Works unchanged under CUDA-graph capture.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
// Dependents are released right after the wait (shortest chain).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

// A/B knob: launch priority of a kernel class (kept by the graph node when captured).  `FCN_PRIO_PN` /
// `FCN_PRIO_CONV` = integer in the device's stream-priority range (lower = scheduled first); unset = no attribute.
// With several forwards in flight the block scheduler then places e.g. the persistent PointNet CTAs before the
// conv CTAs of the other forwards instead of in arrival order.
constexpr int FCN_NO_PRIORITY = -1000000;
inline int env_priority(const char *name) {
    const char *v = getenv(name);
    return (v != nullptr && *v != 0) ? atoi(v) : FCN_NO_PRIORITY;
}

// `cluster` > 1: thread-block clusters of that many CTAs along x
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(int priority, int cluster, void (*kern)(KArgs...), dim3 grid, dim3 block,
                                      size_t smem, cudaStream_t stream, Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[3];
    static const bool no_pdl = getenv("FCN_NO_PDL") != nullptr;   // diagnostics
    unsigned n = 0;
    if (!no_pdl) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (priority != FCN_NO_PRIORITY) {
        attr[n].id = cudaLaunchAttributePriority;
        attr[n].val.priority = priority;
        ++n;
    }
    if (cluster > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_prio(int priority, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                   cudaStream_t stream, Args &&...args) {
    return launch_pdl_cluster(priority, 1, kern, grid, block, smem, stream, std::forward<Args>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args &&...args) {
    return launch_pdl_prio(FCN_NO_PRIORITY, kern, grid, block, smem, stream, std::forward<Args>(args)...);
}

}  // namespace fcn
