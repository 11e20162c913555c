// Kernel launches of the step-wise pipeline with programmatic dependent launch (PDL).
//
// A search step is a chain of small dependent kernels (tower -> heads -> tower -> heads -> tree step) replayed from
// a CUDA graph.  With the programmatic-stream-serialization attribute a kernel's CTAs may start while the previous
// kernel is still draining: everything up to `pdl_wait()` (barrier set-up, staging of weights - data no
// kernel of the chain writes) overlaps the predecessor's tail, `pdl_wait()` then blocks until the predecessor has
// completed and its writes are visible.  Every kernel calls `pdl_launch_dependents()` first thing, so its successor
// is released as early as the hardware has room for it.  MZ_NO_PDL=1 launches without the attribute (the device-side
// instructions are then no-ops).
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <utility>

namespace mz {

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

inline bool pdl_enabled() {
    const char* e = getenv("MZ_NO_PDL");
    return !(e && e[0] == '1');
}

template <typename... KArgs, typename... Args>
cudaError_t launch_chained(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// launch_chained for a kernel launched in thread-block clusters of `cluster` CTAs (the grid a multiple of it)
template <typename... KArgs, typename... Args>
cudaError_t launch_chained_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, dim3 cluster, size_t smem, cudaStream_t stream,
                                   Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster.x; attr[1].val.clusterDim.y = cluster.y; attr[1].val.clusterDim.z = cluster.z;
    cfg.attrs = attr; cfg.numAttrs = 2;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace mz
