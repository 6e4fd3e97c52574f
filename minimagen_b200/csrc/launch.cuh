// Kernel launch helper: every kernel of the library goes through launch_k so that programmatic dependent launch (PDL)
// can be switched on for the whole step.  With PDL the next kernel's CTAs are scheduled, and run their prologue
// (barrier init, tensor-map prefetch, coefficient set-up), while the tail of the previous kernel is
// still draining; every kernel executes pdl_wait() before its first global-memory access, so ordering is unchanged.
#pragma once
#include <cuda_runtime.h>

namespace mi {

bool pdl_enabled();          // capi.cu (mi_set_launch_mode)

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Lets the NEXT kernel of the stream be scheduled (on SMs this grid no longer occupies) as soon as every CTA of this grid
// has passed this point; the dependent still blocks in pdl_wait() until this grid has completed and flushed its memory, so
// only its private prologue overlaps.  A no-op unless the dependent was launched with the programmatic-serialization attribute.
// Placement: elementwise kernels trigger at their top (the dependent's CTAs appear during the last wave); the persistent
// tensor-core kernels trigger when their TMA producer has issued its last loads, i.e. about one tile before the end -- a trigger
// at their top parked thousands of waiting CTAs of the next elementwise kernel on the SMs for the whole conv (measured: eager
// step 28 -> 45 ms).
__device__ __forceinline__ void pdl_trigger() {
#ifndef MI_PDL_NO_EARLY_TRIGGER
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace mi
