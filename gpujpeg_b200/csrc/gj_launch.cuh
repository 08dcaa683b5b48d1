/*
 * gj_launch.cuh -- programmatic dependent launch (sm_90+) for the kernels of one frame.
 *
 * The six kernels of a frame run back to back on one stream and each needs its predecessor's output, so nothing can overlap
 * but the launch itself: with cudaLaunchAttributeProgrammaticStreamSerialization the next grid is set up (CTAs resident,
 * parameters fetched) while the previous one drains, and waits at `griddepcontrol.wait` -- the first statement of every such
 * kernel -- until the previous grid has completed and its writes are visible.  Because every kernel of the chain waits
 * before it touches memory, the order of all memory operations is the plain stream order.  A kernel launched this way behind
 * something that is not a kernel (memset, copy) is serialised as usual; GPUJPEG_B200_PDL=0 turns the attribute off.
 * Letting the dependents become resident earlier (`griddepcontrol.launch_dependents` at the top of every kernel, table
 * copies in front of the wait) made every stage faster when timed alone and the chain slower: waiting CTAs share the SMs
 * with the grid that still works.
 */
#ifndef GJ_LAUNCH_CUH
#define GJ_LAUNCH_CUH

#include <cuda_runtime.h>
#include <stdlib.h>

#include <utility>

__device__ __forceinline__ void gj_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

static inline int gj_pdl_enabled()
{
    static int on = -1;
    if ( on < 0 ) {
        const char* e = getenv("GPUJPEG_B200_PDL");
        on = !(e && e[0] == '0');
    }
    return on;
}

template <typename... KArgs, typename... Args>
static inline cudaError_t gj_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = gj_pdl_enabled();
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

#endif
