// api_util.cuh -- error reporting, and the one launcher every kernel of the C ABI translation units goes through.
#pragma once
#include <cuda_runtime.h>

#include <utility>

#include "../../include/b200raster.h"  // kernel ids B200R_K_* for b200r_profile_read

int b200r_fail(int code, const char* fmt, ...);            // records message, returns code
int b200r_cuda_fail(cudaError_t e, const char* what);      // records message, returns (int)e

// Implementation of b200r_launch.  When profiling is enabled (b200r_profile_enable(1)) each launch is bracketed by a
// pair of CUDA events recorded on the launch stream; otherwise the two calls are no-ops.
void b200r_prof_begin(int kernel, cudaStream_t st);
void b200r_prof_end(int kernel, cudaStream_t st);
void b200r_count_launch(void);

// Launches kernel<<<grid, block, smem, st>>>(args...) inside one profiler span under prof_id (a B200R_K_* id), counts
// it in b200r_launch_count, and returns 0, or the launch error recorded under the kernel's name.
template <typename... KernelArgs, typename... Args>
int b200r_launch(const char* name, int prof_id, void (*kernel)(KernelArgs...), dim3 grid, dim3 block, size_t smem,
                 cudaStream_t st, Args&&... args) {
    b200r_prof_begin(prof_id, st);
    kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
    b200r_prof_end(prof_id, st);
    b200r_count_launch();
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : b200r_cuda_fail(e, name);
}

// cudaMemsetAsync(p, 0, bytes, st); returns 0, or the error recorded under `what`.
inline int b200r_zero(void* p, size_t bytes, cudaStream_t st, const char* what) {
    const cudaError_t e = cudaMemsetAsync(p, 0, bytes, st);
    return e == cudaSuccess ? 0 : b200r_cuda_fail(e, what);
}
