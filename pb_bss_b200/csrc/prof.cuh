// Launching the library's own kernels, with launch accounting and optional CUDA-event timing
// (pbb_launch_count / pbb_profile_* in include/pbb.h).  bench.py uses it to time the dominant kernel with events
// on the launching stream.  Every kernel launch goes through launch_kernel or launch_ex, so each launch is counted
// once, gets its own profile record, and a failed launch names its kernel in pbb_last_error().
#pragma once
#include <cuda_runtime.h>

#include <utility>

#include "common.cuh"

namespace pbb {

void prof_begin(const char* name, cudaStream_t st);
void prof_end(cudaStream_t st);

struct LaunchScope {
  cudaStream_t st;
  LaunchScope(const char* name, cudaStream_t s) : st(s) { prof_begin(name, s); }
  ~LaunchScope() { prof_end(st); }
};

inline int launch_result(cudaError_t e, const char* name) { return e == cudaSuccess ? 0 : cuda_fail(e, name); }

// kern<<<grid, block, smem, st>>>(args...) recorded under `name`
template <typename Kern, typename... Args>
int launch_kernel(const char* name, Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  LaunchScope ls(name, st);
  kern<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
  return launch_result(cudaGetLastError(), name);
}

// A launch with attributes (ClusterLaunch, CoopLaunch): the typed cudaLaunchKernelEx converts args to the kernel's
// parameter types.
template <typename... Params, typename... Args>
int launch_ex(const char* name, const cudaLaunchConfig_t& cfg, void (*kern)(Params...), Args&&... args) {
  LaunchScope ls(name, cfg.stream);
  return launch_result(cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...), name);
}

}  // namespace pbb
