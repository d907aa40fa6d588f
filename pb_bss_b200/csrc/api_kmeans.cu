// C-ABI entry points of the k-means of BinaryGMMTrainer (pb_bss/distribution/gmm.py:176-230, sklearn's
// KMeans(n_clusters=K)) -- see include/pbb.h and csrc/kmeans.cuh.
#include <algorithm>

#include "common.cuh"
#include "kmeans.cuh"
#include "prof.cuh"

namespace pbb {

static bool km_shape_ok(long long N, int E, int K) {
  return N >= 1 && N <= 0x7fffffffll && E >= 1 && E <= kKmMaxE && K >= 1 && K <= kKmMaxK;
}

// Cooperative grid: every chunk its own CTA where the device holds them all at once, else as many as it holds.
static int km_grid(const void* kernel, size_t smem, int nch, int max_ctas, int* grid) {
  int dev = 0, coop = 0, per_sm = 0, sms = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  PBB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) { set_error("k-means: device %d does not support cooperative launch", dev); return 1; }
  PBB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kKmThreads, smem));
  PBB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int g = std::min(nch, per_sm * sms);
  if (max_ctas > 0) g = std::min(g, max_ctas);
  *grid = std::max(1, g);
  return 0;
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_kmeans_workspace_bytes(long long N, int E, int K) {
  if (!km_shape_ok(N, E, K)) return 0;
  return km_layout(N, E, K, nullptr, nullptr);
}

int pbb_kmeans_fit(const double* x, long long N, int E, int K, long long first, const double* uniforms,
                   const double* init, int max_iter, void* workspace, size_t workspace_bytes, double* centres,
                   int* labels, double* inertia, int* n_iter, int* status, int max_ctas, void* stream) {
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(N >= 1 && N <= 0x7fffffffll, 2, "N must be in [1, 2^31)");
  PBB_CHECK_ARG(E >= 1 && E <= kKmMaxE, 3, "E must be in [1, PBB_KMEANS_MAX_E]");
  PBB_CHECK_ARG(K >= 1 && K <= kKmMaxK && K <= N, 4, "K must be in [1, PBB_KMEANS_MAX_K] and not above N");
  PBB_CHECK_ARG(init != nullptr || (first >= 0 && first < N), 5, "first must be in [0, N)");
  PBB_CHECK_ARG(init != nullptr || K == 1 || uniforms != nullptr, 6, "uniforms is null");
  PBB_CHECK_ARG(max_iter >= 1, 8, "max_iter must be positive");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_kmeans_workspace_bytes(N, E, K), 9,
                "workspace too small (pbb_kmeans_workspace_bytes)");
  PBB_CHECK_ARG(centres != nullptr && labels != nullptr && inertia != nullptr && n_iter != nullptr, 11,
                "an output is null");
  PBB_CHECK_ARG(status != nullptr, 15, "status is null");
  PBB_CHECK_ARG(max_ctas >= 0, 16, "max_ctas must not be negative");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  KmWork w;
  km_layout(N, E, K, static_cast<char*>(workspace), &w);
  const int nch = km_chunking(N).nch;
  PBB_CUDA(cudaMemsetAsync(w.bar, 0, 4 * sizeof(unsigned), st));
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  PBB_CUDA(cudaMemsetAsync(labels, 0xff, (size_t)N * sizeof(int), st));  // -1: every label changes at first
  {
    int grid = 0;
    if (int rc = km_grid((const void*)kmeans_init_kernel, 0, nch, max_ctas, &grid)) return rc;
    const CoopLaunch cl(grid, kKmThreads, 0, st);
    PBB_TRY(launch_ex("kmeans_init_kernel", cl.cfg, kmeans_init_kernel, x, N, E, K, first, uniforms, init, w, status));
  }
  {
    const size_t smem = km_lloyd_smem(E, K);
    PBB_CUDA(cudaFuncSetAttribute(kmeans_lloyd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = 0;
    if (int rc = km_grid((const void*)kmeans_lloyd_kernel, smem, nch, max_ctas, &grid)) return rc;
    KmWork wl = w;
    wl.bar = w.bar + 1;
    const CoopLaunch cl(grid, kKmThreads, smem, st);
    PBB_TRY(launch_ex("kmeans_lloyd_kernel", cl.cfg, kmeans_lloyd_kernel, N, E, K, max_iter, wl, centres, labels,
                      inertia, n_iter, status));
  }
  return 0;
}

int pbb_kmeans_predict(const double* x, long long N, int E, int K, const double* centres, int* labels,
                       double* one_hot, void* stream) {
  PBB_CHECK_ARG(x != nullptr || N == 0, 1, "x is null");
  PBB_CHECK_ARG(N >= 0 && N <= 0x7fffffffll, 2, "N must be in [0, 2^31)");
  PBB_CHECK_ARG(E >= 1 && E <= kKmMaxE, 3, "E must be in [1, PBB_KMEANS_MAX_E]");
  PBB_CHECK_ARG(K >= 1 && K <= kKmMaxK, 4, "K must be in [1, PBB_KMEANS_MAX_K]");
  PBB_CHECK_ARG(centres != nullptr, 5, "centres is null");
  PBB_CHECK_ARG(labels != nullptr || one_hot != nullptr || N == 0, 6, "no output");
  if (N == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("kmeans_predict_kernel", kmeans_predict_kernel, (unsigned)((N + kKmThreads - 1) / kKmThreads),
                       kKmThreads, 0, st, x, N, E, K, centres, labels, one_hot);
}

}  // extern "C"
