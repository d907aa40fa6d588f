// C-ABI entry points for the beamforming side: batched small-matrix linear algebra,
// PSD estimation and beamformer application (see include/pbb.h).
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include "em_args.cuh"
#include "heig.cuh"
#include "linalg_kernels.cuh"
#include "extraction.cuh"
#include "distribution.cuh"
#include "prof.cuh"

namespace pbb {

// one warp per matrix
__global__ void heig_batched_kernel(const double2* __restrict__ a, int n, int D, double* __restrict__ w,
                                    double2* __restrict__ v, int* status, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  const size_t per = (jacobi_smem_bytes(D) + 15) & ~(size_t)15;
  double2* A = reinterpret_cast<double2*>(smem_raw + per * warp);
  double2* V = A + D * D;
  double* rot = reinterpret_cast<double*>(V + D * D);
  // Hermitian part of the input times 2^-escale (linalg_kernels.cuh: heig_prepare)
  int escale;
  bool bad;
  heig_prepare(a + (size_t)m * D * D, D, lane, A, escale, bad);
  const int sweeps = warp_jacobi_any(A, V, rot, D, lane);
  if ((__any_sync(0xffffffffu, bad) || sweeps > kJacobiMaxSweeps) && lane == 0 && status) record_first(status, m + 1);
  for (int x = lane; x < D; x += 32) {
    const int r = eig_rank(A, D, x);
    w[(size_t)m * D + r] = scalbn(A[x * D + x].x, escale);
    for (int d = 0; d < D; ++d) v[(size_t)m * D * D + d * D + r] = V[d * D + x];
  }
}

// out[j] = sum_i in[i * C + j] (fixed order)
__global__ void colsum_kernel(const double* __restrict__ in, double* __restrict__ out, int rows, int C) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= C) return;
  double s = 0.0;
  for (int i = 0; i < rows; ++i) s += in[(size_t)i * C + j];
  out[j] = s;
}

static int warps_for(size_t per_warp_bytes) {
  int w = (int)((size_t)(96 * 1024) / per_warp_bytes);
  if (w > 4) w = 4;
  if (w < 1) w = 1;
  return w;
}

static int solve_launch(const void* a, const void* b, int n, int D, int R, int hermitize, void* x, int* status,
                        int strict, cudaStream_t st, int* fallback = nullptr) {
  const size_t per = solve_smem_per_warp(D, R);
  const int warps = warps_for(per);
  PBB_CUDA(cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return launch_kernel("solve_kernel", solve_kernel, (n + warps - 1) / warps, 32 * warps, per * warps, st,
                       reinterpret_cast<const double2*>(a), reinterpret_cast<const double2*>(b), n, D, R, hermitize,
                       reinterpret_cast<double2*>(x), status, warps, strict, fallback);
}

static unsigned blocks_for(size_t count, int threads) { return (unsigned)((count + threads - 1) / threads); }

}  // namespace pbb

using namespace pbb;

extern "C" {

int pbb_heig_batched(const void* a, int n, int D, double* w, void* v, int* status, void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "a is null");
  PBB_CHECK_ARG(n > 0, 2, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 3, "need 0 < D <= 64");
  PBB_CHECK_ARG(w != nullptr, 4, "w is null");
  PBB_CHECK_ARG(v != nullptr, 5, "v is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t per = (jacobi_smem_bytes(D) + 15) & ~(size_t)15;
  const int warps = warps_for(per);
  PBB_CUDA(cudaFuncSetAttribute(heig_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return launch_kernel("heig_batched_kernel", heig_batched_kernel, (n + warps - 1) / warps, 32 * warps, per * warps, st,
                       reinterpret_cast<const double2*>(a), n, D, w, reinterpret_cast<double2*>(v), status, warps);
}

int pbb_gev_batched(const void* a, const void* b, int n, int D, void* w, int* status, void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "target PSD is null");
  PBB_CHECK_ARG(b != nullptr, 2, "noise PSD is null");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 4, "need 0 < D <= 64");
  PBB_CHECK_ARG(w != nullptr, 5, "w is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t per = ((size_t)3 * D * D * sizeof(double2) + (size_t)((D + 1) / 2) * 6 * sizeof(double) + 15) &
                     ~(size_t)15;
  const int warps = warps_for(per);
  PBB_CUDA(cudaFuncSetAttribute(gev_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return launch_kernel("gev_kernel", gev_kernel, (n + warps - 1) / warps, 32 * warps, per * warps, st,
                       reinterpret_cast<const double2*>(a), reinterpret_cast<const double2*>(b), n, D,
                       reinterpret_cast<double2*>(w), status, warps);
}

int pbb_solve_batched(const void* a, const void* b, int n, int D, int R, int hermitize, void* x, int* status,
                      void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "a is null");
  PBB_CHECK_ARG(b != nullptr, 2, "b is null");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 4, "need 0 < D <= 64");
  PBB_CHECK_ARG(R > 0 && R <= 64, 5, "need 0 < R <= 64");
  PBB_CHECK_ARG(x != nullptr, 7, "x is null");
  return solve_launch(a, b, n, D, R, hermitize, x, status, 0, reinterpret_cast<cudaStream_t>(stream));
}

int pbb_solve_batched_strict(const void* a, const void* b, int n, int D, int R, void* x, int* status, void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "a is null");
  PBB_CHECK_ARG(b != nullptr, 2, "b is null");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 4, "need 0 < D <= 64");
  PBB_CHECK_ARG(R > 0 && R <= 64, 5, "need 0 < R <= 64");
  PBB_CHECK_ARG(x != nullptr, 6, "x is null");
  PBB_CHECK_ARG(status != nullptr, 7, "status is null");
  return solve_launch(a, b, n, D, R, 0, x, status, 1, reinterpret_cast<cudaStream_t>(stream));
}

int pbb_mvdr(const void* atf, const void* noise_psd, int n, int D, void* w, void* scratch, int* status,
             void* stream) {
  PBB_CHECK_ARG(atf != nullptr, 1, "atf is null");
  PBB_CHECK_ARG(noise_psd != nullptr, 2, "noise PSD is null");
  PBB_CHECK_ARG(w != nullptr, 5, "w is null");
  PBB_CHECK_ARG(scratch != nullptr, 6, "scratch (n * D complex128) is null");
  int r = pbb_solve_batched(noise_psd, atf, n, D, 1, 1, scratch, status, stream);
  if (r) return r;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("mvdr_scale_kernel", mvdr_scale_kernel, (n + 127) / 128, 128, 0, st,
                       reinterpret_cast<const double2*>(atf), reinterpret_cast<const double2*>(scratch), n, D,
                       reinterpret_cast<double2*>(w));
}

int pbb_souden(const void* phi, const void* target_psd, const void* noise_psd, int n, int D, double eps, void* mat,
               void* num, void* den, void* num_sum, void* den_sum, void* stream) {
  PBB_CHECK_ARG(phi && target_psd && noise_psd, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(mat && num && den && num_sum && den_sum, 7, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PBB_TRY(launch_kernel("souden_kernel", souden_kernel, n, 64, 0, st, reinterpret_cast<const double2*>(phi),
                        reinterpret_cast<const double2*>(target_psd), reinterpret_cast<const double2*>(noise_psd), n, D,
                        eps, reinterpret_cast<double2*>(mat), reinterpret_cast<double2*>(num),
                        reinterpret_cast<double2*>(den)));
  PBB_TRY(launch_kernel("colsum_kernel", colsum_kernel, 1, 128, 0, st, reinterpret_cast<const double*>(num),
                        reinterpret_cast<double*>(num_sum), n, 2 * D));
  return launch_kernel("colsum_kernel", colsum_kernel, 1, 128, 0, st, reinterpret_cast<const double*>(den),
                       reinterpret_cast<double*>(den_sum), n, 2 * D);
}

int pbb_blind_analytic_normalization(const void* vector, const void* noise_psd, int n, int D, void* out,
                                     void* stream) {
  PBB_CHECK_ARG(vector && noise_psd, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0, 3, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("ban_kernel", ban_kernel, (n + 127) / 128, 128, 0, st, reinterpret_cast<const double2*>(vector),
                       reinterpret_cast<const double2*>(noise_psd), n, D, reinterpret_cast<double2*>(out));
}

static int apply_bf_launch(const void* vector, const void* mix, int dtype, int B, int F, int D, int T, void* out,
                           void* stream) {
  PBB_CHECK_ARG(vector && mix, 1, "input is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 3, "bad dtype");
  PBB_CHECK_ARG(B > 0 && B <= 65535 && F > 0 && D > 0 && T > 0, 4, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 7, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid((T + 255) / 256, F < 65535 ? F : 65535, B);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("apply_bf_kernel", apply_bf_kernel<CT>, grid, 256, 0, st,
                         reinterpret_cast<const double2*>(vector), reinterpret_cast<const CT*>(mix), F, D, T,
                         reinterpret_cast<double2*>(out));
  });
}

int pbb_apply_beamforming_vector(const void* vector, const void* mix, int dtype, int F, int D, int T, void* out,
                                 void* stream) {
  return apply_bf_launch(vector, mix, dtype, 1, F, D, T, out, stream);
}

int pbb_apply_beamforming_vector_shared(const void* vector, const void* mix, int dtype, int B, int F, int D, int T,
                                        void* out, void* stream) {
  return apply_bf_launch(vector, mix, dtype, B, F, D, T, out, stream);
}

int pbb_rank_one_estimate(const void* vector, const void* covariance, int n, int D, void* out, void* stream) {
  PBB_CHECK_ARG(vector && covariance, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 3, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("rank_one_kernel", rank_one_kernel, n, 64, 0, st, reinterpret_cast<const double2*>(vector),
                       reinterpret_cast<const double2*>(covariance), n, D, reinterpret_cast<double2*>(out));
}

int pbb_matvec_batched(const void* matrix, const void* vector, int n, int D, void* out, void* stream) {
  PBB_CHECK_ARG(matrix && vector, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 3, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("matvec_kernel", matvec_kernel, (n + 127) / 128, 128, 0, st,
                       reinterpret_cast<const double2*>(matrix), reinterpret_cast<const double2*>(vector), n, D,
                       reinterpret_cast<double2*>(out));
}

size_t pbb_psd_workspace_bytes(int F, int T, int D, int K) {
  if (F <= 0 || T <= 0 || D <= 0 || K <= 0) return 0;
  return (size_t)F * ((T + 31) / 32) * K * ((size_t)D * D + 1) * sizeof(double) + 256;
}

int pbb_power_spectral_density(const void* observation, int dtype, int F, int D, int T, const double* mask, int K,
                               int normalize, void* psd, void* workspace, size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(observation != nullptr, 1, "observation is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "bad dtype");
  PBB_CHECK_ARG(F > 0 && D > 0 && D < 35 && T > 0, 3, "bad shape");
  PBB_CHECK_ARG(K > 0 && K < kMaxK, 7, "need 0 < K < 20");
  PBB_CHECK_ARG(psd != nullptr, 9, "psd is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_psd_workspace_bytes(F, T, D, K), 10,
                "workspace too small (pbb_psd_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = observation; a.zs = T; a.F = F; a.T = T; a.D = D; a.K = K;
  a.mode = kModeM; a.aff_in = mask; a.q_in = nullptr;
  a.part = reinterpret_cast<double*>(workspace);
  const int nch = launch_em(a, dtype, 0, st);
  if (nch <= 0) return nch ? nch : 1;
  const int scale = mask == nullptr ? 2 : (normalize ? 1 : 0);
  return launch_kernel("psd_finalize_kernel", psd_finalize_kernel, dim3(F, K), 64, 0, st, a.part, nch, F, K, D, T,
                       scale, reinterpret_cast<double2*>(psd));
}

// ---- backward passes of the mask-based beamforming chain (linalg_kernels.cuh) --------------------------------------

int pbb_power_spectral_density_backward(const void* observation, int dtype, int F, int D, int T, const double* mask,
                                        int K, int normalize, const void* psd, const void* grad_psd,
                                        void* grad_observation, double* grad_mask, void* stream) {
  PBB_CHECK_ARG(observation != nullptr, 1, "observation is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "bad dtype");
  PBB_CHECK_ARG(F > 0 && D > 0 && D < 35 && T > 0, 3, "bad shape");
  PBB_CHECK_ARG(K > 0 && K < kMaxK, 7, "need 0 < K < 20");
  PBB_CHECK_ARG(mask != nullptr || K == 1, 6, "mask is null and K != 1");
  PBB_CHECK_ARG(psd != nullptr, 9, "psd is null");
  PBB_CHECK_ARG(grad_psd != nullptr, 10, "grad_psd is null");
  PBB_CHECK_ARG(grad_observation != nullptr || grad_mask != nullptr, 11, "both gradients are null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t smem = psd_backward_smem(D, K);
  const long long ctas = (long long)F * ((T + kPsdBwdThreads - 1) / kPsdBwdThreads);
  PBB_CHECK_ARG(ctas <= 0x7fffffffll, 3, "F * ceil(T / 64) exceeds the grid");
  const unsigned grid = (unsigned)ctas;
  const double2* P = reinterpret_cast<const double2*>(psd);
  const double2* G = reinterpret_cast<const double2*>(grad_psd);
  double2* gy = reinterpret_cast<double2*>(grad_observation);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    PBB_CUDA(cudaFuncSetAttribute(psd_backward_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return launch_kernel("psd_backward_kernel", psd_backward_kernel<CT>, grid, kPsdBwdThreads, smem, st,
                         reinterpret_cast<const CT*>(observation), mask, P, G, F, D, T, K, normalize, gy, grad_mask);
  });
}

int pbb_souden_backward(const void* phi, const void* noise_psd, const void* grad_w, int n, int D, int ref_channel,
                        double eps, void* grad_target_psd, void* grad_noise_psd, void* stream) {
  PBB_CHECK_ARG(phi && noise_psd && grad_w, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(ref_channel >= 0 && ref_channel < D, 6, "ref_channel must be in [0, D)");
  PBB_CHECK_ARG(grad_target_psd && grad_noise_psd, 8, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  {
    // grad Phi goes to grad_noise_psd, which the last kernel overwrites
    PBB_TRY(launch_kernel("souden_backward_kernel", souden_backward_kernel, n, 64, 0, st,
                          reinterpret_cast<const double2*>(phi), reinterpret_cast<const double2*>(grad_w), n, D,
                          ref_channel, eps, reinterpret_cast<double2*>(grad_noise_psd)));
  }
  // grad X = N^-H grad Phi; a zero pivot (no derivative: the forward's minimum-norm branch) or non-finite N gives NaN
  const int rc = solve_launch(noise_psd, grad_noise_psd, n, D, D, 2, grad_target_psd, nullptr, 2, st);
  if (rc) return rc;
  return launch_kernel("souden_noise_backward_kernel", souden_noise_backward_kernel, blocks_for((size_t)n * D * D, 128),
                       128, 0, st, reinterpret_cast<const double2*>(grad_target_psd),
                       reinterpret_cast<const double2*>(phi), n, D, reinterpret_cast<double2*>(grad_noise_psd));
}

// ---- backward passes of the get_bf_vector beamformers (linalg_kernels.cuh) ------------------------------------------

int pbb_eigenvector_backward(const void* a, const void* b, const void* w, const void* grad_w, const double* grad_lambda,
                             int n, int D, void* grad_a, void* grad_b, void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "a is null");
  PBB_CHECK_ARG(w != nullptr, 3, "w is null");
  PBB_CHECK_ARG(grad_w != nullptr, 4, "grad_w is null");
  PBB_CHECK_ARG(n > 0, 6, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 7, "need 0 < D <= 64");
  PBB_CHECK_ARG(grad_a != nullptr, 8, "grad_a is null");
  PBB_CHECK_ARG(b == nullptr || grad_b != nullptr, 9, "grad_b is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t per = eig_backward_smem_per_warp(D, b != nullptr);
  const int warps = warps_for(per);
  PBB_CUDA(cudaFuncSetAttribute(eig_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return launch_kernel("eig_backward_kernel", eig_backward_kernel, (n + warps - 1) / warps, 32 * warps, per * warps, st,
                       reinterpret_cast<const double2*>(a), reinterpret_cast<const double2*>(b),
                       reinterpret_cast<const double2*>(w), reinterpret_cast<const double2*>(grad_w), grad_lambda, n, D,
                       reinterpret_cast<double2*>(grad_a), reinterpret_cast<double2*>(grad_b), warps);
}

int pbb_mvdr_backward(const void* atf, const void* noise_psd, const void* x, const void* w, const void* grad_w, int n,
                      int D, void* grad_atf, void* grad_noise_psd, void* scratch, void* stream) {
  PBB_CHECK_ARG(atf && noise_psd && x && w && grad_w, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 6, "bad shape");
  PBB_CHECK_ARG(grad_atf && grad_noise_psd, 8, "output is null");
  PBB_CHECK_ARG(scratch != nullptr, 10, "scratch (n * D complex128) is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const double2* X = reinterpret_cast<const double2*>(x);
  const double2* W = reinterpret_cast<const double2*>(w);
  const double2* G = reinterpret_cast<const double2*>(grad_w);
  double2* q = reinterpret_cast<double2*>(grad_atf);  // overwritten by the last kernel
  double2* p = reinterpret_cast<double2*>(scratch);
  PBB_TRY(launch_kernel("mvdr_backward_rhs_kernel", mvdr_backward_rhs_kernel, blocks_for(n, 128), 128, 0, st,
                        reinterpret_cast<const double2*>(atf), X, W, G, n, D, q));
  // p = N_h^-1 q; a zero pivot (the forward's minimum-norm branch, no derivative) or non-finite N gives NaN
  const int rc = solve_launch(noise_psd, q, n, D, 1, 1, p, nullptr, 2, st);
  if (rc) return rc;
  return launch_kernel("mvdr_backward_kernel", mvdr_backward_kernel, blocks_for((size_t)n * D * D, 128), 128, 0, st, p,
                       X, W, G, n, D, reinterpret_cast<double2*>(grad_atf), reinterpret_cast<double2*>(grad_noise_psd));
}

constexpr int kBanBackwardMaxD = 1024;

int pbb_blind_analytic_normalization_backward(const void* vector, const void* noise_psd, const void* grad_out, int n,
                                              int D, void* grad_vector, void* grad_noise_psd, void* stream) {
  PBB_CHECK_ARG(vector && noise_psd && grad_out, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= kBanBackwardMaxD, 4, "need n > 0 and 0 < D <= 1024");
  PBB_CHECK_ARG(grad_vector && grad_noise_psd, 6, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int warps = 4;
  const size_t smem = (size_t)warps * 2 * D * sizeof(double2);
  PBB_CUDA(cudaFuncSetAttribute(ban_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel("ban_backward_kernel", ban_backward_kernel, (n + warps - 1) / warps, 32 * warps, smem, st,
                       reinterpret_cast<const double2*>(vector), reinterpret_cast<const double2*>(noise_psd),
                       reinterpret_cast<const double2*>(grad_out), n, D, reinterpret_cast<double2*>(grad_vector),
                       reinterpret_cast<double2*>(grad_noise_psd), warps);
}

int pbb_rank_one_estimate_backward(const void* vector, const void* covariance, const void* grad_out, int n, int D,
                                   void* grad_vector, void* grad_covariance, void* stream) {
  PBB_CHECK_ARG(vector && covariance && grad_out, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(grad_vector && grad_covariance, 6, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("rank_one_backward_kernel", rank_one_backward_kernel, n, 64, 0, st,
                       reinterpret_cast<const double2*>(vector), reinterpret_cast<const double2*>(covariance),
                       reinterpret_cast<const double2*>(grad_out), n, D, reinterpret_cast<double2*>(grad_vector),
                       reinterpret_cast<double2*>(grad_covariance));
}

int pbb_matvec_batched_backward(const void* matrix, const void* vector, const void* grad_out, int n, int D,
                                void* grad_matrix, void* grad_vector, void* stream) {
  PBB_CHECK_ARG(matrix && vector && grad_out, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(grad_matrix && grad_vector, 6, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("matvec_backward_kernel", matvec_backward_kernel, blocks_for((size_t)n * D, 128), 128, 0, st,
                       reinterpret_cast<const double2*>(matrix), reinterpret_cast<const double2*>(vector),
                       reinterpret_cast<const double2*>(grad_out), n, D, reinterpret_cast<double2*>(grad_matrix),
                       reinterpret_cast<double2*>(grad_vector));
}

static int apply_bf_backward_launch(const void* vector, const void* mix, int dtype, int B, int F, int D, int T,
                                    const void* grad_out, void* grad_vector, void* grad_mix, void* stream) {
  PBB_CHECK_ARG(vector && mix && grad_out, 1, "input is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 3, "bad dtype");
  PBB_CHECK_ARG(B > 0 && B <= 65535 && F > 0 && D > 0 && T > 0, 4, "bad shape");
  PBB_CHECK_ARG(grad_vector != nullptr || grad_mix != nullptr, 8, "both gradients are null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const double2* g = reinterpret_cast<const double2*>(grad_out);
  if (grad_vector) {
    const unsigned blocks = blocks_for((size_t)B * F * D * 32, 256);
    PBB_TRY(with_ct(dtype, [&](auto ct) {
      using CT = decltype(ct);
      return launch_kernel("apply_bf_vector_backward_kernel", apply_bf_vector_backward_kernel<CT>, blocks, 256, 0, st,
                           reinterpret_cast<const CT*>(mix), g, B, F, D, T, reinterpret_cast<double2*>(grad_vector));
    }));
  }
  if (grad_mix) {
    PBB_TRY(launch_kernel("apply_bf_mix_backward_kernel", apply_bf_mix_backward_kernel,
                          dim3((T + 255) / 256, F < 65535 ? F : 65535), 256, 0, st,
                          reinterpret_cast<const double2*>(vector), g, B, F, D, T,
                          reinterpret_cast<double2*>(grad_mix)));
  }
  return 0;
}

int pbb_apply_beamforming_vector_backward(const void* vector, const void* mix, int dtype, int F, int D, int T,
                                          const void* grad_out, void* grad_vector, void* grad_mix, void* stream) {
  return apply_bf_backward_launch(vector, mix, dtype, 1, F, D, T, grad_out, grad_vector, grad_mix, stream);
}

int pbb_apply_beamforming_vector_shared_backward(const void* vector, const void* mix, int dtype, int B, int F, int D,
                                                 int T, const void* grad_out, void* grad_vector, void* grad_mix,
                                                 void* stream) {
  return apply_bf_backward_launch(vector, mix, dtype, B, F, D, T, grad_out, grad_vector, grad_mix, stream);
}

// ---- multi-source beamformers and vector post-processing (csrc/extraction.cuh) ----------------------------------

int pbb_lcmv(const void* atf, const void* response, const void* noise_psd, int K, int F, int D, void* w,
             void* scratch, int* status, void* stream) {
  PBB_CHECK_ARG(atf != nullptr, 1, "atf is null");
  PBB_CHECK_ARG(response != nullptr, 2, "response is null");
  PBB_CHECK_ARG(noise_psd != nullptr, 3, "noise PSD is null");
  PBB_CHECK_ARG(K > 0 && K <= 64, 4, "need 0 < K <= 64");
  PBB_CHECK_ARG(F > 0, 5, "F must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 6, "need 0 < D <= 64");
  PBB_CHECK_ARG(w != nullptr, 7, "w is null");
  PBB_CHECK_ARG(scratch != nullptr, 8, "scratch (F * (2 * D * K + K * K + 2 * K) + 1 complex128) is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double2* H = reinterpret_cast<double2*>(scratch);
  double2* X = H + (size_t)F * D * K;
  double2* G = X + (size_t)F * D * K;
  double2* rhs = G + (size_t)F * K * K;
  double2* y = rhs + (size_t)F * K;
  int* fallback = reinterpret_cast<int*>(y + (size_t)F * K);
  PBB_CUDA(cudaMemsetAsync(fallback, 0, sizeof(int), st));
  PBB_TRY(launch_kernel("lcmv_rhs_kernel", lcmv_rhs_kernel, blocks_for((size_t)K * F * D, 256), 256, 0, st,
                        reinterpret_cast<const double2*>(atf), K, F, D, H));
  int r = solve_launch(noise_psd, H, F, D, K, 0, X, status, 0, st);  // Phi_N X = H, stable_solve (:432-435)
  if (r) return r;
  PBB_TRY(launch_kernel("lcmv_gram_kernel", lcmv_gram_kernel, blocks_for((size_t)F * K * K, 128), 128, 0, st,
                        reinterpret_cast<const double2*>(atf), X, reinterpret_cast<const double2*>(response), K, F, D,
                        G, rhs));
  r = solve_launch(G, rhs, F, K, 1, 0, y, status, 0, st, fallback);  // (H^H Phi_N^-1 H) y = r (:446-449)
  if (r) return r;
  return launch_kernel("lcmv_combine_kernel", lcmv_combine_kernel, blocks_for((size_t)F * D, 128), 128, 0, st, X, y,
                       fallback, K, F, D, reinterpret_cast<double2*>(w));
}

int pbb_wmwf(const void* target_psd, const void* noise_psd, int n, int D, int frequency_dependent,
             double distortion_weight, void* filter, void* scratch, int* status, void* stream) {
  PBB_CHECK_ARG(target_psd != nullptr, 1, "target PSD is null");
  PBB_CHECK_ARG(noise_psd != nullptr, 2, "noise PSD is null");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 4, "need 0 < D <= 64");
  PBB_CHECK_ARG(filter != nullptr, 7, "filter is null");
  PBB_CHECK_ARG(scratch != nullptr, 8, "scratch (n * D * D complex128) is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int r = solve_launch(noise_psd, target_psd, n, D, D, 0, scratch, status, 0, st);  // phi, stable_solve (:735)
  if (r) return r;
  return launch_kernel("wmwf_filter_kernel", wmwf_filter_kernel, blocks_for((size_t)n * D * D, 256), 256, 0, st,
                       reinterpret_cast<const double2*>(scratch), reinterpret_cast<const double2*>(target_psd), n, D,
                       frequency_dependent, distortion_weight, reinterpret_cast<double2*>(filter));
}

int pbb_weighted_channel_sum(const void* filter, const void* weight, int n, int D, void* out, void* stream) {
  PBB_CHECK_ARG(filter != nullptr, 1, "filter is null");
  PBB_CHECK_ARG(weight != nullptr, 2, "weight is null");
  PBB_CHECK_ARG(n > 0 && D > 0, 3, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("weighted_channel_sum_kernel", weighted_channel_sum_kernel, blocks_for((size_t)n * D, 256), 256,
                       0, st, reinterpret_cast<const double2*>(filter), reinterpret_cast<const double2*>(weight), n, D,
                       reinterpret_cast<double2*>(out));
}

int pbb_reference_channel_snr(const void* w_mat, const void* target_psd, const void* noise_psd, int n, int D,
                              void* num, void* den, void* num_sum, void* den_sum, void* stream) {
  PBB_CHECK_ARG(w_mat && target_psd && noise_psd, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(num && den && num_sum && den_sum, 6, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PBB_TRY(launch_kernel("reference_snr_kernel", reference_snr_kernel, n, 64, 0, st,
                        reinterpret_cast<const double2*>(w_mat), reinterpret_cast<const double2*>(target_psd),
                        reinterpret_cast<const double2*>(noise_psd), n, D, reinterpret_cast<double2*>(num),
                        reinterpret_cast<double2*>(den)));
  PBB_TRY(launch_kernel("colsum_kernel", colsum_kernel, 1, 128, 0, st, reinterpret_cast<const double*>(num),
                        reinterpret_cast<double*>(num_sum), n, 2 * D));
  return launch_kernel("colsum_kernel", colsum_kernel, 1, 128, 0, st, reinterpret_cast<const double*>(den),
                       reinterpret_cast<double*>(den_sum), n, 2 * D);
}

int pbb_mvdr_merl(const void* target_psd, const void* noise_psd, int n, int D, void* w, void* scratch, int* status,
                  void* stream) {
  PBB_CHECK_ARG(target_psd != nullptr, 1, "target PSD is null");
  PBB_CHECK_ARG(noise_psd != nullptr, 2, "noise PSD is null");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= 64, 4, "need 0 < D <= 64");
  PBB_CHECK_ARG(w != nullptr, 5, "w is null");
  PBB_CHECK_ARG(scratch != nullptr, 6, "scratch (n * D * D complex128) is null");
  PBB_CHECK_ARG(status != nullptr, 7, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int r = solve_launch(noise_psd, target_psd, n, D, D, 0, scratch, status, 1, st);  // np.linalg.solve (:277)
  if (r) return r;
  return launch_kernel("merl_kernel", merl_kernel, blocks_for(n, 128), 128, 0, st,
                       reinterpret_cast<const double2*>(scratch), n, D, reinterpret_cast<double2*>(w));
}

int pbb_condition_covariance(const void* x, int n, int D, double gamma, void* out, void* stream) {
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(n > 0 && D > 0, 2, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("condition_covariance_kernel", condition_covariance_kernel, blocks_for((size_t)n * D * D, 256),
                       256, 0, st, reinterpret_cast<const double2*>(x), n, D, gamma, reinterpret_cast<double2*>(out));
}

int pbb_distortionless_normalization(const void* vector, const void* atf, const void* noise_psd, int n, int D,
                                     void* out, void* stream) {
  PBB_CHECK_ARG(vector && atf && noise_psd, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 6, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("distortionless_kernel", distortionless_kernel, blocks_for(n, 128), 128, 0, st,
                       reinterpret_cast<const double2*>(vector), reinterpret_cast<const double2*>(atf),
                       reinterpret_cast<const double2*>(noise_psd), n, D, reinterpret_cast<double2*>(out));
}

int pbb_mvdr_snr_postfilter(const void* vector, const void* target_psd, const void* noise_psd, int n, int D,
                            void* out, void* stream) {
  PBB_CHECK_ARG(vector && target_psd && noise_psd, 1, "input is null");
  PBB_CHECK_ARG(n > 0 && D > 0 && D <= 64, 4, "bad shape");
  PBB_CHECK_ARG(out != nullptr, 6, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("snr_postfilter_kernel", snr_postfilter_kernel, blocks_for(n, 128), 128, 0, st,
                       reinterpret_cast<const double2*>(vector), reinterpret_cast<const double2*>(target_psd),
                       reinterpret_cast<const double2*>(noise_psd), n, D, reinterpret_cast<double2*>(out));
}

int pbb_zero_degree_normalization(const void* vector, int n, int D, int reference_channel, void* out, void* stream) {
  PBB_CHECK_ARG(vector != nullptr, 1, "vector is null");
  PBB_CHECK_ARG(n > 0 && D > 0, 2, "bad shape");
  PBB_CHECK_ARG(reference_channel >= 0 && reference_channel < D, 4, "need 0 <= reference_channel < D");
  PBB_CHECK_ARG(out != nullptr, 5, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("zero_degree_kernel", zero_degree_kernel, blocks_for((size_t)n * D, 256), 256, 0, st,
                       reinterpret_cast<const double2*>(vector), n, D, reference_channel,
                       reinterpret_cast<double2*>(out));
}

int pbb_phase_correction(const void* vector, int A, int M, int F, int D, int scan_bins, void* out, void* stream) {
  PBB_CHECK_ARG(vector != nullptr, 1, "vector is null");
  PBB_CHECK_ARG(A > 0 && M > 0 && F > 0 && D > 0, 2, "bad shape");
  PBB_CHECK_ARG(!scan_bins || (A == 1 && M == 1), 6, "scan_bins needs A = M = 1");
  PBB_CHECK_ARG(out != nullptr, 7, "out is null");
  PBB_CHECK_ARG(out != vector, 7, "out must not alias vector");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t threads = scan_bins ? 1 : (size_t)M * F;
  return launch_kernel("phase_correction_kernel", phase_correction_kernel, blocks_for(threads, 128), 128, 0, st,
                       reinterpret_cast<const double2*>(vector), A, M, F, D, scan_bins,
                       reinterpret_cast<double2*>(out));
}

int pbb_apply_online_beamforming_vector(const void* vector, const void* mix, int dtype, int B, int F, int D, int T,
                                        long long vector_frame_stride, long long vector_bin_stride,
                                        long long mix_batch_stride, long long mix_bin_stride, void* out,
                                        void* stream) {
  PBB_CHECK_ARG(vector && mix, 1, "input is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 3, "bad dtype");
  PBB_CHECK_ARG(B > 0 && F > 0 && F <= 65535 && D > 0 && T > 0, 4, "bad shape");
  PBB_CHECK_ARG(vector_frame_stride >= 0 && vector_bin_stride >= 0 && mix_batch_stride >= 0 && mix_bin_stride >= 0,
                8, "strides must be non-negative");
  PBB_CHECK_ARG(out != nullptr, 12, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid((T + 127) / 128, F);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("apply_online_kernel", apply_online_kernel<CT>, grid, 128, 0, st,
                         reinterpret_cast<const double2*>(vector), reinterpret_cast<const CT*>(mix), B, F, D, T,
                         vector_frame_stride, vector_bin_stride, mix_batch_stride, mix_bin_stride,
                         reinterpret_cast<double2*>(out));
  });
}

// ---- single distributions of pb_bss/distribution (csrc/distribution.cuh) -----------------------------------------

int pbb_cacg_from_covariance(const void* covariance, int n, int D, int covariance_norm, double eigenvalue_floor,
                             void* eigenvectors, double* eigenvalues, int* status, void* stream) {
  PBB_CHECK_ARG(covariance != nullptr, 1, "covariance is null");
  PBB_CHECK_ARG(n > 0, 2, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= kDistMaxD, 3, "need 0 < D <= 64");
  PBB_CHECK_ARG(covariance_norm >= PBB_NORM_NONE && covariance_norm <= PBB_NORM_TRACE, 4, "bad covariance_norm");
  PBB_CHECK_ARG(eigenvectors != nullptr && eigenvalues != nullptr, 6, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t per = from_covariance_smem_per_warp(D);
  const int warps = warps_for(per);
  if (status) PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  PBB_CUDA(cudaFuncSetAttribute(cacg_from_covariance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return launch_kernel("cacg_from_covariance_kernel", cacg_from_covariance_kernel, (n + warps - 1) / warps, 32 * warps,
                       per * warps, st, reinterpret_cast<const double2*>(covariance), n, D, covariance_norm,
                       eigenvalue_floor, reinterpret_cast<double2*>(eigenvectors), eigenvalues, status, warps);
}

int pbb_cw_log_norm(const double* kappa, long long n, int D, int variant, double* log_norm, void* stream) {
  PBB_CHECK_ARG(kappa != nullptr, 1, "kappa is null");
  PBB_CHECK_ARG(n > 0, 2, "n must be positive");
  PBB_CHECK_ARG(D > 0 && D <= kDistMaxD, 3, "need 0 < D <= 64");
  PBB_CHECK_ARG(variant >= PBB_CW_NORM_1F1 && variant <= PBB_CW_NORM_TRAN_VU, 4, "bad variant");
  PBB_CHECK_ARG(log_norm != nullptr, 5, "log_norm is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("cw_log_norm_kernel", cw_log_norm_kernel, blocks_for((size_t)n, 256), 256, 0, st, kappa, n, D,
                       variant, log_norm);
}

int pbb_cw_log_pdf(const void* y, int dtype, long long y_stride, int M, int N, int D, const void* mode,
                   const double* concentration, double* log_pdf, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "bad dtype");
  PBB_CHECK_ARG(y_stride >= 0, 3, "y_stride must be non-negative");
  PBB_CHECK_ARG(M > 0 && N > 0 && D > 0 && D <= kDistMaxD, 4, "bad shape");
  PBB_CHECK_ARG(mode != nullptr && concentration != nullptr, 7, "model is null");
  PBB_CHECK_ARG(log_pdf != nullptr, 9, "log_pdf is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(blocks_for((size_t)N, 256), std::min(M, kDistMaxGridY));
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("cw_log_pdf_kernel", cw_log_pdf_kernel<CT>, grid, 256, 0, st, reinterpret_cast<const CT*>(y),
                         y_stride, M, N, D, reinterpret_cast<const double2*>(mode), concentration, log_pdf);
  });
}

// workspace of pbb_ccsg_log_pdf (LU (M, D, D) | perm (M, D) | logdet (M)) and of pbb_ccsg_sample (L (M, D, D))
size_t pbb_ccsg_workspace_bytes(int M, int D) {
  if (M <= 0 || D <= 0 || D > kDistMaxD) return 0;
  const size_t lu = (size_t)M * D * D * sizeof(double2);
  const size_t perm = ((size_t)M * D * sizeof(int) + 15) & ~(size_t)15;
  return lu + perm + (size_t)M * sizeof(double);
}

int pbb_ccsg_log_pdf(const void* y, int dtype, long long y_stride, int M, int N, int D, const void* covariance,
                     double* log_pdf, void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "bad dtype");
  PBB_CHECK_ARG(y_stride >= 0, 3, "y_stride must be non-negative");
  PBB_CHECK_ARG(M > 0 && N > 0 && D > 0 && D <= kDistMaxD, 4, "bad shape");
  PBB_CHECK_ARG(covariance != nullptr, 7, "covariance is null");
  PBB_CHECK_ARG(log_pdf != nullptr, 8, "log_pdf is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_ccsg_workspace_bytes(M, D), 9,
                "workspace too small (pbb_ccsg_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 11, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double2* lu = reinterpret_cast<double2*>(workspace);
  int* perm = reinterpret_cast<int*>(lu + (size_t)M * D * D);
  double* logdet = reinterpret_cast<double*>(reinterpret_cast<char*>(perm) +
                                             (((size_t)M * D * sizeof(int) + 15) & ~(size_t)15));
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  // one factorisation per warp: as many warps per CTA as their shared memory allows (one at D = 64)
  const size_t lu_per_warp = (size_t)D * D * sizeof(double2) + kDistMaxD * sizeof(int);
  const int warps = warps_for(lu_per_warp);
  const size_t lu_smem = (size_t)warps * lu_per_warp;
  PBB_CUDA(cudaFuncSetAttribute(ccsg_lu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  PBB_TRY(launch_kernel("ccsg_lu_kernel", ccsg_lu_kernel, (M + warps - 1) / warps, 32 * warps, lu_smem, st,
                        reinterpret_cast<const double2*>(covariance), M, D, lu, perm, logdet, status, warps));
  const size_t smem = ccsg_log_pdf_smem(D);
  const dim3 grid(blocks_for((size_t)N, kCcsgThreads), std::min(M, kDistMaxGridY));
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    PBB_CUDA(cudaFuncSetAttribute(ccsg_log_pdf_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return launch_kernel("ccsg_log_pdf_kernel", ccsg_log_pdf_kernel<CT>, grid, kCcsgThreads, smem, st,
                         reinterpret_cast<const CT*>(y), y_stride, M, N, D, lu, perm, logdet, log_pdf);
  });
}

int pbb_ccsg_sample(const void* a, const double* eigenvalues, int C, int D, const double* normals,
                    const long long* offsets, const long long* dest, long long S, int unit_norm, void* out,
                    void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(a != nullptr, 1, "covariance / eigenvectors are null");
  PBB_CHECK_ARG(C > 0 && D > 0 && D <= kDistMaxD, 3, "bad shape");
  PBB_CHECK_ARG(S >= 0, 8, "S must be non-negative");
  PBB_CHECK_ARG(S == 0 || (normals != nullptr && offsets != nullptr && out != nullptr), 5, "samples are null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_ccsg_workspace_bytes(C, D), 11,
                "workspace too small (pbb_ccsg_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 13, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double2* L = reinterpret_cast<double2*>(workspace);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  const size_t chol_per_warp = (size_t)D * D * sizeof(double2);
  const int warps = warps_for(chol_per_warp);
  PBB_CUDA(cudaFuncSetAttribute(ccsg_cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  PBB_TRY(launch_kernel("ccsg_cholesky_kernel", ccsg_cholesky_kernel, (C + warps - 1) / warps, 32 * warps,
                        (size_t)warps * chol_per_warp, st, reinterpret_cast<const double2*>(a), eigenvalues, C, D, L,
                        status, warps));
  if (S == 0) return 0;
  return launch_kernel("ccsg_sample_kernel", ccsg_sample_kernel, blocks_for((size_t)S, 128), 128, 0, st, L, C, D,
                       normals, offsets, dest, S, unit_norm, reinterpret_cast<double2*>(out));
}

int pbb_ccsg_fit(const void* observation, int dtype, int F, int D, int N, const double* saliency,
                 double denominator_floor, void* covariance, void* workspace, size_t workspace_bytes, void* stream) {
  int r = pbb_power_spectral_density(observation, dtype, F, D, N, saliency, 1, 0, covariance, workspace,
                                     workspace_bytes, stream);
  if (r || saliency == nullptr) return r;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("ccsg_fit_scale_kernel", ccsg_fit_scale_kernel, F, 256, 0, st, saliency, N, D, denominator_floor,
                       reinterpret_cast<double2*>(covariance));
}

}  // extern "C"
