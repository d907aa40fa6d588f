// C-ABI entry points for the integrated spatial + spectral mixture model (pb_bss/distribution/gcacgmm.py: the cACG
// of the multi-channel observation combined with a Gaussian over per-(bin, frame) embedding vectors) -- see
// include/pbb.h.  The spatial part reuses the cACGMM kernels (quadratic form, M-step, eigendecomposition); this
// unit adds the small HBM-streaming pieces around them:
//   pbb_cacg_log_pdf              -D log q - sum log lambda                      (cacg.py:198-201)
//   pbb_gaussian_log_pdf          diagonal / spherical Gaussian over (F, T, E)   (gaussian.py:57-135)
//   pbb_gaussian_fit              weighted mean + variance, two passes           (gaussian.py:155-193)
//   pbb_log_pdf_to_affiliation    softmax * weight, clip (mixture_model_utils.py:7-55), optionally after the
//                                 per-bin search over the K! pairings of spatial and spectral classes (:58-130)
// and the batched pieces of the embedding mixture models GMM / VMFMM (gmm.py, vmfmm.py), B independent models:
//   pbb_gaussian_full_log_pdf     full-covariance Gaussian, the reference's U d form (gaussian.py:36-56)
//   pbb_gaussian_full_fit         weighted mean + full scatter, N split over CTAs (gaussian.py:152-193)
//   pbb_precision_cholesky        sklearn's precision Cholesky + log det, one warp per matrix
//   pbb_vmf_log_pdf / pbb_vmf_resultant
// All reductions run in a fixed order (bit-reproducible).
#include <cstring>

#include "common.cuh"
#include "em_args.cuh"
#include "prof.cuh"

namespace pbb {

constexpr int kIntMaxK = 6;    // K! permutations are enumerated per bin
constexpr int kIntMaxE = 64;   // embedding dimension held in registers / shared memory

__device__ inline double block_sum_256(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  return s;
}

// q_out (may be null, never q) receives the floored quadratic form
__global__ void cacg_log_pdf_kernel(const double* __restrict__ q, const double* __restrict__ eigenvalues, int F, int K,
                                    int T, int D, double* __restrict__ out, double q_floor = kTiny,
                                    double* __restrict__ q_out = nullptr) {
  const int fk = blockIdx.y;
  double ld = 0.0;
  for (int d = 0; d < D; ++d) ld += log(eigenvalues[(size_t)fk * D + d]);
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const double qq = fmax(fabs(q[(size_t)fk * T + t]), q_floor);
  if (q_out) q_out[(size_t)fk * T + t] = qq;
  out[(size_t)fk * T + t] = -(double)D * log(qq) - ld;
}

// out[f][k][t] = -E/2 log(2 pi) + log_det[k] - 1/2 sum_e (pc[k][e] (x[f][t][e] - mean[k][e]))^2           (spherical)
// diagonal != 0: the reference's DiagonalGaussian.log_pdf contracts its (K, E) precision_cholesky with the einsum
// '...dD,...nD->...nd' (gaussian.py:79-87), i.e. white[k][n][d] = sum_e pc[d][e] (x[n][e] - mean[k][e]) with d running
// over the CLASSES, and log_pdf = ... - 1/2 sum_d white^2.  A drop-in has to return what the reference returns, so this
// branch evaluates exactly that expression.
__global__ void gaussian_log_pdf_kernel(const double* __restrict__ x, const double* __restrict__ mean,
                                        const double* __restrict__ pc, const double* __restrict__ log_det, int F, int T,
                                        int E, int K, int diagonal, double* __restrict__ out) {
  extern __shared__ double sm[];  // mean [K][E], pc [K][E]
  for (int i = threadIdx.x; i < 2 * K * E; i += blockDim.x) sm[i] = i < K * E ? mean[i] : pc[i - K * E];
  __syncthreads();
  const int f = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const double* __restrict__ xr = x + ((size_t)f * T + t) * E;
  double xe[kIntMaxE];
  for (int e = 0; e < E; ++e) xe[e] = xr[e];
  const double c0 = -0.5 * (double)E * log(2.0 * 3.14159265358979323846);
  for (int k = 0; k < K; ++k) {
    double s = 0.0;
    if (diagonal == 2) {
      // von Mises-Fisher (von_mises_fisher.py:66-81): concentration * <mean, x / max(||x||, tiny)> - log_norm;
      // pc[k][0] = concentration, log_det[k] = log_norm
      double dot = 0.0, n2 = 0.0;
      for (int e = 0; e < E; ++e) { dot += sm[k * E + e] * xe[e]; n2 += xe[e] * xe[e]; }
      out[((size_t)f * K + k) * T + t] = sm[K * E + k * E] * (dot / fmax(sqrt(n2), kTiny)) - log_det[k];
      continue;
    }
    if (diagonal) {
      for (int d = 0; d < K; ++d) {
        double w = 0.0;
        for (int e = 0; e < E; ++e) w += sm[K * E + d * E + e] * (xe[e] - sm[k * E + e]);
        s += w * w;
      }
    } else {
      for (int e = 0; e < E; ++e) {
        const double w = sm[K * E + k * E + e] * (xe[e] - sm[k * E + e]);
        s += w * w;
      }
    }
    out[((size_t)f * K + k) * T + t] = c0 + log_det[k] - 0.5 * s;
  }
}

// pass 0: partial[f][k][0..E) = sum_t w x, [E] = sum_t w ; pass 1: partial[f][k][0..E) = sum_t w (x - mean)^2
__global__ void gaussian_fit_partial_kernel(const double* __restrict__ x, const double* __restrict__ w,
                                            const double* __restrict__ mean, int F, int T, int E, int K, int pass,
                                            double* __restrict__ partial) {
  __shared__ double red[8];
  const int f = blockIdx.x, k = blockIdx.y;
  const double* __restrict__ wr = w + ((size_t)f * K + k) * T;
  for (int e = 0; e <= E; ++e) {
    if (pass == 1 && e == E) break;
    double s = 0.0;
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
      const double ww = wr[t];
      if (e == E) s += ww;
      else {
        const double xv = x[((size_t)f * T + t) * E + e];
        if (pass == 0) s += ww * xv;
        else { const double d = xv - mean[k * E + e]; s += ww * d * d; }
      }
    }
    s = block_sum_256(s, red);
    if (threadIdx.x == 0) partial[((size_t)f * K + k) * (E + 1) + e] = s;
  }
}
// mean[k][e] = sum_f partial / max(denominator, tiny); the unclamped denominator sum_t w is kept in denom[k]: the
// von Mises-Fisher fit divides by it as it is (von_mises_fisher.py:137)
__global__ void gaussian_fit_mean_kernel(const double* __restrict__ partial, int F, int E, int K,
                                         double* __restrict__ mean, double* __restrict__ denom) {
  const int k = blockIdx.x, e = threadIdx.x;
  if (e > E) return;
  double s = 0.0;
  for (int f = 0; f < F; ++f) s += partial[((size_t)f * K + k) * (E + 1) + e];
  __shared__ double den;
  if (e == E) { den = fmax(s, kTiny); denom[k] = s; }
  __syncthreads();
  if (e < E) mean[k * E + e] = s / den;
}
// covariance: diagonal (K, E) or spherical (K)
__global__ void gaussian_fit_cov_kernel(const double* __restrict__ partial, const double* __restrict__ denom, int F, int E,
                                        int K, int spherical, double* __restrict__ cov) {
  const int k = blockIdx.x, e = threadIdx.x;
  __shared__ double v[kIntMaxE];
  if (e < E) {
    double s = 0.0;
    for (int f = 0; f < F; ++f) s += partial[((size_t)f * K + k) * (E + 1) + e];
    v[e] = s;
    if (!spherical) cov[k * E + e] = s / fmax(denom[k], kTiny);
  }
  __syncthreads();
  if (spherical && e == 0) {
    double s = 0.0;
    for (int i = 0; i < E; ++i) s += v[i];
    cov[k] = s / (fmax(denom[k], kTiny) * (double)E);
  }
}

__device__ __forceinline__ double weight_of(const double* __restrict__ w, int mode, int f, int k, int t, int K, int T) {
  if (mode >= PBB_WEIGHT_BCAST) {  // (F', K', T') with stride 0 along the dims whose bit is clear
    const int kn = mode & 2 ? K : 1, tn = mode & 4 ? T : 1;
    return w[((size_t)(mode & 1 ? f : 0) * kn + (mode & 2 ? k : 0)) * tn + (mode & 4 ? t : 0)];
  }
  switch (mode) {
    case PBB_WEIGHT_CONST: return 1.0 / K;
    case PBB_WEIGHT_TIED_TIME: return w[(size_t)k * T + t];
    case PBB_WEIGHT_TIED: return w[k];
    case PBB_WEIGHT_FRAME: return w[(size_t)f * T + t];
    default: return w[(size_t)f * K + k];
  }
}

// One CTA per bin.  lp[k][t] = sa * a[f][perm(k)][t] + sb * b[f][k][t]; perm = identity, or (inline_pa) the first of
// itertools.permutations(range(K)) that maximises sum_{k,t} softmax_k(lp) * lp (mixture_model_utils.py:93-115).
__global__ void __launch_bounds__(256) log_pdf_to_affiliation_kernel(
    const double* __restrict__ a, const double* __restrict__ b, double sa, double sb, const double* __restrict__ weight,
    int weight_mode, const uint8_t* __restrict__ activity, double eps, int inline_pa, int F, int K, int T,
    double* __restrict__ out, int* __restrict__ chosen) {
  __shared__ double red[8];
  __shared__ int best_perm[kIntMaxK];
  const int f = blockIdx.x, tid = threadIdx.x;
  const double* __restrict__ af = a + (size_t)f * K * T;
  const double* __restrict__ bf = b ? b + (size_t)f * K * T : nullptr;
  int perm[kIntMaxK];
  for (int k = 0; k < K; ++k) perm[k] = k;
  if (inline_pa && bf != nullptr) {
    int cand[kIntMaxK];
    for (int k = 0; k < K; ++k) cand[k] = k;
    double best = -INFINITY;
    bool have = false;
    while (true) {
      double aux = 0.0;
      for (int t = tid; t < T; t += blockDim.x) {
        double lp[kIntMaxK], m = -INFINITY;
        for (int k = 0; k < K; ++k) { lp[k] = sa * af[(size_t)cand[k] * T + t] + sb * bf[(size_t)k * T + t]; m = fmax(m, lp[k]); }
        double den = 0.0, ex[kIntMaxK];
        for (int k = 0; k < K; ++k) { ex[k] = exp(lp[k] - m); den += ex[k]; }
        den = fmax(den, kTiny);
        for (int k = 0; k < K; ++k) aux += (ex[k] / den) * lp[k];
      }
      aux = block_sum_256(aux, red);
      if (!have || aux > best) {
        best = aux; have = true;
        for (int k = 0; k < K; ++k) perm[k] = cand[k];
      }
      int i = K - 2;  // next lexicographic permutation
      while (i >= 0 && cand[i] > cand[i + 1]) --i;
      if (i < 0) break;
      int j = K - 1;
      while (cand[j] < cand[i]) --j;
      { const int tmp = cand[i]; cand[i] = cand[j]; cand[j] = tmp; }
      for (int x = i + 1, y = K - 1; x < y; ++x, --y) { const int tmp = cand[x]; cand[x] = cand[y]; cand[y] = tmp; }
    }
    if (tid == 0 && chosen != nullptr)
      for (int k = 0; k < K; ++k) chosen[(size_t)f * K + k] = perm[k];
  }
  (void)best_perm;
  for (int t = tid; t < T; t += blockDim.x) {
    double lp[kIntMaxK], m = -INFINITY;
    for (int k = 0; k < K; ++k) {
      lp[k] = sa * af[(size_t)perm[k] * T + t] + (bf ? sb * bf[(size_t)k * T + t] : 0.0);
      m = fmax(m, lp[k]);
    }
    double g[kIntMaxK], den = 0.0;
    for (int k = 0; k < K; ++k) {
      g[k] = exp(lp[k] - m) * weight_of(weight, weight_mode, f, k, t, K, T);
      if (activity != nullptr && !activity[((size_t)f * K + k) * T + t]) g[k] = 0.0;
      den += g[k];
    }
    den = fmax(den, kTiny);
    for (int k = 0; k < K; ++k) {
      double v = g[k] / den;
      if (eps != 0.0) v = fmin(fmax(v, eps), 1.0 - eps);
      out[((size_t)f * K + k) * T + t] = v;
    }
  }
}

// ---- embedding mixture models with independent leading dims: B models, each (K, E[, E]) over N observations ----

// Full-covariance Gaussian.log_pdf (gaussian.py:36-56) with the reference's einsum '...dD,...nD->...nd': white = U d
// (sklearn's own log pdf uses U^T d), so the quadratic form is d^T U^T U d.  One thread per observation; the centred
// row d lives in EM registers, U_k (upper triangle, the rest is zero) and mean_k are staged in shared memory per class.
template <int EM>
__global__ void __launch_bounds__(128) gaussian_full_log_pdf_kernel(
    const double* __restrict__ x, const double* __restrict__ mean, const double* __restrict__ U,
    const double* __restrict__ log_det, int N, int E, int K, double* __restrict__ out) {
  extern __shared__ double sm[];  // U_k [E][E], mean_k [E]
  double* us = sm;
  double* ms = sm + E * E;
  const int b = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  const double c0 = -0.5 * (double)E * log(2.0 * 3.14159265358979323846);
  const double* __restrict__ xr = x + ((size_t)b * N + (n < N ? n : 0)) * E;
  for (int k = 0; k < K; ++k) {
    const size_t bk = (size_t)b * K + k;
    __syncthreads();
    for (int i = threadIdx.x; i < E * E; i += blockDim.x) us[i] = U[bk * E * E + i];
    for (int i = threadIdx.x; i < E; i += blockDim.x) ms[i] = mean[bk * E + i];
    __syncthreads();
    if (n >= N) continue;
    double d[EM];
#pragma unroll
    for (int j = 0; j < EM; ++j) d[j] = j < E ? xr[j] - ms[j] : 0.0;
    double s = 0.0;
    for (int i = 0; i < E; ++i) {
      double w = 0.0;
#pragma unroll
      for (int j = 0; j < EM; ++j)
        if (j >= i && j < E) w += us[i * E + j] * d[j];
      s += w * w;
    }
    out[bk * N + n] = c0 + log_det[bk] - 0.5 * s;
  }
}

constexpr int kFitTileN = 32;       // observations staged in shared memory per step
constexpr int kFitThreads = 256;
constexpr int kFitMaxAcc = (kIntMaxE * (kIntMaxE + 1) / 2 + kFitThreads - 1) / kFitThreads;
constexpr int kFitTargetCtas = 528;  // 4 per SM of a 132-SM H100; the chunking depends on the shape only

__host__ __device__ inline int fit_entries(int E) { return E * (E + 1) / 2 > E + 1 ? E * (E + 1) / 2 : E + 1; }

// Weighted moments of one chunk of observations for one (b, k); xs holds the staged rows plus a column E of ones, so
// both passes are acc += w * xs[n][i] * xs[n][j]:
//   pass 0: entry e < E: (i, j) = (e, E) -> sum w x_e;  entry E: (E, E) -> sum w.  normalize != 0 stages the rows as
//           x / max(||x||, tiny) (the von Mises-Fisher trainer's observations, von_mises_fisher.py:106-109)
//   pass 1: entry p = packed upper triangle (i <= j, row-major): sum w (x_i - mean_i)(x_j - mean_j)
// partial[c][bk][entry].  Every chunk has a fixed range of observations and a fixed thread order: bit-reproducible.
__global__ void __launch_bounds__(kFitThreads, 1) gaussian_full_partial_kernel(
    const double* __restrict__ x, const double* __restrict__ w, const double* __restrict__ mean, int N, int E, int K,
    int chunk_len, int pass, int normalize, double* __restrict__ partial) {
  __shared__ double xs[kFitTileN][kIntMaxE + 1];
  __shared__ double ws[kFitTileN];
  const int c = blockIdx.x, bk = blockIdx.y, b = bk / K, tid = threadIdx.x;
  const int P = pass == 0 ? E + 1 : E * (E + 1) / 2;
  int ij[kFitMaxAcc];  // i | j << 8
  double acc[kFitMaxAcc];
#pragma unroll
  for (int r = 0; r < kFitMaxAcc; ++r) {
    const int p = tid + r * kFitThreads;
    acc[r] = 0.0;
    ij[r] = 0;
    if (p < P) {
      if (pass == 0) ij[r] = p | E << 8;
      else {
        int i = 0, off = 0;
        while (off + (E - i) <= p) { off += E - i; ++i; }
        ij[r] = i | (i + (p - off)) << 8;
      }
    }
  }
  const double* __restrict__ xb = x + (size_t)b * N * E;
  const double* __restrict__ wb = w + (size_t)bk * N;
  const int n_begin = c * chunk_len, n_end = min(N, n_begin + chunk_len);
  for (int n0 = n_begin; n0 < n_end; n0 += kFitTileN) {
    const int rows = min(kFitTileN, n_end - n0);
    __syncthreads();
    for (int idx = tid; idx < kFitTileN * E; idx += kFitThreads) {
      const int r = idx / E, e = idx - r * E;
      double v = r < rows ? xb[(size_t)(n0 + r) * E + e] : 0.0;
      if (pass == 1) v -= mean[(size_t)bk * E + e];
      xs[r][e] = v;
    }
    if (tid < kFitTileN) { xs[tid][E] = 1.0; ws[tid] = tid < rows ? wb[n0 + tid] : 0.0; }
    __syncthreads();
    if (normalize) {
      if (tid < kFitTileN) {
        double n2 = 0.0;
        for (int e = 0; e < E; ++e) n2 += xs[tid][e] * xs[tid][e];
        const double nrm = fmax(sqrt(n2), kTiny);
        for (int e = 0; e < E; ++e) xs[tid][e] /= nrm;
      }
      __syncthreads();
    }
    for (int r = 0; r < rows; ++r) {
      const double wr = ws[r];
#pragma unroll
      for (int a = 0; a < kFitMaxAcc; ++a)
        if (tid + a * kFitThreads < P) acc[a] += wr * xs[r][ij[a] & 255] * xs[r][ij[a] >> 8];
    }
  }
  const size_t BK = gridDim.y;
#pragma unroll
  for (int a = 0; a < kFitMaxAcc; ++a) {
    const int p = tid + a * kFitThreads;
    if (p < P) partial[((size_t)c * BK + bk) * P + p] = acc[a];
  }
}

// Sums the chunks in chunk order.  pass 0: denom[bk] = max(sum w, tiny), mean = sum w x / denom (if mean != null);
// resultant = sum w x and total = sum w unscaled (if resultant != null).  pass 1: covariance[bk] = scatter / denom,
// both triangles.
__global__ void __launch_bounds__(kFitThreads) gaussian_full_reduce_kernel(
    const double* __restrict__ partial, int nchunks, int E, int pass, double* __restrict__ denom,
    double* __restrict__ mean, double* __restrict__ resultant, double* __restrict__ total,
    double* __restrict__ covariance) {
  __shared__ double den;
  const int bk = blockIdx.x, BK = gridDim.x, tid = threadIdx.x;
  const int P = pass == 0 ? E + 1 : E * (E + 1) / 2;
  for (int p0 = 0; p0 < P; p0 += kFitThreads) {
    const int p = p0 + tid;
    double s = 0.0;
    if (p < P)
      for (int c = 0; c < nchunks; ++c) s += partial[((size_t)c * BK + bk) * P + p];
    if (pass == 0) {  // P = E + 1 <= 65: a single round
      if (p == E) {
        den = fmax(s, kTiny);
        denom[bk] = den;
        if (total) total[bk] = s;
      }
      __syncthreads();
      if (p < E) {
        if (mean) mean[(size_t)bk * E + p] = s / den;
        if (resultant) resultant[(size_t)bk * E + p] = s;
      }
    } else if (p < P) {
      int i = 0, off = 0;
      while (off + (E - i) <= p) { off += E - i; ++i; }
      const int j = i + (p - off);
      const double v = s / denom[bk];
      covariance[((size_t)bk * E + i) * E + j] = v;
      covariance[((size_t)bk * E + j) * E + i] = v;
    }
  }
}

// sklearn's _compute_precision_cholesky(covariance, 'full') (gaussian.py:26-34): L = cholesky(Sigma) (lower triangle
// read, LAPACK potrf order), U = (L^-1)^T, log_det = sum log diag U.  One warp per matrix, L in shared memory; lane j
// solves column j of L^-1 and keeps it in row j of U.  A pivot that is not > 0 (or NaN) stops the matrix and records
// 1 + its index in *status (the smallest failing index wins).
__global__ void __launch_bounds__(32) precision_cholesky_kernel(const double* __restrict__ cov, int E,
                                                                double* __restrict__ U, double* __restrict__ log_det,
                                                                int* __restrict__ status) {
  extern __shared__ double L[];  // [E][E]
  const int m = blockIdx.x, lane = threadIdx.x;
  const double* __restrict__ A = cov + (size_t)m * E * E;
  double* __restrict__ Um = U + (size_t)m * E * E;
  for (int i = lane; i < E * E; i += 32) L[i] = A[i];
  __syncwarp();
  for (int j = 0; j < E; ++j) {
    double djj = L[j * E + j];
    for (int k = 0; k < j; ++k) djj -= L[j * E + k] * L[j * E + k];
    if (!(djj > 0.0)) {
      if (lane == 0) {
        int old = atomicCAS(status, 0, m + 1);
        while (old != 0 && old > m + 1) {
          const int seen = atomicCAS(status, old, m + 1);
          if (seen == old) break;
          old = seen;
        }
        log_det[m] = NAN;
      }
      for (int i = lane; i < E * E; i += 32) Um[i] = NAN;
      return;
    }
    const double ljj = sqrt(djj);
    for (int i = j + 1 + lane; i < E; i += 32) {
      double v = L[i * E + j];
      for (int k = 0; k < j; ++k) v -= L[i * E + k] * L[j * E + k];
      L[i * E + j] = v / ljj;
    }
    __syncwarp();
    if (lane == 0) L[j * E + j] = ljj;
    __syncwarp();
  }
  for (int j = lane; j < E; j += 32) {  // column j of X = L^-1 (forward substitution on e_j) -> row j of U
    double* __restrict__ uj = Um + (size_t)j * E;
    for (int i = 0; i < j; ++i) uj[i] = 0.0;
    for (int i = j; i < E; ++i) {
      double v = i == j ? 1.0 : 0.0;
      for (int k = j; k < i; ++k) v -= L[i * E + k] * uj[k];
      uj[i] = v / L[i * E + i];
    }
  }
  __syncwarp();
  if (lane == 0) {
    double s = 0.0;
    for (int i = 0; i < E; ++i) s += log(Um[(size_t)i * E + i]);
    log_det[m] = s;
  }
}

// VonMisesFisher.log_pdf (von_mises_fisher.py:65-79) for B models: out[b][k][n] = concentration[b][k]
// <mean[b][k], x / max(||x||, tiny)> - log_norm[b][k].
template <bool EXP>
__global__ void __launch_bounds__(128) vmf_log_pdf_kernel(const double* __restrict__ x, const double* __restrict__ mean,
                                                          const double* __restrict__ concentration,
                                                          const double* __restrict__ log_norm, int N, int E, int K,
                                                          double* __restrict__ out) {
  __shared__ double ms[kIntMaxK * kIntMaxE];
  const int b = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  for (int i = threadIdx.x; i < K * E; i += blockDim.x) ms[i] = mean[(size_t)b * K * E + i];
  __syncthreads();
  if (n >= N) return;
  const double* __restrict__ xr = x + ((size_t)b * N + n) * E;
  double dot[kIntMaxK], n2 = 0.0;
#pragma unroll
  for (int k = 0; k < kIntMaxK; ++k) dot[k] = 0.0;
  for (int e = 0; e < E; ++e) {
    const double v = xr[e];
    n2 += v * v;
#pragma unroll
    for (int k = 0; k < kIntMaxK; ++k)
      if (k < K) dot[k] += v * ms[k * E + e];
  }
  const double nrm = fmax(sqrt(n2), kTiny);
#pragma unroll
  for (int k = 0; k < kIntMaxK; ++k)
    if (k < K) {
      const size_t bk = (size_t)b * K + k;
      const double lp = concentration[bk] * (dot[k] / nrm) - log_norm[bk];
      out[bk * N + n] = EXP ? exp(lp) : lp;  // EXP: VonMisesFisher.pdf
    }
}

struct FullFitChunks { int nchunks, chunk_len; };
inline FullFitChunks full_fit_chunks(int B, int N, int K) {
  const long long BK = (long long)B * K;
  const int tiles = (N + kFitTileN - 1) / kFitTileN;
  long long want = (kFitTargetCtas + BK - 1) / BK;
  if (want > tiles) want = tiles;
  if (want < 1) want = 1;
  const int per = (int)((tiles + want - 1) / want);
  FullFitChunks c;
  c.chunk_len = per * kFitTileN;
  c.nchunks = (N + c.chunk_len - 1) / c.chunk_len;
  return c;
}

template <bool EXP>
static int vmf_log_pdf_launch(const double* embedding, const double* mean, const double* concentration,
                              const double* log_norm, int B, int N, int E, int K, double* out, void* stream) {
  PBB_CHECK_ARG(embedding && mean && concentration && log_norm, 1, "input is null");
  PBB_CHECK_ARG(B > 0 && B <= 65535 && N > 0, 5, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 7, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && K <= kIntMaxK, 8, "need 0 < K <= 6");
  PBB_CHECK_ARG(out != nullptr, 9, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel(EXP ? "vmf_pdf_kernel" : "vmf_log_pdf_kernel", vmf_log_pdf_kernel<EXP>, dim3((N + 127) / 128, B),
                       128, 0, st, embedding, mean, concentration, log_norm, N, E, K, out);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

int pbb_cacg_log_pdf(const double* quadratic, const double* eigenvalues, int F, int K, int T, int D, double* log_pdf,
                     void* stream) {
  PBB_CHECK_ARG(quadratic && eigenvalues, 1, "input is null");
  PBB_CHECK_ARG(F > 0 && K > 0 && T > 0 && D > 0, 3, "bad shape");
  PBB_CHECK_ARG(log_pdf != nullptr, 7, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("cacg_log_pdf_kernel", cacg_log_pdf_kernel, dim3((T + 127) / 128, F * K), 128, 0, st, quadratic,
                       eigenvalues, F, K, T, D, log_pdf, kTiny, nullptr);
}

int pbb_cacg_log_pdf_floor(const double* quadratic, const double* eigenvalues, int F, int K, int T, int D,
                           double q_floor, double* quadratic_out, double* log_pdf, void* stream) {
  PBB_CHECK_ARG(quadratic && eigenvalues, 1, "input is null");
  PBB_CHECK_ARG(F > 0 && K > 0 && T > 0 && D > 0 && F * K <= 65535, 3, "bad shape");
  PBB_CHECK_ARG(quadratic_out != nullptr && quadratic_out != quadratic, 8, "quadratic_out is null or the input");
  PBB_CHECK_ARG(log_pdf != nullptr, 9, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("cacg_log_pdf_kernel", cacg_log_pdf_kernel, dim3((T + 127) / 128, F * K), 128, 0, st, quadratic,
                       eigenvalues, F, K, T, D, log_pdf, q_floor, quadratic_out);
}

int pbb_gaussian_log_pdf(const double* embedding, const double* mean, const double* precision_cholesky,
                         const double* log_det, int F, int T, int E, int K, int diagonal, double* log_pdf,
                         void* stream) {
  PBB_CHECK_ARG(embedding && mean && precision_cholesky && log_det, 1, "input is null");
  PBB_CHECK_ARG(F > 0 && T > 0, 5, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 7, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && K < kMaxK, 8, "bad K");
  PBB_CHECK_ARG(log_pdf != nullptr, 10, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("gaussian_log_pdf_kernel", gaussian_log_pdf_kernel, dim3((T + 127) / 128, F), 128,
                       (size_t)2 * K * E * sizeof(double), st, embedding, mean, precision_cholesky, log_det, F, T, E, K,
                       diagonal, log_pdf);
}

size_t pbb_gaussian_fit_scratch_doubles(int F, int E, int K) { return (size_t)F * K * (E + 1) + K; }

int pbb_gaussian_fit(const double* embedding, const double* weight, int F, int T, int E, int K, int spherical,
                     double* mean, double* covariance, double* scratch, void* stream) {
  PBB_CHECK_ARG(embedding && weight, 1, "input is null");
  PBB_CHECK_ARG(F > 0 && T > 0, 3, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 5, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && K < kMaxK, 6, "bad K");
  PBB_CHECK_ARG(mean && covariance && scratch, 8, "output / scratch is null (pbb_gaussian_fit_scratch_doubles)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double* partial = scratch;
  double* denom = scratch + (size_t)F * K * (E + 1);
  PBB_TRY(launch_kernel("gaussian_fit_partial_kernel", gaussian_fit_partial_kernel, dim3(F, K), 256, 0, st, embedding,
                        weight, mean, F, T, E, K, 0, partial));
  PBB_TRY(launch_kernel("gaussian_fit_mean_kernel", gaussian_fit_mean_kernel, K, kIntMaxE + 1, 0, st, partial, F, E, K,
                        mean, denom));
  PBB_TRY(launch_kernel("gaussian_fit_partial_kernel", gaussian_fit_partial_kernel, dim3(F, K), 256, 0, st, embedding,
                        weight, mean, F, T, E, K, 1, partial));
  return launch_kernel("gaussian_fit_cov_kernel", gaussian_fit_cov_kernel, K, kIntMaxE, 0, st, partial, denom, F, E, K,
                       spherical, covariance);
}

int pbb_log_pdf_to_affiliation(const double* log_pdf_a, const double* log_pdf_b, double scale_a, double scale_b,
                               const double* weight, int weight_mode, const uint8_t* activity, double affiliation_eps,
                               int inline_pa, int F, int K, int T, double* affiliation, int* permutation,
                               void* stream) {
  PBB_CHECK_ARG(log_pdf_a != nullptr, 1, "log pdf is null");
  PBB_CHECK_ARG(weight != nullptr || weight_mode == PBB_WEIGHT_CONST, 5, "weight is null");
  PBB_CHECK_ARG((weight_mode >= 0 && weight_mode <= PBB_WEIGHT_FRAME) ||
                    (weight_mode >= PBB_WEIGHT_BCAST && weight_mode < 2 * PBB_WEIGHT_BCAST),
                6, "bad weight_mode");
  PBB_CHECK_ARG(F > 0 && T > 0, 10, "bad shape");
  PBB_CHECK_ARG(K > 0 && K <= kIntMaxK, 11, "need 0 < K <= 6 (K! pairings per bin)");
  PBB_CHECK_ARG(!inline_pa || log_pdf_b != nullptr, 9, "the inline alignment pairs TWO log pdfs");
  PBB_CHECK_ARG(affiliation != nullptr, 13, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("log_pdf_to_affiliation_kernel", log_pdf_to_affiliation_kernel, F, 256, 0, st, log_pdf_a,
                       log_pdf_b, scale_a, scale_b, weight, weight_mode, activity, affiliation_eps, inline_pa, F, K, T,
                       affiliation, permutation);
}

int pbb_gaussian_full_log_pdf(const double* embedding, const double* mean, const double* precision_cholesky,
                              const double* log_det, int B, int N, int E, int K, double* log_pdf, void* stream) {
  PBB_CHECK_ARG(embedding && mean && precision_cholesky && log_det, 1, "input is null");
  PBB_CHECK_ARG(B > 0 && B <= 65535 && N > 0, 5, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 7, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && K <= kIntMaxK, 8, "need 0 < K <= 6");
  PBB_CHECK_ARG(log_pdf != nullptr, 9, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid((N + 127) / 128, B);
  const size_t smem = (size_t)(E * E + E) * sizeof(double);
  const auto kern = E <= 8    ? gaussian_full_log_pdf_kernel<8>
                    : E <= 16 ? gaussian_full_log_pdf_kernel<16>
                    : E <= 32 ? gaussian_full_log_pdf_kernel<32>
                              : gaussian_full_log_pdf_kernel<64>;
  return launch_kernel("gaussian_full_log_pdf_kernel", kern, grid, 128, smem, st, embedding, mean, precision_cholesky,
                       log_det, N, E, K, log_pdf);
}

size_t pbb_gaussian_full_fit_scratch_doubles(int B, int N, int E, int K) {
  if (B <= 0 || N <= 0 || E <= 0 || K <= 0) return 0;
  const FullFitChunks c = full_fit_chunks(B, N, K);
  return (size_t)c.nchunks * B * K * fit_entries(E) + (size_t)B * K;
}

int pbb_gaussian_full_fit(const double* embedding, const double* weight, int B, int N, int E, int K, double* mean,
                          double* covariance, double* scratch, void* stream) {
  PBB_CHECK_ARG(embedding && weight, 1, "input is null");
  PBB_CHECK_ARG(B > 0 && N > 0, 3, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 5, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && (long long)B * K <= 65535, 6, "need 0 < K and B * K <= 65535");
  PBB_CHECK_ARG(mean && covariance && scratch, 7, "output / scratch is null (pbb_gaussian_full_fit_scratch_doubles)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const FullFitChunks c = full_fit_chunks(B, N, K);
  const int BK = B * K;
  double* partial = scratch;
  double* denom = scratch + (size_t)c.nchunks * BK * fit_entries(E);
  PBB_TRY(launch_kernel("gaussian_full_partial_kernel", gaussian_full_partial_kernel, dim3(c.nchunks, BK), kFitThreads,
                        0, st, embedding, weight, nullptr, N, E, K, c.chunk_len, 0, 0, partial));
  PBB_TRY(launch_kernel("gaussian_full_reduce_kernel", gaussian_full_reduce_kernel, BK, kFitThreads, 0, st, partial,
                        c.nchunks, E, 0, denom, mean, nullptr, nullptr, nullptr));
  PBB_TRY(launch_kernel("gaussian_full_partial_kernel", gaussian_full_partial_kernel, dim3(c.nchunks, BK), kFitThreads,
                        0, st, embedding, weight, mean, N, E, K, c.chunk_len, 1, 0, partial));
  return launch_kernel("gaussian_full_reduce_kernel", gaussian_full_reduce_kernel, BK, kFitThreads, 0, st, partial,
                       c.nchunks, E, 1, denom, nullptr, nullptr, nullptr, covariance);
}

int pbb_precision_cholesky(const double* covariance, int M, int E, double* precision_cholesky, double* log_det,
                           int* status, void* stream) {
  PBB_CHECK_ARG(covariance != nullptr, 1, "input is null");
  PBB_CHECK_ARG(M > 0, 2, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 3, "need 0 < E <= 64");
  PBB_CHECK_ARG(precision_cholesky && log_det && status, 4, "output / status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  return launch_kernel("precision_cholesky_kernel", precision_cholesky_kernel, M, 32, (size_t)E * E * sizeof(double),
                       st, covariance, E, precision_cholesky, log_det, status);
}

int pbb_vmf_log_pdf(const double* embedding, const double* mean, const double* concentration, const double* log_norm,
                    int B, int N, int E, int K, double* log_pdf, void* stream) {
  return vmf_log_pdf_launch<false>(embedding, mean, concentration, log_norm, B, N, E, K, log_pdf, stream);
}

int pbb_vmf_pdf(const double* embedding, const double* mean, const double* concentration, const double* log_norm,
                int B, int N, int E, int K, double* pdf, void* stream) {
  return vmf_log_pdf_launch<true>(embedding, mean, concentration, log_norm, B, N, E, K, pdf, stream);
}

int pbb_vmf_resultant(const double* embedding, const double* weight, int B, int N, int E, int K, double* resultant,
                      double* total, double* scratch, void* stream) {
  PBB_CHECK_ARG(embedding && weight, 1, "input is null");
  PBB_CHECK_ARG(B > 0 && N > 0, 3, "bad shape");
  PBB_CHECK_ARG(E > 0 && E <= kIntMaxE, 5, "need 0 < E <= 64");
  PBB_CHECK_ARG(K > 0 && (long long)B * K <= 65535, 6, "need 0 < K and B * K <= 65535");
  PBB_CHECK_ARG(resultant && total && scratch, 7, "output / scratch is null (pbb_gaussian_full_fit_scratch_doubles)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const FullFitChunks c = full_fit_chunks(B, N, K);
  const int BK = B * K;
  double* partial = scratch;
  double* denom = scratch + (size_t)c.nchunks * BK * fit_entries(E);
  PBB_TRY(launch_kernel("gaussian_full_partial_kernel", gaussian_full_partial_kernel, dim3(c.nchunks, BK), kFitThreads,
                        0, st, embedding, weight, nullptr, N, E, K, c.chunk_len, 0, 1, partial));
  return launch_kernel("gaussian_full_reduce_kernel", gaussian_full_reduce_kernel, BK, kFitThreads, 0, st, partial,
                       c.nchunks, E, 0, denom, nullptr, resultant, total, nullptr);
}

}  // extern "C"
