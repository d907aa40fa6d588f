// The single distributions of pb_bss/distribution (complex_angular_central_gaussian.py, complex_watson.py,
// complex_circular_symmetric_gaussian.py): the pieces the mixture-model kernels do not already provide.
//   cacg_from_covariance_kernel   from_covariance: trace norm, Hermitian eigh, eigenvalue norm and floor
//   cw_log_norm_kernel            the five Watson log normalisers of any array of kappa
//   cw_log_pdf_kernel             kappa |m^H y|^2 - log_norm_1f1, one pass over y
//   ccsg_lu_kernel                LU with partial pivoting and log|det| per covariance, one warp per matrix
//   ccsg_log_pdf_kernel           -D log pi - log|det S| - Re(y^H S^-1 y), one thread per frame
//   ccsg_cholesky_kernel          L = cholesky(S) per class (S given, or V diag(lambda) V^H)
//   ccsg_sample_kernel            L (re + i im) / sqrt(2), optionally scaled to unit norm, one thread per sample
// Every sum runs in a fixed order, so results do not depend on the launch shape.
#pragma once
#include "common.cuh"
#include "heig.cuh"
#include "linalg_kernels.cuh"

namespace pbb {

constexpr int kDistMaxD = 64;
constexpr int kCcsgThreads = 128;   // frames per CTA of ccsg_log_pdf_kernel
constexpr int kDistMaxGridY = 65535;
constexpr double kPi = 3.14159265358979323846;

// ---- ComplexAngularCentralGaussian.from_covariance (complex_angular_central_gaussian.py:81-132) ----------------
__host__ __device__ inline size_t from_covariance_smem_per_warp(int D) {
  return (jacobi_smem_bytes(D) + (size_t)D * sizeof(double) + 15) & ~(size_t)15;
}

__global__ void cacg_from_covariance_kernel(const double2* __restrict__ a, int n, int D, int norm, double floor_,
                                            double2* __restrict__ v, double* __restrict__ w, int* status, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  double2* A = reinterpret_cast<double2*>(smem_raw + from_covariance_smem_per_warp(D) * warp);
  double2* V = A + D * D;
  double* rot = reinterpret_cast<double*>(V + D * D);
  double* lam = rot + ((D + 1) / 2) * 6;
  const double2* __restrict__ am = a + (size_t)m * D * D;
  // 'trace' (:88-90): covariance / max(trace, tiny).  NumPy divides by the complex trace t + 0j, which is the
  // multiplication by 1 / t; the diagonal of a covariance is real, so its imaginary part is not read.
  double it = 1.0;
  if (norm == PBB_NORM_TRACE) {
    double tr = 0.0;
    for (int d = 0; d < D; ++d) tr += am[d * D + d].x;
    it = 1.0 / fmax(tr, kTiny);
  }
  bool bad = false;
  double amax = 0.0;
  for (int i = lane; i < D * D; i += 32) {
    const int r = i / D, c = i - r * D;
    const double2 x = am[r * D + c], y = am[c * D + r];
    const double2 h = make_double2(0.5 * (x.x * it + y.x * it), r == c ? 0.0 : 0.5 * (x.y * it - y.y * it));
    bad |= !isfinite(h.x) || !isfinite(h.y);
    A[i] = h;
    amax = cabs_max(amax, h);
  }
  const int escale = even_exponent(amax);
  for (int i = lane; i < D * D; i += 32) A[i] = cscalbn(A[i], -escale);
  __syncwarp();
  const int sweeps = warp_jacobi_any(A, V, rot, D, lane);
  double lmax = -INFINITY;
  for (int d = lane; d < D; d += 32) lmax = fmax(lmax, scalbn(A[d * D + d].x, escale));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmax(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  // (:111-126) eigenvalue: lambda / max(lambda_max, tiny), floored at eigenvalue_floor; else floored at
  // lambda_max * eigenvalue_floor
  for (int d = lane; d < D; d += 32) {
    double l = scalbn(A[d * D + d].x, escale);
    if (norm == PBB_NORM_EIGENVALUE) l = fmax(l / fmax(lmax, kTiny), floor_);
    else l = fmax(l, lmax * floor_);
    bad |= !isfinite(l);
    lam[d] = l;
  }
  if ((__any_sync(0xffffffffu, bad) || sweeps > kJacobiMaxSweeps) && lane == 0 && status) record_first(status, m + 1);
  __syncwarp();
  for (int x = lane; x < D; x += 32) {  // ascending, like np.linalg.eigh
    const int r = eig_rank(A, D, x);
    w[(size_t)m * D + r] = lam[x];
    for (int d = 0; d < D; ++d) v[(size_t)m * D * D + d * D + r] = V[d * D + x];
  }
}

// ---- ComplexWatson log normalisers (complex_watson.py:89-214) ---------------------------------------------------
// Each formula is evaluated in the reference's order of operations, without FMA contraction.
__device__ inline double cw_base(int D) {  // log(2) + D log(pi)
  return __dadd_rn(log(2.0), __dmul_rn((double)D, log(kPi)));
}

__device__ inline double cw_log_norm_low(double k, int D) {  // :90-107, Mardia Eq. 4, 20 Taylor terms
  double fact = 1.0;
  for (int r = 2; r < D; ++r) fact *= (double)r;
  double c = 1.0, s = 0.0;
  for (int b = D; b < D + 20; ++b) {
    c = __dmul_rn(c, __ddiv_rn(k, (double)b));  // cumprod
    s = __dadd_rn(s, c);
  }
  return __dadd_rn(__dsub_rn(cw_base(D), log(fact)), log(__dadd_rn(1.0, s)));
}

__device__ inline double cw_log_norm_closed(double k, int D, bool with_series) {  // :110-154, Mardia Eq. 3
  double v = __dadd_rn(__dadd_rn(cw_base(D), __dmul_rn(1.0 - (double)D, log(k))), k);
  if (!with_series) return v;
  const double e = exp(-k);
  double s = 0.0, fact = 1.0;
  for (int r = 0; r <= D - 2; ++r) {
    if (r > 0) fact *= (double)r;
    s = __dadd_rn(s, __ddiv_rn(__dmul_rn(pow(k, (double)r), e), fact));
  }
  return __dadd_rn(v, log(__dsub_rn(1.0, s)));
}

__device__ inline double cw_log_norm_variant(double k, int D, int variant) {
  switch (variant) {
    case PBB_CW_NORM_LOW: return cw_log_norm_low(k, D);
    case PBB_CW_NORM_MEDIUM: return cw_log_norm_closed(k < 1e-2 ? 1e-2 : k, D, true);  // :118-120 clamp
    case PBB_CW_NORM_HIGH: return cw_log_norm_closed(k, D, false);
    case PBB_CW_NORM_TRAN_VU:  // :205-214: low below 1/D, the unclamped medium formula from there on
      return k >= 1.0 / (double)D ? cw_log_norm_closed(k, D, true) : cw_log_norm_low(k, D);
    default: return cw_log_norm(k, D);
  }
}

__global__ void cw_log_norm_kernel(const double* __restrict__ kappa, long long n, int D, int variant,
                                   double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = cw_log_norm_variant(kappa[i], D, variant);
}

// ---- ComplexWatson.log_pdf (complex_watson.py:73-87) ------------------------------------------------------------
// y (M, N, D) with y_stride elements between models (0: one y shared by every model), mode (M, D), kappa (M).
template <class T>
__global__ void cw_log_pdf_kernel(const T* __restrict__ y, long long y_stride, int M, int N, int D,
                                  const double2* __restrict__ mode, const double* __restrict__ kappa,
                                  double* __restrict__ out) {
  __shared__ double ln;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  for (int m = blockIdx.y; m < M; m += gridDim.y) {
    __syncthreads();
    if (threadIdx.x == 0) ln = cw_log_norm(kappa[m], D);
    __syncthreads();
    if (n >= N) continue;
    const T* __restrict__ yr = y + (size_t)m * y_stride + (size_t)n * D;
    const double2* __restrict__ mm = mode + (size_t)m * D;
    double re = 0.0, im = 0.0;  // sum_d y_d conj(m_d)
    for (int d = 0; d < D; ++d) {
      const double2 yv = ld_cplx(yr + d), mv = mm[d];
      re += yv.x * mv.x + yv.y * mv.y;
      im += yv.y * mv.x - yv.x * mv.y;
    }
    out[(size_t)m * N + n] = __dsub_rn(__dmul_rn(abs2_rn(make_double2(re, im)), kappa[m]), ln);
  }
}

// ---- ComplexCircularSymmetricGaussian.log_pdf (complex_circular_symmetric_gaussian.py:26-48) ---------------------
// LU = P A with partial pivoting (LAPACK zgetrf: pivot = first max of |re| + |im|), stored in place: unit lower L
// below the diagonal, U on and above it; perm[i] = the row of A that became row i.  logdet = sum log|u_ii| in
// order, like np.linalg.slogdet.  status = 1 + the first model with an exactly zero pivot (np.linalg.solve raises
// LinAlgError there); its logdet is -inf.  Non-finite input gives logdet = NaN and no status, as LAPACK does.
__global__ void ccsg_lu_kernel(const double2* __restrict__ a, int M, int D, double2* __restrict__ lu,
                               int* __restrict__ perm, double* __restrict__ logdet, int* status, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= M) return;
  double2* A = reinterpret_cast<double2*>(smem_raw) + (size_t)warp * D * D;
  int* P = reinterpret_cast<int*>(reinterpret_cast<double2*>(smem_raw) + (size_t)warps * D * D) + warp * kDistMaxD;
  const double2* __restrict__ am = a + (size_t)m * D * D;
  bool bad = false;
  for (int i = lane; i < D * D; i += 32) {
    A[i] = am[i];
    bad |= !isfinite(A[i].x) || !isfinite(A[i].y);
  }
  for (int i = lane; i < D; i += 32) P[i] = i;
  __syncwarp();
  const bool nonfinite = __any_sync(0xffffffffu, bad);
  bool singular = false;
  for (int j = 0; j < D && !nonfinite; ++j) {
    int piv = j;
    double best = -1.0;
    for (int i = j; i < D; ++i) {
      const double2 v = A[i * D + j];
      const double mag = fabs(v.x) + fabs(v.y);
      if (mag > best) { best = mag; piv = i; }
    }
    if (!(best > 0.0)) { singular = true; break; }
    if (piv != j) {
      for (int c = lane; c < D; c += 32) { const double2 t = A[j * D + c]; A[j * D + c] = A[piv * D + c]; A[piv * D + c] = t; }
      if (lane == 0) { const int t = P[j]; P[j] = P[piv]; P[piv] = t; }
    }
    __syncwarp();
    const double2 p = A[j * D + j];
    for (int i = j + 1 + lane; i < D; i += 32) A[i * D + j] = cdiv(A[i * D + j], p);
    __syncwarp();
    const int w = D - j - 1;
    for (int idx = lane; idx < w * w; idx += 32) {
      const int i = j + 1 + idx / w, c = j + 1 + idx % w;
      const double2 q = cmul(A[i * D + j], A[j * D + c]);
      A[i * D + c].x -= q.x;
      A[i * D + c].y -= q.y;
    }
    __syncwarp();
  }
  double2* __restrict__ lo = lu + (size_t)m * D * D;
  for (int i = lane; i < D * D; i += 32) lo[i] = A[i];
  for (int i = lane; i < D; i += 32) perm[(size_t)m * D + i] = P[i];
  if (lane == 0) {
    double ld = 0.0;
    if (nonfinite) ld = NAN;
    else if (singular) ld = -INFINITY;
    else for (int d = 0; d < D; ++d) ld += log(hypot(A[d * D + d].x, A[d * D + d].y));
    logdet[m] = ld;
    if (singular && status) record_first(status, m + 1);
  }
}

__host__ __device__ inline size_t ccsg_log_pdf_smem(int D) {
  const size_t head = ((size_t)D * D * sizeof(double2) + (size_t)D * sizeof(int) + 15) & ~(size_t)15;
  return head + (size_t)D * kCcsgThreads * sizeof(double2);
}

// One thread per frame, the factorisation of its model in shared memory, the frame's solve in a shared column.
// x = U^-1 L^-1 P y (LAPACK zgetrs), out = (-D log pi - logdet) - Re(sum_d conj(y_d) x_d).
template <class T>
__global__ void __launch_bounds__(kCcsgThreads) ccsg_log_pdf_kernel(
    const T* __restrict__ y, long long y_stride, int M, int N, int D, const double2* __restrict__ lu,
    const int* __restrict__ perm, const double* __restrict__ logdet, double* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* L = reinterpret_cast<double2*>(smem_raw);
  int* P = reinterpret_cast<int*>(L + D * D);
  double2* X = reinterpret_cast<double2*>(
      smem_raw + (((size_t)D * D * sizeof(double2) + (size_t)D * sizeof(int) + 15) & ~(size_t)15));
  const int B = blockDim.x, tid = threadIdx.x;
  const int n = blockIdx.x * B + tid;
  double2* x = X + tid;
  for (int m = blockIdx.y; m < M; m += gridDim.y) {
    __syncthreads();
    for (int i = tid; i < D * D; i += B) L[i] = lu[(size_t)m * D * D + i];
    for (int i = tid; i < D; i += B) P[i] = perm[(size_t)m * D + i];
    __syncthreads();
    if (n >= N) continue;
    const T* __restrict__ yr = y + (size_t)m * y_stride + (size_t)n * D;
    for (int i = 0; i < D; ++i) x[i * B] = ld_cplx(yr + P[i]);
    for (int i = 1; i < D; ++i) {
      double2 s = x[i * B];
      for (int k = 0; k < i; ++k) {
        const double2 q = cmul(L[i * D + k], x[k * B]);
        s.x -= q.x; s.y -= q.y;
      }
      x[i * B] = s;
    }
    for (int i = D - 1; i >= 0; --i) {
      double2 s = x[i * B];
      for (int k = i + 1; k < D; ++k) {
        const double2 q = cmul(L[i * D + k], x[k * B]);
        s.x -= q.x; s.y -= q.y;
      }
      x[i * B] = cdiv(s, L[i * D + i]);
    }
    double q = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 yv = ld_cplx(yr + d), xv = x[d * B];
      q += yv.x * xv.x + yv.y * xv.y;
    }
    out[(size_t)m * N + n] = __dsub_rn(__dsub_rn(-(double)D * log(kPi), logdet[m]), q);
  }
}

// ---- ComplexCircularSymmetricGaussian.sample (complex_circular_symmetric_gaussian.py:50-72) -----------------------
// L (C, D, D) = np.linalg.cholesky of covariance c (lower triangle read), zero above the diagonal.  With eigenvalues
// the covariance is V diag(lambda) V^H of eigenvectors a (ComplexAngularCentralGaussian.covariance, :140-148).
// status = 1 + the first class that is not positive definite (LinAlgError in NumPy).
__global__ void ccsg_cholesky_kernel(const double2* __restrict__ a, const double* __restrict__ eigenvalues, int C,
                                     int D, double2* __restrict__ L, int* status, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * warps + warp;
  if (c >= C) return;
  double2* Bm = reinterpret_cast<double2*>(smem_raw) + (size_t)warp * D * D;
  const double2* __restrict__ ac = a + (size_t)c * D * D;
  for (int i = lane; i < D * D; i += 32) {
    if (eigenvalues == nullptr) { Bm[i] = ac[i]; continue; }
    const int r = i / D, col = i - r * D;
    double re = 0.0, im = 0.0;  // sum_x V[r][x] lambda[x] conj(V[col][x])
    for (int x = 0; x < D; ++x) {
      const double l = eigenvalues[(size_t)c * D + x];
      const double2 p = cmulc(ac[r * D + x], ac[col * D + x]);
      re += p.x * l;
      im += p.y * l;
    }
    Bm[i] = make_double2(re, im);
  }
  __syncwarp();
  const bool pd = warp_cholesky(Bm, D, lane);
  for (int i = lane; i < D * D; i += 32) {
    const int r = i / D, col = i - r * D;
    L[(size_t)c * D * D + i] = col <= r ? Bm[i] : make_double2(0.0, 0.0);
  }
  if (!pd && lane == 0 && status) record_first(status, c + 1);
}

// One thread per sample row i of class c (offsets[c] <= i < offsets[c + 1]): the standard normals re (S, D) and
// im (S, D) follow each other in `normals`.  x = (re + i im) * (1 / sqrt 2) -- NumPy's division by the complex
// sqrt(2) + 0j -- then y = L x, and with unit_norm y * (1 / ||y||) (sample_complex_angular_central_gaussian,
// complex_angular_central_gaussian.py:58-65).  Row i goes to out row dest[i] (identity without dest).
__global__ void ccsg_sample_kernel(const double2* __restrict__ L, int C, int D, const double* __restrict__ normals,
                                   const long long* __restrict__ offsets, const long long* __restrict__ dest,
                                   long long S, int unit_norm, double2* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S) return;
  int lo = 0, hi = C;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= i) lo = mid; else hi = mid;
  }
  const double2* __restrict__ Lc = L + (size_t)lo * D * D;
  const double* __restrict__ re = normals + (size_t)i * D;
  const double* __restrict__ im = normals + (size_t)S * D + (size_t)i * D;
  const double s2 = 1.0 / sqrt(2.0);
  double scale = 1.0;
  for (int pass = unit_norm ? 0 : 1; pass < 2; ++pass) {
    double nrm2 = 0.0;
    for (int r = 0; r < D; ++r) {
      double2 yr = make_double2(0.0, 0.0);
      for (int j = 0; j <= r; ++j) {
        const double2 q = cmul(Lc[r * D + j], make_double2(re[j] * s2, im[j] * s2));
        yr.x += q.x; yr.y += q.y;
      }
      if (pass == 0) nrm2 = __dadd_rn(nrm2, abs2_rn(yr));
      else out[(size_t)(dest ? dest[i] : i) * D + r] = make_double2(yr.x * scale, yr.y * scale);
    }
    if (pass == 0) scale = 1.0 / sqrt(nrm2);
  }
}

// CCSGTrainer._fit with a saliency (complex_circular_symmetric_gaussian.py:94-116): the PSD accumulation leaves
// sum_n s y y^H; covariance[f] *= 1 / max(sum_n saliency[f][n], floor_), the sum in a fixed order.  floor_ is
// np.finfo(y.dtype).tiny, as in the reference (the float32 tiny for complex64 y).
__global__ void ccsg_fit_scale_kernel(const double* __restrict__ saliency, int N, int D, double floor_,
                                      double2* __restrict__ cov) {
  __shared__ double red[8];
  const int f = blockIdx.x;
  double s = 0.0;
  for (int n = threadIdx.x; n < N; n += blockDim.x) s += saliency[(size_t)f * N + n];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const double inv = 1.0 / fmax(tot, floor_);
  for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
    double2& c = cov[(size_t)f * D * D + i];
    c = make_double2(c.x * inv, c.y * inv);
  }
}

}  // namespace pbb
