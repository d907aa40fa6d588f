// Batched small-matrix kernels of the beamforming side (pb_bss/extraction):
// Hermitian eigendecomposition, generalised Hermitian eigenproblem (GEV),
// linear solves (MVDR, Souden), blind analytic normalisation, PSD assembly and
// beamformer application.  One warp per D x D problem, matrices in shared memory.
#pragma once
#include "common.cuh"
#include "cplx.cuh"
#include "heig.cuh"

namespace pbb {

// status = 1 + the FIRST failing matrix (status starts at 0), like the reference's loop over the bins that raises at
// the first bad one (beamformer.py:395-409)
__device__ inline void record_first(int* status, int v) {
  int old = atomicCAS(status, 0, v);
  while (old != 0 && v < old) {
    const int prev = atomicCAS(status, old, v);
    if (prev == old) break;
    old = prev;
  }
}

// ---- Cholesky B = L L^H, lower triangle in place (warp) ------------------------
// returns false if B is not positive definite (LAPACK zpotrf INFO > 0, which is
// what zhegvd reports as INFO = N + i, get_gev_vector.pyx:130-147)
__device__ inline bool warp_cholesky(double2* __restrict__ B, int D, int lane) {
  bool ok = true;
  for (int j = 0; j < D; ++j) {
    const double djj = B[j * D + j].x;
    ok = ok && (djj > 0.0) && isfinite(djj);
    const double ljj = sqrt(fmax(djj, kTiny));
    __syncwarp();
    for (int i = j + lane; i < D; i += 32) {
      if (i == j) B[j * D + j] = make_double2(ljj, 0.0);
      else { const double2 v = B[i * D + j]; B[i * D + j] = make_double2(v.x / ljj, v.y / ljj); }
    }
    __syncwarp();
    // trailing update: B[i][k] -= L[i][j] conj(L[k][j]) for j < k <= i
    const int n = D - j - 1;
    for (int idx = lane; idx < n * n; idx += 32) {
      const int i = j + 1 + idx / n, k = j + 1 + idx % n;
      if (k <= i) {
        const double2 p = cmulc(B[i * D + j], B[k * D + j]);
        B[i * D + k].x -= p.x;
        B[i * D + k].y -= p.y;
      }
    }
    __syncwarp();
  }
  return ok;
}

// X <- L^{-1} X for lower-triangular L (forward substitution, all columns of X in parallel)
__device__ inline void warp_trsm_lower(const double2* __restrict__ L, double2* __restrict__ X, int D, int ncol,
                                       int lane) {
  for (int c = lane; c < ncol; c += 32) {
    for (int i = 0; i < D; ++i) {
      double2 s = X[i * ncol + c];
      for (int k = 0; k < i; ++k) {
        const double2 p = cmul(L[i * D + k], X[k * ncol + c]);
        s.x -= p.x; s.y -= p.y;
      }
      const double d = L[i * D + i].x;
      X[i * ncol + c] = make_double2(s.x / d, s.y / d);
    }
  }
  __syncwarp();
}

// X <- L^{-H} X (backward substitution with the conjugate transpose of L)
__device__ inline void warp_trsm_lower_h(const double2* __restrict__ L, double2* __restrict__ X, int D, int ncol,
                                         int lane) {
  for (int c = lane; c < ncol; c += 32) {
    for (int i = D - 1; i >= 0; --i) {
      double2 s = X[i * ncol + c];
      for (int k = i + 1; k < D; ++k) {
        const double2 lk = L[k * D + i];  // (L^H)[i][k] = conj(L[k][i])
        const double2 p = cmul(make_double2(lk.x, -lk.y), X[k * ncol + c]);
        s.x -= p.x; s.y -= p.y;
      }
      const double d = L[i * D + i].x;
      X[i * ncol + c] = make_double2(s.x / d, s.y / d);
    }
  }
  __syncwarp();
}

// ---- generalised Hermitian eigenproblem: top eigenvector ---------------------
// scipy.linalg.eigh(a, b) / LAPACK zhegvd ITYPE=1 (beamformer.py:367-411,
// get_gev_vector.pyx:124-150): B = L L^H, C = L^{-1} A L^{-H}, C y = lambda y,
// w = L^{-H} y, so w^H B w = 1.  out (n, D): eigenvector of the LARGEST eigenvalue.
//
// gev_reduce is the part before the Jacobi solver, shared by gev_kernel and its backward (eig_backward_kernel):
// C = the Hermitian part of 2^-ea A, L = the Cholesky factor of the Hermitian part of 2^-eb B, then C <- L^-1 C L^-H.
// V is scratch.  Returns false if B is not positive definite; bad (per lane) flags non-finite input.
__device__ __forceinline__ bool gev_reduce(const double2* __restrict__ am, const double2* __restrict__ bm, int D,
                                           int lane, double2* __restrict__ C, double2* __restrict__ V,
                                           double2* __restrict__ L, int& ea, int& eb, bool& bad) {
  bad = false;
  double amax = 0.0, bmax = 0.0;
  // zhegvd reads the lower triangles (UPLO = 'L'); use the Hermitian parts
  for (int i = lane; i < D * D; i += 32) {
    const int r = i / D, c = i - r * D;
    const double2 x = am[r * D + c], y = am[c * D + r];
    const double2 p = bm[r * D + c], q = bm[c * D + r];
    C[i] = make_double2(0.5 * (x.x + y.x), r == c ? 0.0 : 0.5 * (x.y - y.y));
    L[i] = make_double2(0.5 * (p.x + q.x), r == c ? 0.0 : 0.5 * (p.y - q.y));
    bad |= !isfinite(C[i].x) || !isfinite(C[i].y) || !isfinite(L[i].x) || !isfinite(L[i].y);
    amax = cabs_max(amax, C[i]);
    bmax = cabs_max(bmax, L[i]);
  }
  // solve with 2^-ea A and 2^-eb B: y does not change, and w = 2^(-eb/2) times the w of the scaled pair
  ea = even_exponent(amax);
  eb = even_exponent(bmax);
  for (int i = lane; i < D * D; i += 32) {
    C[i] = cscalbn(C[i], -ea);
    L[i] = cscalbn(L[i], -eb);
  }
  __syncwarp();
  const bool pd = warp_cholesky(L, D, lane);
  // C <- L^{-1} C L^{-H}:  first C <- L^{-1} C (columns), then C <- (L^{-1} C^H)^H
  warp_trsm_lower(L, C, D, D, lane);
  for (int i = lane; i < D * D; i += 32) {  // conjugate transpose into V (scratch)
    const int r = i / D, c = i - r * D;
    const double2 v = C[c * D + r];
    V[i] = make_double2(v.x, -v.y);
  }
  __syncwarp();
  warp_trsm_lower(L, V, D, D, lane);
  for (int i = lane; i < D * D; i += 32) {  // hermitise the result back into C
    const int r = i / D, c = i - r * D;
    const double2 u = V[c * D + r], v = V[r * D + c];  // conj(V^T) and V agree up to rounding
    C[i] = make_double2(0.5 * (u.x + v.x), r == c ? 0.0 : 0.5 * (-u.y + v.y));
  }
  __syncwarp();
  return pd;
}

// index of the largest eigenvalue on the diagonal of the diagonalised C, the last one of a tie (as eig_rank orders)
__device__ __forceinline__ int top_eigen_index(const double2* __restrict__ C, int D) {
  int best = 0;
  double lmax = C[0].x;
  for (int d = 1; d < D; ++d) {
    const double l = C[d * D + d].x;
    if (l >= lmax) { lmax = l; best = d; }
  }
  return best;
}

__global__ void gev_kernel(const double2* __restrict__ a, const double2* __restrict__ b, int n, int D,
                           double2* __restrict__ out, int* status, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  const size_t per = ((size_t)3 * D * D * sizeof(double2) + (size_t)((D + 1) / 2) * 6 * sizeof(double) + 15) &
                     ~(size_t)15;
  double2* C = reinterpret_cast<double2*>(smem_raw + per * warp);  // A -> C (Jacobi input)
  double2* V = C + D * D;
  double2* L = V + D * D;
  double* rot = reinterpret_cast<double*>(L + D * D);
  int ea, eb;
  bool bad;
  const bool pd = gev_reduce(a + (size_t)m * D * D, b + (size_t)m * D * D, D, lane, C, V, L, ea, eb, bad);
  const int sweeps = warp_jacobi_any(C, V, rot, D, lane);
  const int best = top_eigen_index(C, D);
  // w = L^{-H} y
  double2* yv = C;                                // reuse C's first column block as the rhs (D x 1)
  __syncwarp();
  for (int d = lane; d < D; d += 32) yv[d] = V[d * D + best];
  __syncwarp();
  warp_trsm_lower_h(L, yv, D, 1, lane);
  for (int d = lane; d < D; d += 32) out[(size_t)m * D + d] = cscalbn(yv[d], -eb / 2);
  if ((!pd || __any_sync(0xffffffffu, bad) || sweeps > kJacobiMaxSweeps) && lane == 0 && status)
    record_first(status, m + 1);
}

// The part of heig_batched_kernel (api_linalg.cu) before the Jacobi solver, shared with eig_backward_kernel: A = the
// Hermitian part (a + a^H) / 2 (LAPACK reads one triangle only), times 2^-escale (even_exponent): the same V,
// eigenvalues times 2^escale.  bad (per lane) flags non-finite input.
__device__ __forceinline__ void heig_prepare(const double2* __restrict__ am, int D, int lane, double2* __restrict__ A,
                                             int& escale, bool& bad) {
  bad = false;
  double amax = 0.0;
  for (int i = lane; i < D * D; i += 32) {
    const int r = i / D, c = i - r * D;
    const double2 x = am[r * D + c], y = am[c * D + r];
    const double2 h = make_double2(0.5 * (x.x + y.x), r == c ? 0.0 : 0.5 * (x.y - y.y));
    bad |= !isfinite(h.x) || !isfinite(h.y);
    A[i] = h;
    amax = cabs_max(amax, h);
  }
  escale = even_exponent(amax);
  for (int i = lane; i < D * D; i += 32) A[i] = cscalbn(A[i], -escale);
  __syncwarp();
}

// shared memory of one warp of solve_kernel: A, X and -- when the minimum-norm fallback is available (D <= kLstsqMaxD)
// -- a second matrix, the eigenvectors, a right-hand-side scratch and the Jacobi rotations
constexpr int kLstsqMaxD = 40;
__host__ __device__ inline size_t solve_smem_per_warp(int D, int R) {
  size_t b = (size_t)(D * D + D * R) * sizeof(double2);
  if (D <= kLstsqMaxD) b += (size_t)(2 * D * D + D * R) * sizeof(double2) + (size_t)((D + 1) / 2) * 6 * sizeof(double);
  return (b + 15) & ~(size_t)15;
}

// ---- general complex solve A X = B with partial pivoting (np.linalg.solve / zgesv) ----
// A (n, D, D), B (n, D, R) -> X (n, D, R).  hermitize: use (A + A^H) / 2 (beamformer.py:246-248); hermitize = 2 solves
// with A^H (the Souden backward, pbb_souden_backward).
// An exactly singular system (zero pivot: LinAlgError in the reference) takes the reference's fallback,
// np.linalg.lstsq (beamformer.py:251-256, math/solve.py:95-114): the minimum-norm solution X = A^+ B.  A Hermitian A
// (the PSD matrices of this path) is pseudo-inverted through its eigendecomposition, eigenvalues below
// eps * D * max|lambda| count as zero like LAPACK's rcond; a non-Hermitian A through A^H A (singular values below
// ~1e-7 of the largest count as zero there).  An
// all-zero A gives X = 0 (test_beamformer.py:211-376).  Non-finite input propagates as NaN, as it does in LAPACK.
// status (may be null) is only set when the fallback is unavailable (D > kLstsqMaxD).
// strict != 0 is plain np.linalg.solve (get_mvdr_vector_merl, beamformer.py:277): a zero pivot takes no fallback and
// sets status instead; x of that system is then undefined.  strict = 2 writes NaN there instead (no status).  fallback (may be null) is set to 1 when any system of the
// batch met a zero pivot, i.e. when the reference's stable_solve left np.linalg.solve for its per-matrix loop.
__global__ void solve_kernel(const double2* __restrict__ a, const double2* __restrict__ b, int n, int D, int R,
                             int hermitize, double2* __restrict__ x, int* status, int warps, int strict = 0,
                             int* fallback = nullptr) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  const size_t per = solve_smem_per_warp(D, R);
  double2* A = reinterpret_cast<double2*>(smem_raw + per * warp);
  double2* X = A + D * D;
  const double2* __restrict__ am = a + (size_t)m * D * D;
  double amax0 = 0.0;
  bool bad = false;
  for (int i = lane; i < D * D; i += 32) {
    const int r = i / D, c = i - r * D;
    const double2 u = am[i];
    if (hermitize == 2) {
      const double2 v = am[c * D + r];
      A[i] = make_double2(v.x, -v.y);
    } else if (hermitize) {
      const double2 v = am[c * D + r];
      A[i] = make_double2(0.5 * (u.x + v.x), 0.5 * (u.y - v.y));
    } else {
      A[i] = u;
    }
    amax0 = cabs_max(amax0, A[i]);
    bad |= !isfinite(A[i].x) || !isfinite(A[i].y);
  }
  // both branches solve with 2^-escale A: X = 2^-escale times that solution (minimum-norm one included)
  const int escale = even_exponent(amax0);
  for (int i = lane; i < D * D; i += 32) A[i] = cscalbn(A[i], -escale);
  for (int i = lane; i < D * R; i += 32) X[i] = b[(size_t)m * D * R + i];
  __syncwarp();
  // a NaN in A can hide from the pivot search (NaN > best is false) and end as a zero pivot: decide non-finite input
  // up front, so that it gives NaN and never the minimum-norm fallback
  bool singular = false, nonfinite = __any_sync(0xffffffffu, bad);
  for (int j = 0; j < D && !nonfinite; ++j) {
    // pivot search (every lane redundantly: D is tiny)
    int piv = j;
    double best = -1.0;
    for (int i = j; i < D; ++i) {
      const double2 v = A[i * D + j];
      const double mag = fabs(v.x) + fabs(v.y);  // LAPACK izamax uses |re| + |im|
      if (mag > best) { best = mag; piv = i; }
    }
    if (!isfinite(best)) { nonfinite = true; break; }
    if (!(best > 0.0)) { singular = true; break; }
    if (piv != j) {
      for (int c = lane; c < D; c += 32) { const double2 t = A[j * D + c]; A[j * D + c] = A[piv * D + c]; A[piv * D + c] = t; }
      for (int c = lane; c < R; c += 32) { const double2 t = X[j * R + c]; X[j * R + c] = X[piv * R + c]; X[piv * R + c] = t; }
    }
    __syncwarp();
    const double2 p = A[j * D + j];
    // eliminate below
    for (int idx = lane; idx < (D - j - 1) * (D - j - 1 + R); idx += 32) {
      const int w = D - j - 1 + R;
      const int i = j + 1 + idx / w, cc = idx % w;
      const double2 f = cdiv(A[i * D + j], p);
      if (cc < D - j - 1) {
        const int c = j + 1 + cc;
        const double2 q = cmul(f, A[j * D + c]);
        A[i * D + c].x -= q.x; A[i * D + c].y -= q.y;
      } else {
        const int c = cc - (D - j - 1);
        const double2 q = cmul(f, X[j * R + c]);
        X[i * R + c].x -= q.x; X[i * R + c].y -= q.y;
      }
    }
    __syncwarp();
  }
  if (singular && fallback && lane == 0) atomicOr(fallback, 1);
  if (nonfinite || (singular && strict == 2)) {
    for (int i = lane; i < D * R; i += 32) X[i] = make_double2(NAN, NAN);
    __syncwarp();
  } else if (!singular) {
    for (int c = lane; c < R; c += 32) {  // back substitution, columns in parallel
      for (int i = D - 1; i >= 0; --i) {
        double2 s = X[i * R + c];
        for (int k = i + 1; k < D; ++k) {
          const double2 q = cmul(A[i * D + k], X[k * R + c]);
          s.x -= q.x; s.y -= q.y;
        }
        X[i * R + c] = cdiv(s, A[i * D + i]);
      }
    }
    __syncwarp();
  } else if (strict || D > kLstsqMaxD) {
    if (lane == 0 && status) atomicMax(status, m + 1);
  } else {
    // ---- minimum-norm least squares (np.linalg.lstsq) ----
    double2* G = X + D * R;          // matrix to diagonalise
    double2* V = G + D * D;          // its eigenvectors
    double2* Y = V + D * D;          // right-hand side in the eigenbasis
    double* rot = reinterpret_cast<double*>(Y + D * R);
    double asym = 0.0, amax = 0.0;
    for (int i = lane; i < D * D; i += 32) {
      const int r = i / D, c = i - r * D;
      double2 u = cscalbn(am[i], -escale);
      const double2 v = cscalbn(am[c * D + r], -escale);
      if (hermitize) u = make_double2(0.5 * (u.x + v.x), 0.5 * (u.y - v.y));
      A[i] = u;
      asym = fmax(asym, hermitize ? 0.0 : fabs(u.x - v.x) + fabs(u.y + v.y));
      amax = fmax(amax, fabs(u.x) + fabs(u.y));
    }
    for (int i = lane; i < D * R; i += 32) X[i] = b[(size_t)m * D * R + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      asym = fmax(asym, __shfl_xor_sync(0xffffffffu, asym, o));
      amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    }
    __syncwarp();
    const bool herm = asym <= 1e-14 * amax;
    // G = A (Hermitian) or A^H A; Y0 = B or A^H B
    for (int i = lane; i < D * D; i += 32) {
      const int r = i / D, c = i - r * D;
      double2 g = A[i];
      if (!herm) {
        g = make_double2(0.0, 0.0);
        for (int k = 0; k < D; ++k) {
          const double2 q = cmulc(A[k * D + c], A[k * D + r]);  // conj(A[k][r]) * A[k][c]
          g.x += q.x; g.y += q.y;
        }
      }
      G[i] = g;
    }
    for (int i = lane; i < D * R; i += 32) {
      const int r = i / R, c = i - r * R;
      double2 y = X[i];
      if (!herm) {
        y = make_double2(0.0, 0.0);
        for (int k = 0; k < D; ++k) {
          const double2 q = cmulc(X[k * R + c], A[k * D + r]);  // conj(A[k][r]) * B[k][c]
          y.x += q.x; y.y += q.y;
        }
      }
      Y[i] = y;
    }
    __syncwarp();
    warp_jacobi_any(G, V, rot, D, lane);
    __syncwarp();
    double lmax = 0.0;
    for (int i = 0; i < D; ++i) lmax = fmax(lmax, fabs(G[i * D + i].x));
    const double cut = (herm ? 1.0 : 8.0) * DBL_EPSILON * D * lmax;
    // X = V diag(1 / lambda) V^H Y0 over the eigenvalues above the cut-off
    for (int i = lane; i < D * R; i += 32) {  // T = diag^+ V^H Y0, stored in X
      const int e = i / R, c = i - e * R;
      const double l = G[e * D + e].x;
      double2 t = make_double2(0.0, 0.0);
      if (fabs(l) > cut) {
        for (int k = 0; k < D; ++k) {
          const double2 q = cmulc(Y[k * R + c], V[k * D + e]);  // conj(V[k][e]) * Y0[k][c]
          t.x += q.x; t.y += q.y;
        }
        t.x /= l; t.y /= l;
      }
      X[i] = t;
    }
    __syncwarp();
    for (int i = lane; i < D * R; i += 32) {
      const int r = i / R, c = i - r * R;
      double2 o = make_double2(0.0, 0.0);
      for (int e = 0; e < D; ++e) {
        const double2 q = cmul(V[r * D + e], X[e * R + c]);
        o.x += q.x; o.y += q.y;
      }
      Y[i] = o;
    }
    __syncwarp();
    for (int i = lane; i < D * R; i += 32) X[i] = Y[i];
    __syncwarp();
  }
  for (int i = lane; i < D * R; i += 32) x[(size_t)m * D * R + i] = cscalbn(X[i], -escale);
}

// ---- MVDR: w = N^{-1} a / (a^H N^{-1} a) given x = N^{-1} a (beamformer.py:257-258) ----
__global__ void mvdr_scale_kernel(const double2* __restrict__ atf, const double2* __restrict__ x, int n, int D,
                                  double2* __restrict__ w) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  double2 den = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) {
    const double2 a = atf[(size_t)m * D + d], v = x[(size_t)m * D + d];
    const double2 p = cmul(make_double2(a.x, -a.y), v);
    den.x += p.x; den.y += p.y;
  }
  for (int d = 0; d < D; ++d) w[(size_t)m * D + d] = cdiv(x[(size_t)m * D + d], den);
}

// ---- quadratic forms w^H T w and w^H N w of one D-vector, w_d = wat(d) --------------
// The per-channel SNR terms of get_optimal_reference_channel (beamformer.py:616-620, w = w_mat[:, R]) and of
// mvdr_snr_postfilter (:502-509).  T and N point at one D x D matrix each.
template <class W>
__device__ __forceinline__ void quad_forms(W wat, const double2* __restrict__ T, const double2* __restrict__ N, int D,
                                           double2& qt, double2& qn) {
  qt = make_double2(0.0, 0.0);
  qn = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) {
    const double2 w = wat(d);
    const double2 wd = make_double2(w.x, -w.y);  // conj(w_d)
    double2 tt = make_double2(0.0, 0.0), nn = make_double2(0.0, 0.0);
    for (int e = 0; e < D; ++e) {
      const double2 we = wat(e);
      const double2 a = cmul(T[d * D + e], we);
      const double2 b = cmul(N[d * D + e], we);
      tt.x += a.x; tt.y += a.y; nn.x += b.x; nn.y += b.y;
    }
    const double2 a = cmul(wd, tt), b = cmul(wd, nn);
    qt.x += a.x; qt.y += a.y; qn.x += b.x; qn.y += b.y;
  }
}

// ---- Souden MVDR pieces (beamformer.py:601-698) --------------------------------
// mat = phi / max(trace(phi).real, eps); per-bin SNR numerators / denominators for
// every candidate reference channel R: w_R = mat[:, R]
__global__ void souden_kernel(const double2* __restrict__ phi, const double2* __restrict__ target,
                              const double2* __restrict__ noise, int n, int D, double eps, double2* __restrict__ mat,
                              double2* __restrict__ num, double2* __restrict__ den) {
  const int m = blockIdx.x;
  const int R = threadIdx.x;
  if (R >= D) return;
  const double2* __restrict__ ph = phi + (size_t)m * D * D;
  double tr = 0.0;
  for (int d = 0; d < D; ++d) tr += ph[d * D + d].x;
  const double s = 1.0 / fmax(tr, eps);
  for (int d = 0; d < D; ++d) {
    const double2 v = ph[d * D + R];
    mat[(size_t)m * D * D + d * D + R] = make_double2(v.x * s, v.y * s);
  }
  double2 qt, qn;
  quad_forms([&](int d) { return make_double2(ph[d * D + R].x * s, ph[d * D + R].y * s); },
             target + (size_t)m * D * D, noise + (size_t)m * D * D, D, qt, qn);
  num[(size_t)m * D + R] = qt;
  den[(size_t)m * D + R] = qn;
}

// ---- blind analytic normalisation (beamformer.py:459-488) -----------------------
__global__ void ban_kernel(const double2* __restrict__ vec, const double2* __restrict__ noise, int n, int D,
                           double2* __restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  const double2* __restrict__ N = noise + (size_t)m * D * D;
  const double2* __restrict__ w = vec + (size_t)m * D;
  // u = N w ; nominator = sqrt(w^H N N w) = sqrt((N^H w)^H (N w)) ; denominator = |w^H N w|
  double2 nom = make_double2(0.0, 0.0), den = make_double2(0.0, 0.0);
  for (int a = 0; a < D; ++a) {
    double2 left = make_double2(0.0, 0.0);   // sum_x conj(w_x) N[x][a]
    double2 right = make_double2(0.0, 0.0);  // sum_c N[a][c] w_c
    for (int c = 0; c < D; ++c) {
      const double2 p = cmul(make_double2(w[c].x, -w[c].y), N[c * D + a]);
      left.x += p.x; left.y += p.y;
      const double2 q = cmul(N[a * D + c], w[c]);
      right.x += q.x; right.y += q.y;
    }
    const double2 p = cmul(left, right);
    nom.x += p.x; nom.y += p.y;
    const double2 q = cmul(make_double2(w[a].x, -w[a].y), right);
    den.x += q.x; den.y += q.y;
  }
  // complex sqrt of nom, |den|, then |nom_sqrt / den_abs|
  const double nmag = sqrt(sqrt(nom.x * nom.x + nom.y * nom.y));  // |sqrt(z)| = sqrt(|z|)
  const double dmag = sqrt(den.x * den.x + den.y * den.y);        // sqrt(den * conj(den))
  const double scale = dmag != 0.0 ? nmag / dmag : 0.0;
  for (int d = 0; d < D; ++d) out[(size_t)m * D + d] = make_double2(w[d].x * scale, w[d].y * scale);
}

// ---- apply a beamforming vector: out[b][f][t] = sum_d conj(w[b][f][d]) Y[f][d][t] (beamformer.py:572-583);
// blockIdx.z = b runs over beamformers that share one mix (K sources on one STFT), 1 otherwise
// bins beyond gridDim.y (at most 65535) are taken in strides of gridDim.y
template <typename CT>
__global__ void apply_bf_kernel(const double2* __restrict__ w, const CT* __restrict__ Y, int F, int D, int T,
                                double2* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  for (int f = blockIdx.y; f < F; f += gridDim.y) {
    const size_t bf = (size_t)blockIdx.z * F + f;
    double2 s = make_double2(0.0, 0.0);
    for (int d = 0; d < D; ++d) {
      const double2 wd = w[bf * D + d];
      const double2 y = ld_cplx(Y + ((size_t)f * D + d) * T + t);
      s.x += wd.x * y.x + wd.y * y.y;
      s.y += wd.x * y.y - wd.y * y.x;
    }
    out[bf * T + t] = s;
  }
}

// ---- rank-1 PSD approximations (beamformer_wrapper.py:11-69) ---------------------
// out = a a^H * trace(cov) / trace(a a^H)
__global__ void rank_one_kernel(const double2* __restrict__ a, const double2* __restrict__ cov, int n, int D,
                                double2* __restrict__ out) {
  const int m = blockIdx.x;
  if (m >= n) return;
  const double2* __restrict__ am = a + (size_t)m * D;
  double2 tr = make_double2(0.0, 0.0);
  double na = 0.0;
  for (int d = 0; d < D; ++d) {
    const double2 c = cov[(size_t)m * D * D + d * D + d];
    tr.x += c.x; tr.y += c.y;
    na += am[d].x * am[d].x + am[d].y * am[d].y;
  }
  const double2 scale = make_double2(tr.x / na, tr.y / na);
  for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
    const int d = i / D, e = i - d * D;
    out[(size_t)m * D * D + i] = cmul(scale, cmulc(am[d], am[e]));
  }
}

// y = M x per matrix (the "scaled GEV ATF" Phi_nn w, beamformer_wrapper.py:27-46)
__global__ void matvec_kernel(const double2* __restrict__ M, const double2* __restrict__ x, int n, int D,
                              double2* __restrict__ y) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  for (int d = 0; d < D; ++d) {
    double2 s = make_double2(0.0, 0.0);
    for (int e = 0; e < D; ++e) {
      const double2 p = cmul(M[(size_t)m * D * D + d * D + e], x[(size_t)m * D + e]);
      s.x += p.x; s.y += p.y;
    }
    y[(size_t)m * D + d] = s;
  }
}

// ---- PSD assembly from the slot sums of the M-step kernels (beamformer.py:59-160) ----
// part (F, NCH, K, NS + 1) -> psd (F, K, D, D); scale: 0 = none, 1 = 1 / max(sum mask, 1e-10)
// (beamformer.py:127-131), 2 = 1 / T (no mask, beamformer.py:114-117)
__global__ void psd_finalize_kernel(const double* __restrict__ part, int nch, int F, int K, int D, int T, int scale,
                                    double2* __restrict__ psd) {
  const int f = blockIdx.x, k = blockIdx.y;
  const int NS = D * D;
  const double* __restrict__ p0 = part + ((size_t)f * nch * K + k) * (NS + 1);
  double sm = 0.0;
  for (int c = 0; c < nch; ++c) sm += p0[(size_t)c * K * (NS + 1) + NS];
  const double sc = scale == 1 ? 1.0 / fmax(sm, 1e-10) : (scale == 2 ? 1.0 / (double)T : 1.0);
  double2* __restrict__ o = psd + ((size_t)f * K + k) * NS;
  double* od = reinterpret_cast<double*>(o);
  for (int s = threadIdx.x; s < NS; s += blockDim.x) {
    double v = 0.0;
    for (int c = 0; c < nch; ++c) v += p0[(size_t)c * K * (NS + 1) + s];
    v *= sc;
    const SlotInfo si = slot_info(D, s);
    if (si.kind == 0) { od[2 * (si.d * D + si.d)] = v; od[2 * (si.d * D + si.d) + 1] = 0.0; }
    else if (si.kind == 1) { od[2 * (si.d * D + si.e)] = v; od[2 * (si.e * D + si.d)] = v; }
    else { od[2 * (si.d * D + si.e) + 1] = -v; od[2 * (si.e * D + si.d) + 1] = v; }
  }
}

// ================================ backward passes (pb_bss_b200 autograd) ================================
// Gradients follow PyTorch's convention for a real loss L: grad z = dL/dRe z + i dL/dIm z.  fp64, fixed-order sums, no
// atomics.

// ---- Souden MVDR, w = Phi[:, r] / max(Re tr Phi, eps) per bin (pbb_souden_backward) ----
// grad Phi = g e_r^T / lambda - (Re(g^H Phi[:, r]) / lambda^2) I for lambda = Re tr Phi > eps, g e_r^T / eps otherwise.
// One CTA per bin, thread i writes row i.
__global__ void souden_backward_kernel(const double2* __restrict__ phi, const double2* __restrict__ g, int n, int D,
                                       int r, double eps, double2* __restrict__ gphi) {
  const int m = blockIdx.x, i = threadIdx.x;
  if (i >= D) return;
  const double2* __restrict__ ph = phi + (size_t)m * D * D;
  const double2* __restrict__ gm = g + (size_t)m * D;
  double tr = 0.0, c = 0.0;
  for (int d = 0; d < D; ++d) tr += ph[d * D + d].x;  // the forward's order
  for (int d = 0; d < D; ++d) c += gm[d].x * ph[d * D + r].x + gm[d].y * ph[d * D + r].y;
  const bool scaled = tr > eps;
  const double inv = 1.0 / (scaled ? tr : eps), diag = scaled ? c * inv * inv : 0.0;
  const double2 gi = gm[i];
  double2* __restrict__ o = gphi + (size_t)m * D * D + (size_t)i * D;
  for (int j = 0; j < D; ++j) {
    double2 v = j == r ? make_double2(gi.x * inv, gi.y * inv) : make_double2(0.0, 0.0);
    if (j == i) v.x -= diag;
    o[j] = v;
  }
}

// grad N = -grad X Phi^H per bin, one thread per entry
__global__ void souden_noise_backward_kernel(const double2* __restrict__ gx, const double2* __restrict__ phi, int n,
                                             int D, double2* __restrict__ gn) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n * D * D) return;
  const long long m = idx / (D * D);
  const int i = (int)(idx - m * D * D) / D, j = (int)(idx - m * D * D) % D;
  const double2* __restrict__ x = gx + m * D * D + (size_t)i * D;
  const double2* __restrict__ p = phi + m * D * D + (size_t)j * D;
  double2 s = make_double2(0.0, 0.0);
  for (int k = 0; k < D; ++k) {
    const double2 q = cmulc(x[k], p[k]);
    s.x += q.x; s.y += q.y;
  }
  gn[idx] = make_double2(-s.x, -s.y);
}

// ---- apply_beamforming_vector, out[b][f][t] = sum_a conj(w[b][f][a]) Y[f][a][t] ----
// grad w[b][f][a] = sum_t Y[f][a][t] conj(g[b][f][t]): one warp per (b, f, a), lanes stride over t, then a fixed
// butterfly.
template <typename CT>
__global__ void apply_bf_vector_backward_kernel(const CT* __restrict__ Y, const double2* __restrict__ g, int B, int F,
                                                int D, int T, double2* __restrict__ gw) {
  const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)B * F * D) return;
  const long long bf = w / D;
  const int a = (int)(w - bf * D), f = (int)(bf % F);
  const CT* __restrict__ y = Y + ((size_t)f * D + a) * T;
  const double2* __restrict__ gr = g + (size_t)bf * T;
  double2 s = make_double2(0.0, 0.0);
  for (int t = lane; t < T; t += 32) {
    const double2 q = cmulc(ld_cplx(y + t), __ldg(gr + t));
    s.x += q.x; s.y += q.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s.x += __shfl_xor_sync(0xffffffffu, s.x, o);
    s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
  }
  if (lane == 0) gw[w] = s;
}

// grad Y[f][a][t] = sum_b w[b][f][a] g[b][f][t] in increasing b (B beamformers sharing one mix; B = 1 otherwise).  Bins
// beyond gridDim.y are taken in strides of gridDim.y.
__global__ void apply_bf_mix_backward_kernel(const double2* __restrict__ w, const double2* __restrict__ g, int B, int F,
                                             int D, int T, double2* __restrict__ gY) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  for (int f = blockIdx.y; f < F; f += gridDim.y) {
    for (int a = 0; a < D; ++a) {
      double2 s = make_double2(0.0, 0.0);
      for (int b = 0; b < B; ++b) {
        const double2 q = cmul(__ldg(w + ((size_t)b * F + f) * D + a), __ldg(g + ((size_t)b * F + f) * T + t));
        s.x += q.x; s.y += q.y;
      }
      gY[((size_t)f * D + a) * T + t] = s;
    }
  }
}

// ---- get_power_spectral_density_matrix, Phi_fk = sum_t w_fkt y_ft y_ft^H (pbb_power_spectral_density_backward) ----
// w = m / max(S, 1e-10) with S = sum_t m (normalize), m (no normalize), 1 / T (no mask).  With G = grad Phi and
// H = G + G^H:  grad y_t = sum_k w_kt H_k y_t;  dL/dm_kt = (Re(y^H G_k y) - Re<G_k, Phi_k>) / S_k while S_k > 1e-10,
// Re(y^H G_k y) / max(S_k, 1e-10) otherwise or without normalize (times 1 / 1 there).  Re(y^H G y) = Re(y^H H y) / 2.
// One CTA per (tile of kPsdBwdThreads frames, bin); thread = frame.  The frame's y and grad y live in shared memory
// ([d][thread]), H_k is staged per source, so Y is read once for all K sources.
constexpr int kPsdBwdThreads = 64;
__host__ __device__ inline size_t psd_backward_smem(int D, int K) {
  return (size_t)(D * D + 2 * D * kPsdBwdThreads) * sizeof(double2) + (size_t)3 * K * sizeof(double);
}

template <typename CT>
__global__ void __launch_bounds__(kPsdBwdThreads) psd_backward_kernel(
    const CT* __restrict__ Y, const double* __restrict__ mask, const double2* __restrict__ psd,
    const double2* __restrict__ gpsd, int F, int D, int T, int K, int normalize, double2* __restrict__ gy_out,
    double* __restrict__ gm_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* H = reinterpret_cast<double2*>(smem_raw);
  double2* ys = H + D * D;
  double2* gys = ys + D * kPsdBwdThreads;
  double* scale = reinterpret_cast<double*>(gys + D * kPsdBwdThreads);  // w = m * scale[k]
  double* cterm = scale + K;                                             // Re<G_k, Phi_k> (0 where it drops out)
  double* mscale = cterm + K;                                            // dL/dm = (q - cterm) * mscale
  const int tiles = (T + kPsdBwdThreads - 1) / kPsdBwdThreads;
  const int f = blockIdx.x / tiles, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t = (blockIdx.x - f * tiles) * kPsdBwdThreads + tid;
  // per-source scalars: one warp per source, lanes stride, fixed butterfly
  for (int k = warp; k < K; k += kPsdBwdThreads / 32) {
    const double* __restrict__ mk = mask ? mask + ((size_t)f * K + k) * T : nullptr;
    const double2* __restrict__ G = gpsd + ((size_t)f * K + k) * D * D;
    const double2* __restrict__ P = psd + ((size_t)f * K + k) * D * D;
    double S = 0.0, c = 0.0;
    if (mk && normalize)
      for (int i = lane; i < T; i += 32) S += __ldg(mk + i);
    for (int i = lane; i < D * D; i += 32) c += G[i].x * P[i].x + G[i].y * P[i].y;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      S += __shfl_xor_sync(0xffffffffu, S, o);
      c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    if (lane == 0) {
      if (!mk) {
        scale[k] = 1.0 / (double)T;
      } else if (normalize) {
        scale[k] = 1.0 / fmax(S, 1e-10);
        cterm[k] = S > 1e-10 ? c : 0.0;
        mscale[k] = scale[k];
      } else {
        scale[k] = 1.0;
        cterm[k] = 0.0;
        mscale[k] = 1.0;
      }
    }
  }
  const bool live = t < T;
  if (live)
    for (int d = 0; d < D; ++d) {
      ys[d * kPsdBwdThreads + tid] = ld_cplx(Y + ((size_t)f * D + d) * T + t);
      gys[d * kPsdBwdThreads + tid] = make_double2(0.0, 0.0);
    }
  for (int k = 0; k < K; ++k) {
    __syncthreads();
    const double2* __restrict__ G = gpsd + ((size_t)f * K + k) * D * D;
    for (int i = tid; i < D * D; i += kPsdBwdThreads) {
      const int r = i / D, c = i - r * D;
      const double2 a = G[i], b = G[c * D + r];
      H[i] = make_double2(a.x + b.x, a.y - b.y);
    }
    __syncthreads();
    if (!live) continue;
    const double wk = (mask ? __ldg(mask + ((size_t)f * K + k) * T + t) : 1.0) * scale[k];
    double q = 0.0;
    for (int i = 0; i < D; ++i) {
      double2 u = make_double2(0.0, 0.0);
      for (int j = 0; j < D; ++j) {
        const double2 p = cmul(H[i * D + j], ys[j * kPsdBwdThreads + tid]);
        u.x += p.x; u.y += p.y;
      }
      const double2 y = ys[i * kPsdBwdThreads + tid];
      q += y.x * u.x + y.y * u.y;  // Re(conj(y_i) u_i)
      double2& gy = gys[i * kPsdBwdThreads + tid];
      gy.x += wk * u.x;
      gy.y += wk * u.y;
    }
    if (mask && gm_out) gm_out[((size_t)f * K + k) * T + t] = (0.5 * q - cterm[k]) * mscale[k];
  }
  if (live && gy_out)
    for (int d = 0; d < D; ++d) gy_out[((size_t)f * D + d) * T + t] = gys[d * kPsdBwdThreads + tid];
}

// ================================ backward passes of the get_bf_vector beamformers ================================

// ---- top eigenpair (lambda, w) of the Hermitian parts of (A, B), w^H B w = 1 (pbb_eigenvector_backward) ----
// Phase held fixed, Im(w^H B dw) = 0.  u = P g with P = sum_{j != top} w_j w_j^H / (lambda - lambda_j), recomputed
// from the forward's own reduction and Jacobi solver (gev_reduce / heig_prepare, then warp_jacobi_any):
//   P = 2^-ea L^-H (sum_{j != top} y_j y_j^H / (l - l_j)) L^-1 in the scaled pencil, l = eigenvalues of C.
// P does not depend on the phase of the eigenvectors; u w^H is formed with the forward's saved w.
//   grad A = (u w^H + w u^H) / 2 + g_lambda w w^H,
//   grad B = -lambda (u w^H + w u^H) / 2 - (Re(w^H g) / 2 + lambda g_lambda) w w^H        (pencil only).
// b == nullptr is the plain Hermitian case (B = I, PCA).  One warp per bin: C, V (and L) in shared memory like
// gev_kernel, plus two D-vectors.  A tie of the top eigenvalue, a B that is not positive definite, non-finite input or
// no convergence gives NaN in that bin only.
__host__ __device__ inline size_t eig_backward_smem_per_warp(int D, bool pencil) {
  return ((size_t)(pencil ? 3 : 2) * D * D * sizeof(double2) + (size_t)((D + 1) / 2) * 6 * sizeof(double) +
          (size_t)2 * D * sizeof(double2) + 15) & ~(size_t)15;
}

__global__ void eig_backward_kernel(const double2* __restrict__ a, const double2* __restrict__ b,
                                    const double2* __restrict__ w, const double2* __restrict__ g,
                                    const double* __restrict__ glam, int n, int D, double2* __restrict__ ga,
                                    double2* __restrict__ gb, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  const bool pencil = b != nullptr;
  const size_t per = eig_backward_smem_per_warp(D, pencil);
  double2* C = reinterpret_cast<double2*>(smem_raw + per * warp);
  double2* V = C + D * D;
  double2* L = V + D * D;  // pencil only
  double* rot = reinterpret_cast<double*>(pencil ? L + D * D : L);
  double2* h = reinterpret_cast<double2*>(rot + ((D + 1) / 2) * 6);
  double2* z = h + D;
  int ea, eb = 0;
  bool bad, pd = true;
  if (pencil) pd = gev_reduce(a + (size_t)m * D * D, b + (size_t)m * D * D, D, lane, C, V, L, ea, eb, bad);
  else heig_prepare(a + (size_t)m * D * D, D, lane, C, ea, bad);
  const int sweeps = warp_jacobi_any(C, V, rot, D, lane);
  const int top = top_eigen_index(C, D);
  const double lt = C[top * D + top].x;
  bool tied = false;
  for (int j = 0; j < D; ++j) tied |= j != top && C[j * D + j].x == lt;
  const bool nan_bin = tied || !pd || __any_sync(0xffffffffu, bad) || sweeps > kJacobiMaxSweeps;
  const double2* __restrict__ wm = w + (size_t)m * D;
  const double2* __restrict__ gm = g + (size_t)m * D;
  // h = L^-1 g (g in the pencil)
  for (int d = lane; d < D; d += 32) h[d] = gm[d];
  __syncwarp();
  if (pencil) warp_trsm_lower(L, h, D, 1, lane);
  // z_j = y_j^H h / (l - l_j), 0 at the top
  for (int j = lane; j < D; j += 32) {
    double2 s = make_double2(0.0, 0.0);
    for (int k = 0; k < D; ++k) {
      const double2 q = cmulc(h[k], V[k * D + j]);
      s.x += q.x; s.y += q.y;
    }
    const double den = lt - C[j * D + j].x;
    z[j] = j == top ? make_double2(0.0, 0.0) : make_double2(s.x / den, s.y / den);
  }
  __syncwarp();
  // h <- Y z, then L^-H h: u = 2^-ea h
  for (int k = lane; k < D; k += 32) {
    double2 s = make_double2(0.0, 0.0);
    for (int j = 0; j < D; ++j) {
      const double2 q = cmul(V[k * D + j], z[j]);
      s.x += q.x; s.y += q.y;
    }
    h[k] = s;
  }
  __syncwarp();
  if (pencil) warp_trsm_lower_h(L, h, D, 1, lane);
  double rho = 0.0;  // Re(w^H g), every lane in the same order
  for (int k = 0; k < D; ++k) rho += wm[k].x * gm[k].x + wm[k].y * gm[k].y;
  const double lam = scalbn(lt, ea - eb);
  const double gl = glam ? glam[m] : 0.0;
  const double cb = 0.5 * rho + lam * gl;
  for (int idx = lane; idx < D * D; idx += 32) {
    const int i = idx / D, k = idx - i * D;
    double2 oa, ob;
    if (nan_bin) {
      oa = ob = make_double2(NAN, NAN);
    } else {
      const double2 ui = cscalbn(h[i], -ea), uk = cscalbn(h[k], -ea), wi = wm[i], wk = wm[k];
      const double2 p = cmulc(ui, wk), q = cmulc(wi, uk), ww = cmulc(wi, wk);
      const double2 sym = make_double2(0.5 * (p.x + q.x), 0.5 * (p.y + q.y));
      oa = make_double2(sym.x + gl * ww.x, sym.y + gl * ww.y);
      ob = make_double2(-lam * sym.x - cb * ww.x, -lam * sym.y - cb * ww.y);
    }
    ga[(size_t)m * D * D + idx] = oa;
    if (pencil) gb[(size_t)m * D * D + idx] = ob;
  }
}

// ---- MVDR, w = x / s, x = N_h^-1 a, s = a^H x, N_h = (N + N^H) / 2 (pbb_mvdr_backward) ----
// With t = w^H g:  q = (g - t a) / conj(s),  p = N_h^-1 q (solve_kernel, strict = 2),
//   grad a = p - conj(t) w,   grad N = -(p x^H + x p^H) / 2.
// q, one thread per bin, s in mvdr_scale_kernel's order.
__global__ void mvdr_backward_rhs_kernel(const double2* __restrict__ atf, const double2* __restrict__ x,
                                         const double2* __restrict__ w, const double2* __restrict__ g, int n, int D,
                                         double2* __restrict__ q) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  double2 s = make_double2(0.0, 0.0), t = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) {
    const double2 a = atf[(size_t)m * D + d], v = x[(size_t)m * D + d];
    const double2 p = cmul(make_double2(a.x, -a.y), v);
    s.x += p.x; s.y += p.y;
  }
  for (int d = 0; d < D; ++d) {
    const double2 u = cmulc(g[(size_t)m * D + d], w[(size_t)m * D + d]);  // conj(w_d) g_d
    t.x += u.x; t.y += u.y;
  }
  const double2 sc = make_double2(s.x, -s.y);
  for (int d = 0; d < D; ++d) {
    const double2 ta = cmul(t, atf[(size_t)m * D + d]), gd = g[(size_t)m * D + d];
    q[(size_t)m * D + d] = cdiv(make_double2(gd.x - ta.x, gd.y - ta.y), sc);
  }
}

// grad N and grad a from p, one thread per entry of N; the threads of column 0 also write grad a
__global__ void mvdr_backward_kernel(const double2* __restrict__ p, const double2* __restrict__ x,
                                     const double2* __restrict__ w, const double2* __restrict__ g, int n, int D,
                                     double2* __restrict__ ga, double2* __restrict__ gn) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n * D * D) return;
  const long long m = idx / (D * D);
  const int i = (int)(idx - m * D * D) / D, j = (int)(idx - m * D * D) % D;
  const double2* __restrict__ pm = p + m * D;
  const double2* __restrict__ xm = x + m * D;
  const double2 a = cmulc(pm[i], xm[j]), b = cmulc(xm[i], pm[j]);
  gn[idx] = make_double2(-0.5 * (a.x + b.x), -0.5 * (a.y + b.y));
  if (j == 0) {
    const double2* __restrict__ wm = w + m * D;
    double2 t = make_double2(0.0, 0.0);
    for (int d = 0; d < D; ++d) {
      const double2 u = cmulc(g[m * D + d], wm[d]);
      t.x += u.x; t.y += u.y;
    }
    const double2 tw = cmulc(wm[i], t);  // conj(t) w_i
    ga[m * D + i] = make_double2(pm[i].x - tw.x, pm[i].y - tw.y);
  }
}

// ---- blind analytic normalisation, out = c w, c = sqrt|nu| / |delta|, nu = w^H N N w, delta = w^H N w ----
// (pbb_blind_analytic_normalization_backward; N as given, not hermitised).  With r = N w, l = N^H w, rho = Re(w^H g),
// alpha = rho c conj(nu) / (2 |nu|^2) and beta = -rho c conj(delta) / |delta|^2:
//   grad w = c g + alpha N r + conj(alpha) N^H l + beta r + conj(beta) l,
//   grad N = conj(alpha) (w r^H + l w^H) + conj(beta) w w^H.
// delta = 0 (c is the constant 0 there): zero gradients; nu = 0 with delta != 0 (infinite derivative of sqrt|nu|):
// NaN.  One warp per bin; r and l (as ban_kernel forms them, so nu and delta are the forward's) in shared memory.
__global__ void ban_backward_kernel(const double2* __restrict__ vec, const double2* __restrict__ noise,
                                    const double2* __restrict__ g, int n, int D, double2* __restrict__ gv,
                                    double2* __restrict__ gn, int warps) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * warps + warp;
  if (m >= n) return;
  double2* left = reinterpret_cast<double2*>(smem_raw) + (size_t)2 * D * warp;  // w^H N = conj(l)^T
  double2* right = left + D;                                                    // N w = r
  const double2* __restrict__ N = noise + (size_t)m * D * D;
  const double2* __restrict__ w = vec + (size_t)m * D;
  const double2* __restrict__ gm = g + (size_t)m * D;
  for (int a = lane; a < D; a += 32) {
    double2 lf = make_double2(0.0, 0.0), rt = make_double2(0.0, 0.0);
    for (int c = 0; c < D; ++c) {
      const double2 p = cmul(make_double2(w[c].x, -w[c].y), N[c * D + a]);
      lf.x += p.x; lf.y += p.y;
      const double2 q = cmul(N[a * D + c], w[c]);
      rt.x += q.x; rt.y += q.y;
    }
    left[a] = lf;
    right[a] = rt;
  }
  __syncwarp();
  double2 nom = make_double2(0.0, 0.0), den = make_double2(0.0, 0.0);
  double rho = 0.0;
  for (int a = 0; a < D; ++a) {  // ban_kernel's order, every lane
    const double2 p = cmul(left[a], right[a]);
    nom.x += p.x; nom.y += p.y;
    const double2 q = cmul(make_double2(w[a].x, -w[a].y), right[a]);
    den.x += q.x; den.y += q.y;
    rho += w[a].x * gm[a].x + w[a].y * gm[a].y;
  }
  const double nmag = sqrt(sqrt(nom.x * nom.x + nom.y * nom.y));
  const double dmag = sqrt(den.x * den.x + den.y * den.y);
  const bool zero = !(dmag != 0.0), nan_bin = !zero && nom.x == 0.0 && nom.y == 0.0;
  const double c = zero ? 0.0 : nmag / dmag;
  const double n2 = nom.x * nom.x + nom.y * nom.y, d2 = den.x * den.x + den.y * den.y;
  const double fa = zero || nan_bin ? 0.0 : 0.5 * rho * c / n2, fb = zero || nan_bin ? 0.0 : -rho * c / d2;
  const double2 al = make_double2(fa * nom.x, -fa * nom.y), be = make_double2(fb * den.x, -fb * den.y);
  const double2 alc = make_double2(al.x, -al.y), bec = make_double2(be.x, -be.y);
  for (int i = lane; i < D; i += 32) {
    double2 o;
    if (nan_bin) {
      o = make_double2(NAN, NAN);
    } else {
      double2 nr = make_double2(0.0, 0.0), nl = make_double2(0.0, 0.0);  // (N r)_i, (N^H l)_i
      for (int k = 0; k < D; ++k) {
        const double2 p = cmul(N[i * D + k], right[k]);
        nr.x += p.x; nr.y += p.y;
        const double2 q = cmul(N[k * D + i], left[k]);  // conj((N^H l)_i term)
        nl.x += q.x; nl.y -= q.y;
      }
      const double2 t1 = cmul(al, nr), t2 = cmul(alc, nl), t3 = cmul(be, right[i]);
      const double2 t4 = cmulc(bec, left[i]);  // conj(beta) l_i = conj(beta) conj(left_i)
      o = make_double2(c * gm[i].x + t1.x + t2.x + t3.x + t4.x, c * gm[i].y + t1.y + t2.y + t3.y + t4.y);
    }
    gv[(size_t)m * D + i] = o;
  }
  for (int idx = lane; idx < D * D; idx += 32) {
    const int i = idx / D, j = idx - i * D;
    double2 o;
    if (nan_bin) {
      o = make_double2(NAN, NAN);
    } else {
      const double2 wr = cmulc(w[i], right[j]);                             // w_i conj(r_j)
      const double2 lw = cmulc(make_double2(left[i].x, -left[i].y), w[j]);  // l_i conj(w_j)
      const double2 ww = cmulc(w[i], w[j]);
      const double2 s = cmul(alc, make_double2(wr.x + lw.x, wr.y + lw.y)), t = cmul(bec, ww);
      o = make_double2(s.x + t.x, s.y + t.y);
    }
    gn[(size_t)m * D * D + idx] = o;
  }
}

// ---- rank-1 estimate, out = a a^H t / nu, t = sum_d C_dd (complex), nu = |a|^2 (pbb_rank_one_estimate_backward) ----
// With G = grad out and q = a^H G a:
//   grad a = (conj(t) G a + t G^H a) / nu - 2 Re(t conj(q)) / nu^2 a,   grad C = (q / nu) I.
// nu = 0 gives NaN.  One CTA of 64 threads per bin (D <= 64); G a and G^H a in shared memory.
__global__ void rank_one_backward_kernel(const double2* __restrict__ a, const double2* __restrict__ cov,
                                         const double2* __restrict__ gout, int n, int D, double2* __restrict__ ga,
                                         double2* __restrict__ gc) {
  __shared__ double2 Ga[64], GHa[64];
  const int m = blockIdx.x, i = threadIdx.x;
  if (m >= n) return;
  const double2* __restrict__ am = a + (size_t)m * D;
  const double2* __restrict__ G = gout + (size_t)m * D * D;
  if (i < D) {
    double2 s = make_double2(0.0, 0.0), sh = make_double2(0.0, 0.0);
    for (int e = 0; e < D; ++e) {
      const double2 p = cmul(G[i * D + e], am[e]);
      s.x += p.x; s.y += p.y;
      const double2 q = cmulc(am[e], G[e * D + i]);  // conj(G[e][i]) a_e
      sh.x += q.x; sh.y += q.y;
    }
    Ga[i] = s;
    GHa[i] = sh;
  }
  __syncthreads();
  double2 tr = make_double2(0.0, 0.0), q = make_double2(0.0, 0.0);
  double na = 0.0;
  for (int d = 0; d < D; ++d) {  // rank_one_kernel's order for t and nu
    const double2 c = cov[(size_t)m * D * D + d * D + d];
    tr.x += c.x; tr.y += c.y;
    na += am[d].x * am[d].x + am[d].y * am[d].y;
    const double2 p = cmulc(Ga[d], am[d]);  // conj(a_d) (G a)_d
    q.x += p.x; q.y += p.y;
  }
  const bool nan_bin = !(na > 0.0);
  const double inv = 1.0 / na, k = 2.0 * (tr.x * q.x + tr.y * q.y) * inv * inv;
  if (i < D) {
    const double2 p = cmulc(Ga[i], tr), r = cmul(tr, GHa[i]);  // conj(t) G a, t G^H a
    ga[(size_t)m * D + i] = nan_bin ? make_double2(NAN, NAN)
                                    : make_double2((p.x + r.x) * inv - k * am[i].x, (p.y + r.y) * inv - k * am[i].y);
  }
  for (int idx = i; idx < D * D; idx += blockDim.x) {
    const int d = idx / D, e = idx - d * D;
    gc[(size_t)m * D * D + idx] = nan_bin ? make_double2(NAN, NAN)
                                          : (d == e ? make_double2(q.x * inv, q.y * inv) : make_double2(0.0, 0.0));
  }
}

// ---- y = M x per bin (pbb_matvec_batched_backward): grad M = g x^H, grad x = M^H g ----
// One thread per (bin, row i): row i of grad M and entry i of grad x.
__global__ void matvec_backward_kernel(const double2* __restrict__ M, const double2* __restrict__ x,
                                       const double2* __restrict__ g, int n, int D, double2* __restrict__ gm,
                                       double2* __restrict__ gx) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n * D) return;
  const long long m = idx / D;
  const int i = (int)(idx - m * D);
  const double2* __restrict__ Mm = M + m * D * D;
  const double2* __restrict__ xm = x + m * D;
  const double2* __restrict__ gv = g + m * D;
  const double2 gi = gv[i];
  double2 s = make_double2(0.0, 0.0);
  for (int k = 0; k < D; ++k) {
    gm[m * D * D + (size_t)i * D + k] = cmulc(gi, xm[k]);
    const double2 q = cmulc(gv[k], Mm[k * D + i]);  // conj(M[k][i]) g_k
    s.x += q.x; s.y += q.y;
  }
  gx[idx] = s;
}

}  // namespace pbb
