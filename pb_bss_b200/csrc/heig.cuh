// Warp-cooperative complex Hermitian eigensolver (parallel-order cyclic Jacobi).
//
// One warp diagonalises one D x D Hermitian matrix held in shared memory.
// Each round applies D/2 disjoint plane rotations (round-robin tournament
// ordering), so a sweep is D-1 rounds of fully parallel row/column updates.
// The rotation test |a_pq|^2 <= eps^2 |a_pp a_qq| gives the high relative
// accuracy Jacobi is known for on positive definite matrices, which matters
// here because 1/lambda of near-singular speech covariances feeds the E-step.
//
// Replaces np.linalg.eigh at pb_bss/distribution/complex_angular_central_gaussian.py:95,
// pb_bss/utils.py:154 and (after a Cholesky reduction) scipy.linalg.eigh(a, b) /
// LAPACK zhegvd at pb_bss/extraction/cythonized/get_gev_vector.pyx:124.
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kJacobiMaxSweeps = 40;

// shared memory a warp needs: A (D*D double2) + V (D*D double2) + rot ((D+1)/2 * 6 doubles)
__host__ __device__ inline size_t jacobi_smem_bytes(int D) {
  return (size_t)2 * D * D * sizeof(double2) + (size_t)((D + 1) / 2) * 6 * sizeof(double);
}

// In: A Hermitian (row-major, ld = D) in shared memory.  Out: A diagonal holds
// the eigenvalues (unsorted), V the eigenvectors as columns.  If `V_init` is
// true V is taken as given (and must be consistent with A = V0^H A0 V0, the
// warm start); otherwise V is set to the identity.  Returns the number of
// sweeps used.  All 32 lanes must call.
__device__ inline int warp_jacobi(double2* __restrict__ A, double2* __restrict__ V,
                                  double* __restrict__ rot, int D, int lane, bool V_init = false) {
  const int n = D + (D & 1);  // tournament size (a dummy player for odd D)
  const int npair = n / 2;
  const double eps2 = DBL_EPSILON * DBL_EPSILON;
  if (!V_init) {
    for (int i = lane; i < D * D; i += 32) V[i] = make_double2((i / D == i % D) ? 1.0 : 0.0, 0.0);
  }
  __syncwarp();
  int sweep = 0;
  for (; sweep < kJacobiMaxSweeps; ++sweep) {
    unsigned rotated = 0;
    for (int r = 0; r < n - 1; ++r) {
      // ---- (a) rotation parameters, one lane per pair (lanes take pairs l, l + 32, ... for D > 64) ----
      bool act = false;
      for (int pl = lane; pl < npair; pl += 32) {
        const int m = n - 1;
        int p, q;
        if (pl == 0) { p = r % m; q = n - 1; }
        else { p = (r + pl) % m; q = (r - pl + m) % m; }
        if (p > q) { int t = p; p = q; q = t; }
        double c = 1.0, sr = 0.0, si = 0.0, an = 0.0, dn = 0.0;
        bool pact = false;
        if (q < D) {
          const double a = A[p * D + p].x, d = A[q * D + q].x;
          const double2 b = A[p * D + q];
          const double m2 = b.x * b.x + b.y * b.y;
          if (m2 > eps2 * fabs(a * d) && m2 > 1e-300) {
            pact = true;
            const double dl = 0.5 * (d - a);
            const double sg = dl >= 0.0 ? 1.0 : -1.0;
            const double h = fabs(dl) + sqrt(dl * dl + m2);
            const double w = rsqrt(h * h + m2);
            c = h * w;
            sr = sg * b.x * w;
            si = sg * b.y * w;
            const double tb = sg * m2 / h;
            an = a - tb;
            dn = d + tb;
          }
        }
        double* ro = rot + pl * 6;
        ro[0] = c; ro[1] = sr; ro[2] = si; ro[3] = an; ro[4] = dn;
        ro[5] = pact ? (double)(p | (q << 8)) : -1.0;  // packed pair or "inactive"
        act |= pact;
      }
      const unsigned any = __ballot_sync(0xffffffffu, act);
      rotated |= any;
      __syncwarp();
      if (any == 0) continue;
      // ---- (b) column updates of A and V: X <- X J ---------------------------
      for (int task = lane; task < npair * D * 2; task += 32) {
        const int pi = task / (2 * D);
        const int rem = task - pi * 2 * D;
        const double* ro = rot + pi * 6;
        if (ro[5] < 0.0) continue;
        const int pq = (int)ro[5];
        const int p = pq & 255, q = pq >> 8;
        double2* X = rem < D ? A : V;
        const int i = rem < D ? rem : rem - D;
        const double c = ro[0], sr = ro[1], si = ro[2];
        const double2 xp = X[i * D + p], xq = X[i * D + q];
        // x_p' = c x_p - conj(s) x_q ; x_q' = s x_p + c x_q
        X[i * D + p] = make_double2(c * xp.x - (sr * xq.x + si * xq.y), c * xp.y - (sr * xq.y - si * xq.x));
        X[i * D + q] = make_double2(c * xq.x + (sr * xp.x - si * xp.y), c * xq.y + (sr * xp.y + si * xp.x));
      }
      __syncwarp();
      // ---- (c) row updates of A: A <- J^H A ----------------------------------
      for (int task = lane; task < npair * D; task += 32) {
        const int pi = task / D;
        const int j = task - pi * D;
        const double* ro = rot + pi * 6;
        if (ro[5] < 0.0) continue;
        const int pq = (int)ro[5];
        const int p = pq & 255, q = pq >> 8;
        const double c = ro[0], sr = ro[1], si = ro[2];
        const double2 ap = A[p * D + j], aq = A[q * D + j];
        // a_p' = c a_p - s a_q ; a_q' = conj(s) a_p + c a_q
        A[p * D + j] = make_double2(c * ap.x - (sr * aq.x - si * aq.y), c * ap.y - (sr * aq.y + si * aq.x));
        A[q * D + j] = make_double2(c * aq.x + (sr * ap.x + si * ap.y), c * aq.y + (sr * ap.y - si * ap.x));
      }
      __syncwarp();
      // ---- exact values for the rotated 2x2 blocks ---------------------------
      for (int pl = lane; pl < npair; pl += 32) {
        const double* ro = rot + pl * 6;
        if (ro[5] >= 0.0) {
          const int pq = (int)ro[5];
          const int p = pq & 255, q = pq >> 8;
          A[p * D + q] = make_double2(0.0, 0.0);
          A[q * D + p] = make_double2(0.0, 0.0);
          A[p * D + p] = make_double2(ro[3], 0.0);
          A[q * D + q] = make_double2(ro[4], 0.0);
        }
      }
      __syncwarp();
    }
    if (rotated == 0) break;
  }
  return sweep + 1;
}

// Same algorithm for compile-time D <= 8: one lane per (pair, row/column) task -- D/2 pairs x D
// entries fit one warp -- every lane derives its pair's rotation itself (no staging through
// shared memory, no integer division, no task loops): 3 warp syncs per round.
template <int D>
__device__ __forceinline__ int warp_jacobi_small(double2* __restrict__ A, double2* __restrict__ V, int lane) {
  static_assert(D >= 2 && D <= 8, "small-D Jacobi");
  constexpr int n = D + (D & 1), npair = n / 2, m = n - 1;
  const double eps2 = DBL_EPSILON * DBL_EPSILON;
  for (int i = lane; i < D * D; i += 32) V[i] = make_double2((i / D == i % D) ? 1.0 : 0.0, 0.0);
  __syncwarp();
  const int pi = lane / D, idx = lane - pi * D;  // pair index within the round, row / column index
  const bool lane_on = pi < npair;
  int sweep = 0;
  for (; sweep < kJacobiMaxSweeps; ++sweep) {
    unsigned rotated = 0;
#pragma unroll 1
    for (int r = 0; r < m; ++r) {
      int p = 0, q = 0;
      bool act = false;
      double c = 1.0, sr = 0.0, si = 0.0, an = 0.0, dn = 0.0;
      if (lane_on) {
        if (pi == 0) { p = r % m; q = n - 1; }
        else { p = (r + pi) % m; q = (r - pi + m) % m; }
        if (p > q) { const int t = p; p = q; q = t; }
        if (q < D) {
          const double a = A[p * D + p].x, d = A[q * D + q].x;
          const double2 b = A[p * D + q];
          const double m2 = b.x * b.x + b.y * b.y;
          if (m2 > eps2 * fabs(a * d) && m2 > 1e-300) {
            act = true;
            const double dl = 0.5 * (d - a);
            const double sg = dl >= 0.0 ? 1.0 : -1.0;
            const double h = fabs(dl) + sqrt(dl * dl + m2);
            const double w = rsqrt(h * h + m2);
            c = h * w;
            sr = sg * b.x * w;
            si = sg * b.y * w;
            const double tb = sg * m2 / h;
            an = a - tb;
            dn = d + tb;
          }
        }
      }
      const unsigned any = __ballot_sync(0xffffffffu, act);
      rotated |= any;
      if (any == 0) continue;
      __syncwarp();  // everyone has read the pivots
      // column update X <- X J for row idx of A and of V
      if (act) {
        const double2 xp = A[idx * D + p], xq = A[idx * D + q];
        A[idx * D + p] = make_double2(c * xp.x - (sr * xq.x + si * xq.y), c * xp.y - (sr * xq.y - si * xq.x));
        A[idx * D + q] = make_double2(c * xq.x + (sr * xp.x - si * xp.y), c * xq.y + (sr * xp.y + si * xp.x));
        const double2 vp = V[idx * D + p], vq = V[idx * D + q];
        V[idx * D + p] = make_double2(c * vp.x - (sr * vq.x + si * vq.y), c * vp.y - (sr * vq.y - si * vq.x));
        V[idx * D + q] = make_double2(c * vq.x + (sr * vp.x - si * vp.y), c * vq.y + (sr * vp.y + si * vp.x));
      }
      __syncwarp();
      // row update A <- J^H A for column idx
      if (act) {
        const double2 ap = A[p * D + idx], aq = A[q * D + idx];
        A[p * D + idx] = make_double2(c * ap.x - (sr * aq.x - si * aq.y), c * ap.y - (sr * aq.y + si * aq.x));
        A[q * D + idx] = make_double2(c * aq.x + (sr * ap.x + si * ap.y), c * aq.y + (sr * ap.y - si * ap.x));
      }
      __syncwarp();
      if (act && idx == 0) {  // exact values for the rotated 2x2 block
        A[p * D + q] = make_double2(0.0, 0.0);
        A[q * D + p] = make_double2(0.0, 0.0);
        A[p * D + p] = make_double2(an, 0.0);
        A[q * D + q] = make_double2(dn, 0.0);
      }
      __syncwarp();
    }
    if (rotated == 0) break;
  }
  return sweep + 1;
}

// dispatch on the runtime dimension: templated path for D <= 8, generic otherwise
__device__ inline int warp_jacobi_any(double2* __restrict__ A, double2* __restrict__ V, double* __restrict__ rot,
                                      int D, int lane) {
  switch (D) {
    case 2: return warp_jacobi_small<2>(A, V, lane);
    case 3: return warp_jacobi_small<3>(A, V, lane);
    case 4: return warp_jacobi_small<4>(A, V, lane);
    case 5: return warp_jacobi_small<5>(A, V, lane);
    case 6: return warp_jacobi_small<6>(A, V, lane);
    case 7: return warp_jacobi_small<7>(A, V, lane);
    case 8: return warp_jacobi_small<8>(A, V, lane);
    default: return warp_jacobi(A, V, rot, D, lane);
  }
}

// Largest eigenpair of a Hermitian positive semi-definite D x D matrix (D <= 8) WITHOUT a full eigendecomposition:
// B <- A / tr A, then kTopSquarings times B <- B B / tr(B B), which is A^(2^n) up to scale and converges to the
// projector v v^H at the rate (lambda_2 / lambda_1)^(2^n); v is the column of the largest diagonal entry, the
// eigenvalue its Rayleigh quotient with the ORIGINAL A.  Accepted only if the residual |A v - lambda v|_inf is
// below 1e-13 lambda (spectra with lambda_2 / lambda_1 > ~0.9995 fail that test): the caller then runs the
// Jacobi solver, so the result is always as exact as np.linalg.eigh's.  A is left untouched; B, C: D x D scratch.
// One lane per matrix entry (two for D = 8).  x_out: D entries in shared memory.
constexpr int kTopSquarings = 16;
template <int D>
__device__ __forceinline__ bool warp_top_eigenpair(const double2* __restrict__ A, double2* __restrict__ B,
                                                   double2* __restrict__ C, int lane, double* __restrict__ lambda,
                                                   double2* __restrict__ x_out) {
  constexpr int NS = D * D, PER = (NS + 31) / 32;
  double tr = 0.0;
#pragma unroll
  for (int d = 0; d < D; ++d) tr += A[d * D + d].x;
  if (!(tr > 0.0) || !(tr < 1e300)) return false;
  const double itr = 1.0 / tr;
  for (int i = lane; i < NS; i += 32) B[i] = make_double2(A[i].x * itr, A[i].y * itr);
  __syncwarp();
#pragma unroll 1
  for (int n = 0; n < kTopSquarings; ++n) {
    double2 c[PER];
#pragma unroll
    for (int r = 0; r < PER; ++r) {
      const int i = lane + 32 * r;
      c[r] = make_double2(0.0, 0.0);
      if (i < NS) {
        const int row = i / D, col = i - row * D;
#pragma unroll
        for (int k = 0; k < D; ++k) {
          const double2 a = B[row * D + k], b = B[k * D + col];
          c[r].x = fma(a.x, b.x, fma(-a.y, b.y, c[r].x));
          c[r].y = fma(a.x, b.y, fma(a.y, b.x, c[r].y));
        }
        C[i] = c[r];
      }
    }
    __syncwarp();
    double t2 = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) t2 += C[d * D + d].x;
    const double s = 1.0 / t2;
    double change = 0.0;
#pragma unroll
    for (int r = 0; r < PER; ++r) {
      const int i = lane + 32 * r;
      if (i < NS) {
        const double2 nb = make_double2(c[r].x * s, c[r].y * s);
        change = fmax(change, fabs(nb.x - B[i].x) + fabs(nb.y - B[i].y));
        B[i] = nb;
      }
    }
    __syncwarp();
    // B is a fixed point of the squaring (a projector) once nothing moves any more: stop early
    if (n >= 4 && !__any_sync(0xffffffffu, change > 1e-16)) break;
  }
  // dominant column
  int best = 0;
  double bmax = B[0].x;
#pragma unroll
  for (int d = 1; d < D; ++d) {
    const double v = B[d * D + d].x;
    if (v > bmax) { bmax = v; best = d; }
  }
  double n2 = 0.0;
#pragma unroll
  for (int d = 0; d < D; ++d) { const double2 v = B[d * D + best]; n2 += v.x * v.x + v.y * v.y; }
  if (!(n2 > 0.0)) return false;
  const double inv = rsqrt(n2);
  if (lane < D) x_out[lane] = make_double2(B[lane * D + best].x * inv, B[lane * D + best].y * inv);
  __syncwarp();
  // y = A x (every lane computes all of it: D is tiny), lambda = Re(x^H y), residual
  double2 y[D];
  double lam = 0.0;
#pragma unroll
  for (int r = 0; r < D; ++r) {
    y[r] = make_double2(0.0, 0.0);
#pragma unroll
    for (int k = 0; k < D; ++k) {
      const double2 a = A[r * D + k], v = x_out[k];
      y[r].x = fma(a.x, v.x, fma(-a.y, v.y, y[r].x));
      y[r].y = fma(a.x, v.y, fma(a.y, v.x, y[r].y));
    }
    lam += x_out[r].x * y[r].x + x_out[r].y * y[r].y;
  }
  double res = 0.0;
#pragma unroll
  for (int r = 0; r < D; ++r)
    res = fmax(res, fabs(y[r].x - lam * x_out[r].x) + fabs(y[r].y - lam * x_out[r].y));
  *lambda = lam;
  return res <= 1e-13 * lam;
}

// rank of eigenvalue i in ascending order (stable), for i < D; lanes >= D get -1.
// For D > 32 callers loop (i = lane, lane + 32, ...).
__device__ inline int eig_rank(const double2* A, int D, int i) {
  const double li = A[i * D + i].x;
  int rank = 0;
  for (int j = 0; j < D; ++j) {
    const double lj = A[j * D + j].x;
    rank += (lj < li) || (lj == li && j < i);
  }
  return rank;
}

}  // namespace pbb
