// Complex Bingham distribution and its mixture model (pb_bss/distribution/complex_bingham.py, cbmm.py).
//
// Normaliser: c(lambda) = 2 pi^D exp[lambda_1, ..., lambda_D], the divided difference of exp at the
// eigenvalues (complex_bingham.py:153-164 sums the same expression term by term).  Its derivatives are
// divided differences with repeated nodes:
//   d c / d lambda_k               ~ exp[lambda, lambda_k]
//   d2 c / d lambda_k d lambda_l   ~ exp[lambda, lambda_k, lambda_l]   (times 2 for k == l)
// All of them are entries of exp() of an upper bidiagonal ("Opitz") matrix, computed by scaling and squaring
// (dd_exp), so repeated or close eigenvalues need no special case.
//
// Parameter estimation (find_eigenvalues_v3, complex_bingham.py:304-425): the same equations
// grad_lambda log c(lambda) = s, in the same unknowns (the D - 1 differences of neighbouring sorted lambda,
// largest lambda fixed at 0), the same bounds [-max_concentration, -1e-8] and the same start, solved to
// convergence by a projected Gauss-Newton method with an analytic Jacobian instead of scipy's trust region
// least squares with its default tolerances (which stops at residuals of ~1e-7).
#pragma once
#include "common.cuh"
#include "heig.cuh"

namespace pbb {

constexpr double kBinghamNormEps = 1e-8;   // norm()'s eps, always the default in log_pdf (complex_bingham.py:83)
constexpr double kBinghamUpper = -1e-8;    // upper bound of every difference (complex_bingham.py:404)
constexpr double kBinghamZero = 1e-12;     // scatter eigenvalue <= kBinghamZero * largest: numerically zero
constexpr double kBinghamTol = 1e-12;      // stop at max |residual| <= kBinghamTol
constexpr int kBinghamMaxSteps = 100;      // Gauss-Newton steps
constexpr int kBinghamMaxHalvings = 40;    // step halvings per Gauss-Newton step
constexpr int kBinghamTaylor = 24;         // Taylor degree of exp(A / 2^s), ||A / 2^s|| <= 1

// Status word of the CBMM / Bingham entry points (include/pbb.h): ((kCbMaxIndex - index) << 2) | (4 - kind),
// combined with atomicMax: the smallest failing index wins, and at one index the cause (a bad eigenvalue) wins
// over the non-finite values it leaves for the later iterations of the fit.
constexpr int kCbAssert = 1;     // negative or numerically zero scatter eigenvalue (complex_bingham.py:584)
constexpr int kCbValue = 2;      // infeasible start of the parameter solve (complex_bingham.py:398-408)
constexpr int kCbNonFinite = 3;  // non-finite scatter, parameters or normaliser
constexpr int kCbMaxIndex = (1 << 29) - 1;

__device__ __forceinline__ void cb_report(int* status, long long index, int kind) {
  atomicMax(status, ((kCbMaxIndex - (int)index) << 2) | (4 - kind));
}

// packed upper triangle of an N x N matrix
template <int N> __host__ __device__ constexpr int tri(int i, int j) { return i * N - i * (i - 1) / 2 + (j - i); }

// E = exp(A), A upper bidiagonal with diagonal x (x <= 0) and unit superdiagonal: E[i][j] = exp[x_i, ..., x_j].
// A / 2^s with |x| / 2^s <= 1/2 and superdiagonal 2^-s <= 1, Taylor polynomial by Horner, then s squarings.
// Every entry of exp(A / 2^m) is positive, so the squarings add no cancellation and each entry keeps a relative
// accuracy of a few ulps per squaring (McCurdy, Ng & Parlett, Math. Comp. 43 (1984) 501-528).
template <int N>
__device__ __forceinline__ void dd_exp(const double (&x)[N], double (&E)[N * (N + 1) / 2]) {
  double xm = 0.0;
#pragma unroll
  for (int i = 0; i < N; ++i) xm = fmax(xm, fabs(x[i]));
  if (!(xm < 1e300)) {
#pragma unroll
    for (int i = 0; i < N * (N + 1) / 2; ++i) E[i] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  // xm < 2^(e + 1) with e the binary exponent of xm, so xm / 2^(e + 2) < 1/2
  const int s = xm > 0.5 ? (int)((__double_as_longlong(xm) >> 52) & 0x7ff) - 1023 + 2 : 0;
  const double h = __longlong_as_double((long long)(1023 - s) << 52);
  double m[N];
#pragma unroll
  for (int i = 0; i < N; ++i) m[i] = x[i] * h;
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = i; j < N; ++j) E[tri<N>(i, j)] = i == j ? 1.0 : 0.0;
#pragma unroll 1
  for (int k = kBinghamTaylor; k >= 1; --k) {
    const double ik = 1.0 / (double)k;
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
      for (int j = i; j < N; ++j) {
        double v = m[i] * E[tri<N>(i, j)];
        if (j > i) v = fma(h, E[tri<N>(i + 1, j)], v);
        E[tri<N>(i, j)] = fma(v, ik, i == j ? 1.0 : 0.0);
      }
  }
#pragma unroll 1
  for (int r = 0; r < s; ++r) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      double row[N];
#pragma unroll
      for (int j = i; j < N; ++j) {
        double v = 0.0;
#pragma unroll
        for (int k = i; k <= j; ++k) v = fma(E[tri<N>(i, k)], E[tri<N>(k, j)], v);
        row[j] = v;
      }
#pragma unroll
      for (int j = i; j < N; ++j) E[tri<N>(i, j)] = row[j];
    }
  }
}

// Stable ascending ranks of v (ties by index, like np.argsort on <= 16 values).
template <int D>
__device__ __forceinline__ void stable_ranks(const double (&v)[D], int (&rank)[D]) {
#pragma unroll
  for (int i = 0; i < D; ++i) {
    int r = 0;
#pragma unroll
    for (int j = 0; j < D; ++j) r += (v[j] < v[i] || (v[j] == v[i] && j < i)) ? 1 : 0;
    rank[i] = r;
  }
}

// _remove_duplicate_eigenvalues (complex_bingham.py:188-199) on already sorted values:
// out[0] = v[0], out[i] = v[0] + cumsum(max(diff(v), eps))[i - 1].
template <int D>
__device__ __forceinline__ void gap_rule_sorted(double (&v)[D], double eps) {
  double cs = 0.0;
  double prev = v[0];
#pragma unroll
  for (int i = 1; i < D; ++i) {
    const double cur = v[i];
    cs += fmax(cur - prev, eps);
    prev = cur;
    v[i] = v[0] + cs;
  }
}

// sorted[rank[i]] = v[i]
template <int D>
__device__ __forceinline__ void permute_sorted(const double (&v)[D], const int (&rank)[D], double (&sorted)[D]) {
#pragma unroll
  for (int r = 0; r < D; ++r) {
    double a = 0.0;
#pragma unroll
    for (int i = 0; i < D; ++i) a = rank[i] == r ? v[i] : a;
    sorted[r] = a;
  }
}

// log c(lambda) with the gap rule first (ComplexBingham.log_norm, complex_bingham.py:80-164);
// eps <= 0 skips the gap rule (remove_duplicate_eigenvalues=False).
template <int D>
__device__ __forceinline__ double bingham_log_norm(const double (&lam)[D], double eps) {
  int rank[D];
  double x[D];
  stable_ranks<D>(lam, rank);
  permute_sorted<D>(lam, rank, x);
  if (eps > 0.0) gap_rule_sorted<D>(x, eps);
  const double top = x[D - 1];
#pragma unroll
  for (int i = 0; i < D; ++i) x[i] -= top;  // exp[x + t] = e^t exp[x]
  double E[D * (D + 1) / 2];
  dd_exp<D>(x, E);
  return 0.69314718055994530942 + (double)D * 1.14472988584940017414 + top + log(E[tri<D>(0, D - 1)]);
}

// c, grad c and the Hessian of c at lambda (largest lambda = 0), lane p < D (D + 1) / 2 handles the pair
// (k, l), k <= l, in row-major order of the upper triangle.  Every lane returns g = grad log c and
// H = Hessian of log c (identical in all lanes).
template <int D>
__device__ __forceinline__ void bingham_derivatives(const double (&lam)[D], int lane, double (&g)[D],
                                                    double (&H)[D][D]) {
  constexpr int P = D * (D + 1) / 2;
  int pk = 0, pl = 0;
  {
    int p = 0;
#pragma unroll
    for (int k = 0; k < D; ++k)
#pragma unroll
      for (int l = k; l < D; ++l) {
        if (p == (lane < P ? lane : 0)) { pk = k; pl = l; }
        ++p;
      }
  }
  double x[D + 2];
  double lk = 0.0, ll = 0.0;
#pragma unroll
  for (int i = 0; i < D; ++i) {
    x[i] = lam[i];
    lk = i == pk ? lam[i] : lk;
    ll = i == pl ? lam[i] : ll;
  }
  x[D] = lk;
  x[D + 1] = ll;
  constexpr int N = D + 2;
  double E[N * (N + 1) / 2];
  dd_exp<N>(x, E);
  const double c0 = __shfl_sync(0xffffffffu, E[tri<N>(0, D - 1)], 0);
  const double c1 = E[tri<N>(0, D)];
  const double c2 = E[tri<N>(0, D + 1)];
  const double ic = 1.0 / c0;
  {
    int p = 0;
#pragma unroll
    for (int k = 0; k < D; ++k)
#pragma unroll
      for (int l = k; l < D; ++l) {
        const double v2 = __shfl_sync(0xffffffffu, c2, p);
        if (k == l) g[k] = __shfl_sync(0xffffffffu, c1, p) * ic;
        H[k][l] = (k == l ? 2.0 : 1.0) * v2 * ic;
        ++p;
      }
  }
#pragma unroll
  for (int k = 0; k < D; ++k)
#pragma unroll
    for (int l = k; l < D; ++l) {
      H[k][l] -= g[k] * g[l];
      H[l][k] = H[k][l];
    }
}

// lambda from the differences: np.cumsum([*x, 0][::-1])[::-1] (complex_bingham.py:411)
template <int D>
__device__ __forceinline__ void lambda_from_diff(const double (&x)[D - 1], double (&lam)[D]) {
  lam[D - 1] = 0.0;
#pragma unroll
  for (int i = D - 2; i >= 0; --i) lam[i] = lam[i + 1] + x[i];
}

template <int D>
__device__ __forceinline__ double bingham_residual(const double (&lam)[D], const double (&s)[D], int lane,
                                                   double (&g)[D], double (&H)[D][D], double (&r)[D]) {
  bingham_derivatives<D>(lam, lane, g, H);
  double phi = 0.0;
#pragma unroll
  for (int k = 0; k < D; ++k) {
    r[k] = g[k] - s[k];
    phi = fma(r[k], r[k], phi);
  }
  return phi;
}

// find_eigenvalues_v3 for one problem, warp-cooperative; every lane passes the same s and receives the same
// lambda (same order as s).  Returns 0 or kCbValue (infeasible start: a zero or negative eigenvalue).
template <int D>
__device__ __forceinline__ int bingham_parameters_warp(const double (&s_in)[D], double eps, double max_concentration, int lane,
                                       double (&lam_out)[D]) {
  constexpr int M = D - 1;
  int rank[D];
  double s[D];
  stable_ranks<D>(s_in, rank);
  permute_sorted<D>(s_in, rank, s);
  gap_rule_sorted<D>(s, eps);
  const double lb = -max_concentration, ub = kBinghamUpper;
  const bool finite_mc = isfinite(max_concentration);
  // start (:378-395): x0 = -1 / s, x0[-1] = 0, optionally max(x0, -(max_concentration - d)), then -diff
  double x0[D];
#pragma unroll
  for (int i = 0; i < D; ++i) {
    x0[i] = i == D - 1 ? 0.0 : -1.0 / s[i];
    if (finite_mc) x0[i] = fmax(x0[i], -(max_concentration - (double)i));
  }
  double x[M];
  bool feasible = true;
#pragma unroll
  for (int i = 0; i < M; ++i) {
    x[i] = -(x0[i + 1] - x0[i]);
    // scipy: x0 outside the bounds, or non-finite residuals at x0
    feasible &= x[i] >= lb && x[i] <= ub && isfinite(x[i]);
  }
  if (!feasible) {
#pragma unroll
    for (int i = 0; i < D; ++i) lam_out[i] = __longlong_as_double(0x7ff8000000000000ll);
    return kCbValue;
  }
  double lam[D], g[D], H[D][D], r[D];
  lambda_from_diff<D>(x, lam);
  double phi = bingham_residual<D>(lam, s, lane, g, H, r);
#pragma unroll 1
  for (int it = 0; it < kBinghamMaxSteps; ++it) {
    double rmax = 0.0;
#pragma unroll
    for (int k = 0; k < D; ++k) rmax = fmax(rmax, fabs(r[k]));
    if (!(rmax > kBinghamTol)) break;
    // J = dr/dx = H L, L[i][j] = [i <= j]
    double J[D][M];
#pragma unroll
    for (int k = 0; k < D; ++k) {
      double acc = 0.0;
#pragma unroll
      for (int j = 0; j < M; ++j) {
        acc += H[k][j];
        J[k][j] = acc;
      }
    }
    // active bounds: at a bound with the gradient of |r|^2 / 2 pointing outwards
    bool freev[M];
#pragma unroll
    for (int j = 0; j < M; ++j) {
      double gj = 0.0;
#pragma unroll
      for (int k = 0; k < D; ++k) gj = fma(J[k][j], r[k], gj);
      freev[j] = !((x[j] <= lb && gj > 0.0) || (x[j] >= ub && gj < 0.0));
    }
    // least squares min |J_free d + r| by modified Gram-Schmidt on [J_free | r]
    double R[M][M], qr[M];
    double w[D];
#pragma unroll
    for (int k = 0; k < D; ++k) w[k] = -r[k];
#pragma unroll
    for (int j = 0; j < M; ++j) {
#pragma unroll
      for (int i = 0; i < M; ++i) R[i][j] = 0.0;
      if (!freev[j]) { R[j][j] = 1.0; qr[j] = 0.0; continue; }
#pragma unroll
      for (int i = 0; i < j; ++i) {
        if (!freev[i]) continue;
        double d = 0.0;
#pragma unroll
        for (int k = 0; k < D; ++k) d = fma(J[k][i], J[k][j], d);
        R[i][j] = d;
#pragma unroll
        for (int k = 0; k < D; ++k) J[k][j] = fma(-d, J[k][i], J[k][j]);
      }
      double nn = 0.0;
#pragma unroll
      for (int k = 0; k < D; ++k) nn = fma(J[k][j], J[k][j], nn);
      const double n = sqrt(nn);
      R[j][j] = n;
      const double in = n > 0.0 ? 1.0 / n : 0.0;
#pragma unroll
      for (int k = 0; k < D; ++k) J[k][j] *= in;
      double d = 0.0;
#pragma unroll
      for (int k = 0; k < D; ++k) d = fma(J[k][j], w[k], d);
      qr[j] = d;
#pragma unroll
      for (int k = 0; k < D; ++k) w[k] = fma(-d, J[k][j], w[k]);
    }
    double step[M];
#pragma unroll
    for (int j = M - 1; j >= 0; --j) {
      double v = qr[j];
#pragma unroll
      for (int i = j + 1; i < M; ++i) v = fma(-R[j][i], step[i], v);
      step[j] = (freev[j] && R[j][j] > 0.0) ? v / R[j][j] : 0.0;
    }
    // projected step, halved until |r|^2 decreases
    bool accepted = false, moved = false;
    double alpha = 1.0;
#pragma unroll 1
    for (int h = 0; h < kBinghamMaxHalvings; ++h) {
      double xt[M];
      moved = false;
#pragma unroll
      for (int j = 0; j < M; ++j) {
        xt[j] = fmin(fmax(fma(alpha, step[j], x[j]), lb), ub);
        moved |= xt[j] != x[j];
      }
      if (!moved) break;
      double lt[D], gt[D], Ht[D][D], rt[D];
      lambda_from_diff<D>(xt, lt);
      const double pt = bingham_residual<D>(lt, s, lane, gt, Ht, rt);
      if (pt < phi) {
        accepted = true;
        phi = pt;
#pragma unroll
        for (int j = 0; j < M; ++j) x[j] = xt[j];
#pragma unroll
        for (int k = 0; k < D; ++k) {
          lam[k] = lt[k]; g[k] = gt[k]; r[k] = rt[k];
#pragma unroll
          for (int l = 0; l < D; ++l) H[k][l] = Ht[k][l];
        }
        break;
      }
      alpha *= 0.5;
    }
    if (!accepted) break;  // no further decrease in fp64: converged as far as the equations allow
  }
  // (:417-425) optional clamp at -max_concentration and a second gap rule, then the input order
  if (finite_mc) {
#pragma unroll
    for (int i = 0; i < D; ++i) lam[i] = fmax(lam[i], -max_concentration);
    int rk[D];
    double t[D];
    stable_ranks<D>(lam, rk);
    permute_sorted<D>(lam, rk, t);
    gap_rule_sorted<D>(t, eps);
#pragma unroll
    for (int i = 0; i < D; ++i) {
      double a = 0.0;
#pragma unroll
      for (int j = 0; j < D; ++j) a = rk[i] == j ? t[j] : a;
      lam[i] = a;
    }
  }
#pragma unroll
  for (int i = 0; i < D; ++i) {
    double a = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) a = rank[i] == j ? lam[j] : a;
    lam_out[i] = a;
  }
  return 0;
}

// Batched find_eigenvalues_v3: one warp per problem, s (n, D) -> lambda (n, D).
template <int D>
__global__ void __launch_bounds__(128) bingham_parameters_kernel(const double* __restrict__ s, int n, double eps,
                                                                 double max_concentration,
                                                                 double* __restrict__ lam, int* status) {
  const int lane = threadIdx.x & 31;
  const long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= n) return;
  double sv[D], out[D];
#pragma unroll
  for (int i = 0; i < D; ++i) sv[i] = s[p * D + i];
  const int kind = bingham_parameters_warp<D>(sv, eps, max_concentration, lane, out);
  bool bad = kind != 0;
#pragma unroll
  for (int i = 0; i < D; ++i) bad |= !isfinite(out[i]);
  if (lane < D) {
#pragma unroll
    for (int i = 0; i < D; ++i)
      if (i == lane) lam[p * D + i] = out[i];
  }
  if (lane == 0 && bad) cb_report(status, p, kind ? kind : kCbNonFinite);
}

// log c (ComplexBingham.log_norm), one thread per problem.  eps <= 0: no gap rule.
template <int D>
__global__ void bingham_log_norm_kernel(const double* __restrict__ lam, int n, double eps, double* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  double v[D];
#pragma unroll
  for (int i = 0; i < D; ++i) v[i] = lam[p * D + i];
  out[p] = bingham_log_norm<D>(v, eps);
}

// ComplexBingham.log_pdf (complex_bingham.py:59-78): Re(y^H V diag(lambda) V^H y) - log c
// = sum_x lambda_x |(V^H y)_x|^2 - log c for y (M, T, D) as given (not normalised), V (M, D, D),
// lambda (M, D); one thread per (m, t).
template <typename CT>
__global__ void bingham_log_pdf_kernel(const CT* __restrict__ y, const double2* __restrict__ V,
                                       const double* __restrict__ lam, const double* __restrict__ log_norm,
                                       int M, int T, int D, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * T) return;
  const long long m = i / T;
  const CT* yt = y + i * D;
  const double2* Vm = V + m * D * D;
  double q = 0.0;
  for (int x = 0; x < D; ++x) {
    double pr = 0.0, pi = 0.0;  // (V^H y)_x = sum_d conj(V_dx) y_d
    for (int d = 0; d < D; ++d) {
      const double2 v = Vm[d * D + x], yd = ld_cplx(yt + d);
      pr += v.x * yd.x + v.y * yd.y;
      pi += v.x * yd.y - v.y * yd.x;
    }
    q = fma(lam[m * D + x], pr * pr + pi * pi, q);
  }
  out[i] = q - log_norm[m];
}

// --------------------------------------------------------------------------
// CBMM model update: one CTA per bin, one warp per class.  complex_bingham.py:567-594 (scatter, hermitian
// eigh, eigenvalue check, find_eigenvalues_v3) and estimate_mixture_weight's saliency branch
// (cbmm.py:128-129, 222-226).  E-step form for the shared EM kernels (model_kind 1, lp = ew q - ld):
// coef = slots of -B = -V diag(lambda) V^H (positive semi-definite, so the kernels' |q| is q), ew = -1,
// ld = log c(lambda) with the gap rule of norm() (eps 1e-8).
// --------------------------------------------------------------------------
constexpr int kCbWarps = 4;

struct CbUpdArgs {
  int F, T, K;
  int nch;
  const double* part;   // (F, NCH, K, NS + 1)
  int weight_mode;
  double eigenvalue_eps, max_concentration;
  double2* evec;        // (F, K, D, D) out, columns = eigenvectors, ascending eigenvalues
  double* eval;         // (F, K, D) out
  double* weight;       // (F, K) out
  double* coef; double* ld; double* ew;
  int* status;
};

// slots of sum_x w[x] v_x v_x^H, same convention as model_from_eig_warp (em_kernels.cuh)
__device__ inline void slots_from_eig(const double2* __restrict__ V, const double* __restrict__ w,
                                      const int* __restrict__ tab, int D, int lane, double* __restrict__ out) {
  for (int s = lane; s < D * D; s += 32) {
    const int pk = tab[s];
    const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
    double re = 0.0, im = 0.0;
    for (int x = 0; x < D; ++x) {
      const double2 vd = V[d * D + x], ve = V[e * D + x];
      re = fma(vd.x * ve.x + vd.y * ve.y, w[x], re);
      im = fma(vd.y * ve.x - vd.x * ve.y, w[x], im);
    }
    out[s] = kind == 0 ? re : (kind == 1 ? 2.0 * re : -2.0 * im);
  }
}

template <int D>
__global__ void __launch_bounds__(32 * kCbWarps, 1) cb_update_kernel(const CbUpdArgs u) {
  constexpr int NS = D * D;
  __shared__ __align__(16) double2 A_s[kCbWarps][NS];
  __shared__ __align__(16) double2 V_s[kCbWarps][NS];
  __shared__ double S_s[kCbWarps][NS];
  __shared__ double w_s[kCbWarps][D];
  __shared__ double sumg[32];
  __shared__ int tab[NS];
  const int K = u.K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x;
  double2* A = A_s[warp];
  double2* V = V_s[warp];
  double* S = S_s[warp];
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();
  for (int k = warp; k < K; k += kCbWarps) {
    const long long idx = (long long)f * K + k;
    const double* __restrict__ p0 = u.part + ((size_t)f * u.nch * K + k) * (NS + 1);
    for (int s = lane; s <= NS; s += 32) {
      double sum = 0.0;
      for (int c = 0; c < u.nch; ++c) sum += p0[(size_t)c * K * (NS + 1) + s];
      if (s < NS) S[s] = sum; else sumg[k] = sum;
    }
    __syncwarp();
    // 1. S = sum gamma sal y y^H / sum gamma sal (no floor on the denominator, complex_bingham.py:578)
    const double scale = 1.0 / sumg[k];
    bool bad = false;
    double* Ad = reinterpret_cast<double*>(A);
    for (int s = lane; s < NS; s += 32) {
      const int pk = tab[s];
      const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
      const double v = S[s] * scale;
      bad |= !isfinite(v);
      if (kind == 0) { Ad[2 * (d * D + d)] = v; Ad[2 * (d * D + d) + 1] = 0.0; }
      else if (kind == 1) { Ad[2 * (d * D + e)] = v; Ad[2 * (e * D + d)] = v; }
      else { Ad[2 * (d * D + e) + 1] = -v; Ad[2 * (e * D + d) + 1] = v; }
    }
    bad = __any_sync(0xffffffffu, bad);
    __syncwarp();
    // 2. eigh, ascending
    warp_jacobi_small<D>(A, V, lane);
    int rank[D];
    double sv[D], s_sorted[D];
#pragma unroll
    for (int x = 0; x < D; ++x) sv[x] = A[x * D + x].x;
    stable_ranks<D>(sv, rank);
    permute_sorted<D>(sv, rank, s_sorted);
    // 3. assert every scatter eigenvalue >= 0, and not numerically zero
    int kind = bad ? kCbNonFinite : 0;
    if (!kind && !(s_sorted[0] > kBinghamZero * s_sorted[D - 1])) kind = kCbAssert;
    // 4. find_eigenvalues_v3
    double lam[D];
    if (!kind) kind = bingham_parameters_warp<D>(s_sorted, u.eigenvalue_eps, u.max_concentration, lane, lam);
    if (kind) {
#pragma unroll
      for (int i = 0; i < D; ++i) lam[i] = __longlong_as_double(0x7ff8000000000000ll);
    }
    // 5. outputs in eigh order; lambda back in Jacobi order for the E-step form
    double2* __restrict__ Vo = u.evec + (size_t)idx * NS;
    double* __restrict__ lo = u.eval + (size_t)idx * D;
#pragma unroll
    for (int x = 0; x < D; ++x) {
      double lx = 0.0;
#pragma unroll
      for (int r = 0; r < D; ++r) lx = rank[x] == r ? lam[r] : lx;
      if (lane == 0) w_s[warp][x] = -lx;
      if (lane < D) Vo[lane * D + rank[x]] = V[lane * D + x];
    }
    if (lane < D) {
#pragma unroll
      for (int i = 0; i < D; ++i)
        if (i == lane) lo[i] = lam[i];
    }
    __syncwarp();
    if (u.coef != nullptr) slots_from_eig(V, w_s[warp], tab, D, lane, u.coef + (size_t)idx * NS);
    if (lane == 0) {
      const double l = kind ? lam[0] : bingham_log_norm<D>(lam, kBinghamNormEps);
      if (!kind && !isfinite(l)) kind = kCbNonFinite;
      u.ld[idx] = l;
      u.ew[idx] = -1.0;
      if (kind) cb_report(u.status, idx, kind);
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < K) {
    const int k = threadIdx.x;
    double wk;
    if (u.weight_mode == PBB_WEIGHT_CONST) {
      wk = 1.0 / K;
    } else {  // saliency branch of estimate_mixture_weight (cbmm.py:128-129 sets saliency = 1)
      double n1 = 0.0;
      for (int j = 0; j < K; ++j) n1 += fabs(sumg[j]);
      wk = sumg[k] / (n1 == 0.0 ? 1e-10 : n1);
    }
    u.weight[(size_t)f * K + k] = wk;
  }
}

// (eigenvectors, eigenvalues, weight) -> E-step form, for CBMM.predict (cbmm.py:26-55)
struct CbFromModelArgs {
  int F, K;
  const double2* evec; const double* eval; const double* weight;  // weight may be null (1/K)
  double* coef; double* ld; double* ew; double* w;
};

template <int D>
__global__ void __launch_bounds__(32 * kCbWarps) cb_from_model_kernel(const CbFromModelArgs u) {
  constexpr int NS = D * D;
  __shared__ __align__(16) double2 V_s[kCbWarps][NS];
  __shared__ double w_s[kCbWarps][D];
  __shared__ int tab[NS];
  const int K = u.K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x;
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();
  for (int k = warp; k < K; k += kCbWarps) {
    const size_t idx = (size_t)f * K + k;
    for (int i = lane; i < NS; i += 32) V_s[warp][i] = u.evec[idx * NS + i];
    if (lane < D) w_s[warp][lane] = -u.eval[idx * D + lane];
    __syncwarp();
    slots_from_eig(V_s[warp], w_s[warp], tab, D, lane, u.coef + idx * NS);
    if (lane == 0) {
      double lam[D];
#pragma unroll
      for (int i = 0; i < D; ++i) lam[i] = u.eval[idx * D + i];
      u.ld[idx] = bingham_log_norm<D>(lam, kBinghamNormEps);
      u.ew[idx] = -1.0;
      u.w[idx] = u.weight ? u.weight[idx] : 1.0 / K;
    }
    __syncwarp();
  }
}

}  // namespace pbb
