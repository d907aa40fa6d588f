// Backward passes of the cACGMM's M-step (pbb_cacgmm_mstep_backward) and E-step (pbb_cacgmm_predict_backward).
// The closed forms are stated in include/pbb.h.  Every kernel is fp64; the frame sums of the form
// sum_t c_t z z^H run through launch_em in kModeM (the forward's own scatter kernel), so this file holds only
//   cacgmm_estep_bwd_kernel   per (frame chunk, bin): softmax / clip / log adjoint, qbar, zbar = 2 qbar B^-1 z, ybar
//   cacgmm_predict_spec_bwd_kernel  per (class, bin): Bbar^-1 -> (Vbar, lambar), weight and log det partials
//   cacgmm_mstep_spec_bwd_kernel    per (class, bin): (Vbar, lambar, wbar) -> Cbar -> (Psibar, Sbar)
//   cacgmm_mstep_bwd_kernel   per (frame chunk, bin): gammabar, qbar, saliencybar, zbar = 2 c Psibar z, ybar
// All sums run in a fixed order and no kernel uses atomics, so a backward is bitwise repeatable.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "em_args.cuh"

namespace pbb {

constexpr int kBwdFrames = 64;  // frames per CTA of the per-frame backward kernels
// Two unfloored eigenvalues of the M-step backward count as tied where |mu_i - mu_j| <= kTieGap mu_max (= sqrt(u)):
// past it the divided difference loses at most ~u D mu_max / gap <= sqrt(u) D; below it the eigenvectors themselves
// are not determined to better than that.  A floored and an unfloored eigenvalue (both at the floor's kink, where the
// divided difference lies between 0 and -lam' / lam^2) take the divided difference unless their gap is within the
// rounding of the Rayleigh quotients, kKinkGap D mu_max, where they give 0.
constexpr double kTieGap = 0x1p-26;
constexpr double kKinkGap = 64.0 * 0x1p-52;

// Shared memory of the per-frame kernels: z and zbar as [D][kBwdFrames], one D x D class matrix, nk rows of
// per-frame scalars, then the per-frame norm and projection.
__host__ __device__ inline size_t bwd_frame_smem(int D, int nk) {
  return ((size_t)2 * D * kBwdFrames + (size_t)D * D) * sizeof(double2) +
         ((size_t)nk * kBwdFrames + 2 * kBwdFrames) * sizeof(double);
}

// v rounded to the storage precision of CT
template <typename CT>
__device__ __forceinline__ double2 round_to(double2 v) {
  if constexpr (std::is_same_v<CT, float2>) return make_double2((double)(float)v.x, (double)(float)v.y);
  else return v;
}

// y (F, T, D) -> z[d][i] for the CTA's frames, as normalize_kernel forms it (the same division, rounded through
// the storage type CT as the forward's z is); nrm[i] = the frame's norm, 0 for an all-zero frame.
template <typename CT>
__device__ inline void bwd_load_frames(const CT* __restrict__ y, int f, int T, int D, int t0, int nt,
                                       double2* __restrict__ z, double* __restrict__ nrm) {
  const CT* __restrict__ yf = y + ((size_t)f * T + t0) * D;
  for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
    const int tt = i / D, d = i - tt * D;
    z[d * kBwdFrames + tt] = ld_cplx(yf + i);
  }
  __syncthreads();
  const int i = threadIdx.x;
  if (i < nt) {
    double n2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 v = z[d * kBwdFrames + i];
      n2 += v.x * v.x + v.y * v.y;
    }
    double n = sqrt(n2);
    nrm[i] = n2 == 0.0 ? 0.0 : fmax(n, kTiny);
    if (n == 0.0) n = kTiny;
    n = fmax(n, kTiny);
    for (int d = 0; d < D; ++d) {
      const double2 v = z[d * kBwdFrames + i];
      z[d * kBwdFrames + i] = round_to<CT>(make_double2(v.x / n, v.y / n));
    }
  }
  __syncthreads();
}

// Re(z^H M z) for the thread's frame i (M: D x D row-major in shared memory); with c != 0 also zb += 2 c M z
__device__ inline double bwd_quad(const double2* __restrict__ M, const double2* __restrict__ z,
                                  double2* __restrict__ zb, int D, int i, double c) {
  double qr = 0.0;
  for (int d = 0; d < D; ++d) {
    double re = 0.0, im = 0.0;
    for (int e = 0; e < D; ++e) {
      const double2 m = M[d * D + e], v = z[e * kBwdFrames + i];
      re = fma(m.x, v.x, fma(-m.y, v.y, re));
      im = fma(m.x, v.y, fma(m.y, v.x, im));
    }
    const double2 zd = z[d * kBwdFrames + i];
    qr = fma(zd.x, re, fma(zd.y, im, qr));
    if (c != 0.0) {
      double2& g = zb[d * kBwdFrames + i];
      g.x = fma(2.0 * c, re, g.x);
      g.y = fma(2.0 * c, im, g.y);
    }
  }
  return qr;
}

// ybar (F, T, D) complex128 = (zbar - z Re(z^H zbar)) / |y| per frame; an all-zero frame gets zero
__device__ inline void bwd_store_ybar(double2* __restrict__ ybar, int f, int T, int D, int t0, int nt,
                                      const double2* __restrict__ z, const double2* __restrict__ zb,
                                      const double* __restrict__ nrm, double* __restrict__ proj) {
  const int i = threadIdx.x;
  if (i < nt) {
    double p = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 a = z[d * kBwdFrames + i], b = zb[d * kBwdFrames + i];
      p = fma(a.x, b.x, fma(a.y, b.y, p));
    }
    proj[i] = p;
  }
  __syncthreads();
  double2* __restrict__ out = ybar + ((size_t)f * T + t0) * D;
  for (int j = threadIdx.x; j < nt * D; j += blockDim.x) {
    const int tt = j / D, d = j - tt * D;
    const double n = nrm[tt];
    double2 g = make_double2(0.0, 0.0);
    if (n != 0.0) {
      const double2 a = z[d * kBwdFrames + tt], b = zb[d * kBwdFrames + tt];
      g = make_double2((b.x - a.x * proj[tt]) / n, (b.y - a.y * proj[tt]) / n);
    }
    out[j] = g;
  }
}

// A Hermitian matrix from its slot form: kind 0 = M_dd, kind 1 = r Re M_de, kind 2 = -r Im M_de, with r = 1 for
// scatter sums (em kernels' part) and r = 2 for B^-1 (model_from_eig_warp's coef); every entry times scale
__device__ inline void slots_to_hermitian(const double* __restrict__ c, int D, double scale, bool doubled,
                                          double2* __restrict__ M) {
  const int NS = D * D;
  for (int s = threadIdx.x; s < NS; s += blockDim.x) {
    const int pk = slot_pack(D, s);
    const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
    const double v = (doubled && kind != 0) ? 0.5 * (c[s] * scale) : c[s] * scale;
    if (kind == 0) M[d * D + d] = make_double2(v, 0.0);
    else if (kind == 1) { M[d * D + e].x = v; M[e * D + d].x = v; }
    else { M[d * D + e].y = -v; M[e * D + d].y = v; }
  }
}

struct EstepBwdArgs {
  const void* y;           // (F, T, D) CT
  int F, T, D, K, nch;     // nch: frame chunks of kBwdFrames
  const double* coef;      // (F, K, NS) B^-1 slots (cacg_from_eig_kernel)
  const double* ld;        // (F, K) log det B
  const double* w;         // (F, K)
  const uint8_t* activity; // (F, K, T) or null
  double eps;
  const double* aff;       // (F, K, T) forward outputs
  const double* q;
  const double* gaff;      // (F, K, T) or null
  const double* gq;        // (F, K, T) or null
  const double* gll;       // (F) or null
  double* qcoef;           // (F, K, T) out: the coefficient of z z^H in Bbar^-1
  double* part;            // (F, nch, 2K) out: per chunk sums of wbar and ldbar
  double2* ybar;           // (F, T, D) out
};

template <typename CT>
__global__ void __launch_bounds__(kBwdFrames) cacgmm_estep_bwd_kernel(const EstepBwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = a.D, K = a.K, T = a.T, NS = D * D;
  double2* z = reinterpret_cast<double2*>(smem_raw);
  double2* zb = z + (size_t)D * kBwdFrames;
  double2* M = zb + (size_t)D * kBwdFrames;
  double* qb = reinterpret_cast<double*>(M + NS);        // [K][kBwdFrames] qbar of q (total)
  double* red = qb + (size_t)K * kBwdFrames;             // [2K][kBwdFrames] wbar, ldbar contributions
  double* nrm = red + (size_t)2 * K * kBwdFrames;
  double* proj = nrm + kBwdFrames;
  const int f = blockIdx.x, chunk = blockIdx.y, i = threadIdx.x;
  const int t0 = chunk * kBwdFrames, nt = min(kBwdFrames, T - t0), t = t0 + i;
  const bool valid = i < nt;
  bwd_load_frames(reinterpret_cast<const CT*>(a.y), f, T, D, t0, nt, z, nrm);
  for (int d = 0; d < D; ++d) zb[d * kBwdFrames + i] = make_double2(0.0, 0.0);

  // softmax / clip / log adjoint per frame; e_k = exp(lp_k - m) is kept in red's second half until it is used
  if (valid) {
    const size_t o = (size_t)f * K * T + t;
    double m = -INFINITY;
    for (int k = 0; k < K; ++k)
      m = fmax(m, -(double)D * log(a.q[o + (size_t)k * T]) - a.ld[(size_t)f * K + k]);
    double se = 0.0, den = 0.0, dot = 0.0;
    for (int k = 0; k < K; ++k) {
      const size_t ok = o + (size_t)k * T;
      const double e = exp(-(double)D * log(a.q[ok]) - a.ld[(size_t)f * K + k] - m);
      const double act = (a.activity && !a.activity[ok]) ? 0.0 : 1.0;
      se += e;
      den += act == 0.0 ? 0.0 : e * a.w[(size_t)f * K + k];
      const double g = a.aff[ok];
      const bool pass = a.eps == 0.0 || (g > a.eps && g < 1.0 - a.eps);
      const double gb = (a.gaff && pass) ? a.gaff[ok] : 0.0;
      dot += gb * g;
      qb[k * kBwdFrames + i] = gb;
      red[(K + k) * kBwdFrames + i] = e;
    }
    const double inv = 1.0 / fmax(den, kTiny);
    const double gl = a.gll ? a.gll[f] : 0.0;
    for (int k = 0; k < K; ++k) {
      const size_t ok = o + (size_t)k * T;
      const double e = red[(K + k) * kBwdFrames + i];
      const double act = (a.activity && !a.activity[ok]) ? 0.0 : 1.0;
      const double gb = qb[k * kBwdFrames + i];
      const double abar = (den > kTiny ? gb - dot : gb) * inv;
      const double lpb = abar * a.w[(size_t)f * K + k] * act * e + gl * e / se;
      const double q = a.q[ok];
      qb[k * kBwdFrames + i] = (a.gq ? a.gq[ok] : 0.0) - (double)D * lpb / q;
      red[k * kBwdFrames + i] = abar * e * act;   // wbar
      red[(K + k) * kBwdFrames + i] = -lpb;       // ldbar
    }
  } else {
    for (int k = 0; k < 2 * K; ++k) red[k * kBwdFrames + i] = 0.0;
  }
  __syncthreads();
  double* __restrict__ prow = a.part + ((size_t)f * a.nch + chunk) * 2 * K;
  for (int j = i; j < 2 * K; j += blockDim.x) {
    double s = 0.0;
    for (int tt = 0; tt < nt; ++tt) s += red[j * kBwdFrames + tt];
    prow[j] = s;
  }

  // q = max(|z^H B^-1 z|, tiny): qbar_raw = qbar sign(q_raw) where the floor is not active; zbar += 2 qbar_raw u
  for (int k = 0; k < K; ++k) {
    __syncthreads();
    slots_to_hermitian(a.coef + ((size_t)f * K + k) * NS, D, 1.0, true, M);
    __syncthreads();
    if (valid) {
      const double qr = bwd_quad(M, z, zb, D, i, 0.0);
      const size_t ok = ((size_t)f * K + k) * T + t;
      const double c = a.q[ok] > kTiny ? (qr < 0.0 ? -qb[k * kBwdFrames + i] : qb[k * kBwdFrames + i]) : 0.0;
      a.qcoef[ok] = c;
      if (c != 0.0) bwd_quad(M, z, zb, D, i, c);
    }
  }
  __syncthreads();
  bwd_store_ybar(a.ybar, f, T, D, t0, nt, z, zb, nrm, proj);
}

// Reduces launch_em's chunk partials of one class into S (NS slots) and returns the class's sum of coefficients
__device__ inline double sum_part(const double* __restrict__ part, int f, int nch, int K, int k, int NS,
                                  double* __restrict__ S) {
  const double* __restrict__ p0 = part + ((size_t)f * nch * K + k) * (NS + 1);
  double tot = 0.0;
  for (int s = threadIdx.x; s <= NS; s += blockDim.x) {
    double sum = 0.0;
    for (int c = 0; c < nch; ++c) sum += p0[(size_t)c * K * (NS + 1) + s];
    if (s < NS) S[s] = sum;
    else tot = sum;
  }
  return tot;
}

struct PredictSpecBwdArgs {
  int F, D, K;
  int nch;                 // launch_em chunks of part
  int nchb;                // cacgmm_estep_bwd_kernel chunks of wpart
  const double* part;      // (F, nch, K, NS + 1): sum_t qbar_raw z z^H in slot form
  const double* wpart;     // (F, nchb, 2K)
  const double2* V;        // (F, K, D, D)
  const double* lam;       // (F, K, D)
  double2* gV;             // (F, K, D, D) out
  double* glam;            // (F, K, D) out
  double* gw;              // (F, K) out
};

// One warp per (class, bin): Bbar = sum_t qbar_raw z z^H, Vbar = 2 Bbar V diag(1/lam),
// lambar_x = -v_x^H Bbar v_x / lam_x^2 + ldbar / lam_x, wbar = sum of the frame terms
__global__ void __launch_bounds__(32) cacgmm_predict_spec_bwd_kernel(const PredictSpecBwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = a.D, K = a.K, NS = D * D;
  const int f = blockIdx.x, k = blockIdx.y, lane = threadIdx.x;
  double2* B = reinterpret_cast<double2*>(smem_raw);
  double2* W = B + NS;
  double* S = reinterpret_cast<double*>(W + NS);
  sum_part(a.part, f, a.nch, K, k, NS, S);
  __syncwarp();
  slots_to_hermitian(S, D, 1.0, false, B);
  __syncwarp();
  const size_t mo = ((size_t)f * K + k) * NS;
  const double2* __restrict__ V = a.V + mo;
  const double* __restrict__ lam = a.lam + ((size_t)f * K + k) * D;
  for (int j = lane; j < NS; j += 32) {
    const int d = j / D, x = j - d * D;
    double re = 0.0, im = 0.0;
    for (int e = 0; e < D; ++e) {
      const double2 b = B[d * D + e], v = V[e * D + x];
      re = fma(b.x, v.x, fma(-b.y, v.y, re));
      im = fma(b.x, v.y, fma(b.y, v.x, im));
    }
    W[j] = make_double2(re, im);
    a.gV[mo + j] = make_double2(2.0 * re / lam[x], 2.0 * im / lam[x]);
  }
  __syncwarp();
  double wb = 0.0, ldb = 0.0;
  for (int c = 0; c < a.nchb; ++c) {
    wb += a.wpart[((size_t)f * a.nchb + c) * 2 * K + k];
    ldb += a.wpart[((size_t)f * a.nchb + c) * 2 * K + K + k];
  }
  for (int x = lane; x < D; x += 32) {
    double r = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 v = V[d * D + x], w = W[d * D + x];
      r = fma(v.x, w.x, fma(v.y, w.y, r));
    }
    const double l = lam[x];
    a.glam[((size_t)f * K + k) * D + x] = -r / (l * l) + ldb / l;
  }
  if (lane == 0) a.gw[(size_t)f * K + k] = wb;
}

struct MstepSpecBwdArgs {
  int F, T, D, K, nch;
  const double* part;      // (F, nch, K, NS + 1): the forward's scatter sums (launch_em, kModeM)
  int covariance_norm;     // PBB_NORM_*
  int weight_mode;         // PBB_WEIGHT_TIME or PBB_WEIGHT_CONST
  int has_saliency;
  double eigenvalue_floor;
  const double2* V;        // (F, K, D, D) forward output (ascending)
  const double* lam;       // (F, K, D) forward output
  const double2* gV;       // (F, K, D, D) or null
  const double* glam;      // (F, K, D) or null
  const double* gw;        // (F, K) or null
  double2* gpsi;           // (F, K, D, D) out: Psibar (Hermitian)
  double* gS;              // (F, K) out: Sbar
};

__host__ __device__ inline size_t mstep_spec_bwd_smem(int D) {
  return (size_t)5 * D * D * sizeof(double2) + ((size_t)D * D + 2 * D) * sizeof(double);
}

// One warp per (class, bin): the eigen-adjoint of C = V diag(mu) V^H with mu_x = v_x^H C v_x, through the floor,
// the normalisation and the trace, into Psibar = D Cbar / S and Sbar (pbb.h).
__global__ void __launch_bounds__(32) cacgmm_mstep_spec_bwd_kernel(const MstepSpecBwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = a.D, K = a.K, NS = D * D;
  const int f = blockIdx.x, k = blockIdx.y, lane = threadIdx.x;
  double2* C = reinterpret_cast<double2*>(smem_raw);  // C before the trace normalisation
  double2* Vs = C + NS;
  double2* M = Vs + NS;
  double2* X = M + NS;
  double2* G = X + NS;
  double* S = reinterpret_cast<double*>(G + NS);
  double* mu = S + NS;
  double* mub = mu + D;
  const size_t mo = ((size_t)f * K + k) * NS;
  const double Sk = sum_part(a.part, f, a.nch, K, k, NS, S);
  const double Sk_all = __shfl_sync(0xffffffffu, Sk, NS & 31);  // the lane that summed slot NS
  if (!(Sk_all > kTiny)) {  // a class without weight passes no gradient
    for (int j = lane; j < NS; j += 32) a.gpsi[mo + j] = make_double2(0.0, 0.0);
    if (lane == 0) a.gS[(size_t)f * K + k] = 0.0;
    return;
  }
  __syncwarp();
  const double scale = (double)D / Sk_all;
  slots_to_hermitian(S, D, scale, false, C);
  __syncwarp();
  double tau = 1.0;
  if (a.covariance_norm == PBB_NORM_TRACE) {
    double tr = 0.0;
    for (int d = lane; d < D; d += 32) tr += C[d * D + d].x;
    tr = warp_sum(tr);
    tau = fmax(tr, kTiny);
  }
  const double itau = 1.0 / tau;
  const double2* __restrict__ V = a.V + mo;
  const double* __restrict__ lam = a.lam + ((size_t)f * K + k) * D;
  for (int j = lane; j < NS; j += 32) Vs[j] = V[j];
  __syncwarp();
  // X = C' V, mu_x = Re v_x^H C' v_x (C' = C / tau)
  for (int j = lane; j < NS; j += 32) {
    const int d = j / D, x = j - d * D;
    double re = 0.0, im = 0.0;
    for (int e = 0; e < D; ++e) {
      const double2 c = C[d * D + e], v = Vs[e * D + x];
      re = fma(c.x, v.x, fma(-c.y, v.y, re));
      im = fma(c.x, v.y, fma(c.y, v.x, im));
    }
    X[j] = make_double2(re * itau, im * itau);
  }
  __syncwarp();
  for (int x = lane; x < D; x += 32) {
    double r = 0.0;
    for (int d = 0; d < D; ++d) r = fma(Vs[d * D + x].x, X[d * D + x].x, fma(Vs[d * D + x].y, X[d * D + x].y, r));
    mu[x] = r;
  }
  __syncwarp();
  // mubar through the normalisation and the floor; the top eigenvalue's share goes to mu[D - 1]
  if (lane == 0) {
    const double floor_ = a.eigenvalue_floor;
    const int top = D - 1;
    double topb = 0.0;
    if (a.covariance_norm == PBB_NORM_EIGENVALUE) {
      const double m = fmax(mu[top], kTiny);
      for (int x = 0; x < D; ++x) {
        const double lb = a.glam ? a.glam[((size_t)f * K + k) * D + x] : 0.0;
        const bool pass = lam[x] > floor_;
        mub[x] = pass ? lb / m : 0.0;
        if (pass) topb -= lb * mu[x] / (m * m);
      }
      if (!(mu[top] > kTiny)) topb = 0.0;
    } else {
      const double thr = lam[top] * floor_;
      for (int x = 0; x < D; ++x) {
        const double lb = a.glam ? a.glam[((size_t)f * K + k) * D + x] : 0.0;
        const bool pass = lam[x] > thr;
        mub[x] = pass ? lb : 0.0;
        if (!pass) topb += lb * floor_;
      }
    }
    mub[top] += topb;
  }
  __syncwarp();
  // G = V^H Vbar; M = diag(mubar) + the Vbar term of each pair (pbb.h): the divided difference over mu_c - mu_r, or
  // the tie limit for two unfloored eigenvalues within kTieGap mu_max, or 0 for two floored ones and for a floored and
  // an unfloored one within kKinkGap D mu_max.  Every test is on the divisor itself, so no rounding of lam can send a
  // zero gap into the division.
  const bool eig = a.covariance_norm == PBB_NORM_EIGENVALUE;
  const double thr = eig ? a.eigenvalue_floor : lam[D - 1] * a.eigenvalue_floor;  // unfloored: lam > thr
  const double dl = eig ? 1.0 / fmax(mu[D - 1], kTiny) : 1.0;                  // d lam / d mu where unfloored
  const double tie = kTieGap * mu[D - 1], kink = kKinkGap * D * mu[D - 1];
  for (int j = lane; j < NS; j += 32) {
    const int r = j / D, c = j - r * D;
    double re = 0.0, im = 0.0;
    if (a.gV != nullptr) {
      for (int d = 0; d < D; ++d) {
        const double2 v = Vs[d * D + r], g = a.gV[mo + d * D + c];
        re = fma(v.x, g.x, fma(v.y, g.y, re));
        im = fma(v.x, g.y, fma(-v.y, g.x, im));
      }
    }
    G[j] = make_double2(re, im);
  }
  __syncwarp();
  for (int j = lane; j < NS; j += 32) {
    const int r = j / D, c = j - r * D;
    double2 v = make_double2(0.0, 0.0);
    if (r == c) {
      v.x = mub[r];
    } else {
      const double2 g1 = G[r * D + c], g2 = G[c * D + r];
      const bool pr = lam[r] > thr, pc = lam[c] > thr;
      const double gap = fabs(mu[c] - mu[r]);
      if (pr && pc && !(gap > tie)) {
        // tie limit -lam' P_rc / lam^2, P = V^H Bbar V, from G = 2 P diag(1 / lam):
        // M_rc = -lam' (G_rc + conj G_cr) / (2 (lam_r + lam_c)), Hermitian
        const double s = -dl / (2.0 * (lam[r] + lam[c]));
        v = make_double2((g1.x + g2.x) * s, (g1.y - g2.y) * s);
      } else if ((pr && pc) || ((pr || pc) && gap > kink)) {
        // (M + M^H) / 2 with M_rc = G_rc / (mu_c - mu_r)
        const double inv = 0.5 / (mu[c] - mu[r]);
        v = make_double2((g1.x - g2.x) * inv, (g1.y + g2.y) * inv);
      }
    }
    M[j] = v;
  }
  __syncwarp();
  // X = V M; Cbar' = X V^H (stored in G)
  for (int j = lane; j < NS; j += 32) {
    const int d = j / D, x = j - d * D;
    double re = 0.0, im = 0.0;
    for (int i = 0; i < D; ++i) {
      const double2 v = Vs[d * D + i], m = M[i * D + x];
      re = fma(v.x, m.x, fma(-v.y, m.y, re));
      im = fma(v.x, m.y, fma(v.y, m.x, im));
    }
    X[j] = make_double2(re, im);
  }
  __syncwarp();
  double dotn = 0.0;
  for (int j = lane; j < NS; j += 32) {
    const int d = j / D, e = j - d * D;
    double re = 0.0, im = 0.0;
    for (int i = 0; i < D; ++i) {
      const double2 x = X[d * D + i], v = Vs[e * D + i];  // x * conj(v)
      re = fma(x.x, v.x, fma(x.y, v.y, re));
      im = fma(x.y, v.x, fma(-x.x, v.y, im));
    }
    G[j] = make_double2(re, im);
    const double2 c = C[j];
    dotn += re * c.x + im * c.y;  // Re <Cbar', C>
  }
  dotn = warp_sum(dotn);
  // trace: Cbar = Cbar' / tau - Re<Cbar', C'> / tau I;  then Psibar = D Cbar / S, Sbar = -Re<Cbar, C> / S
  double sub = 0.0, gscale = 1.0;
  if (a.covariance_norm == PBB_NORM_TRACE) {
    gscale = itau;
    double tr = 0.0;
    for (int d = lane; d < D; d += 32) tr += C[d * D + d].x;
    tr = warp_sum(tr);
    sub = tr > kTiny ? dotn * itau * itau : 0.0;
  }
  double dot2 = 0.0;
  for (int j = lane; j < NS; j += 32) {
    const int d = j / D, e = j - d * D;
    double2 g = G[j];
    g.x *= gscale; g.y *= gscale;
    if (d == e) g.x -= sub;
    const double2 c = C[j];
    dot2 += g.x * c.x + g.y * c.y;
    a.gpsi[mo + j] = make_double2(g.x * scale, g.y * scale);
  }
  dot2 = warp_sum(dot2);
  if (lane == 0) {
    double sb = -dot2 / Sk_all;
    const double wb = a.gw ? a.gw[(size_t)f * K + k] : 0.0;
    if (a.weight_mode != PBB_WEIGHT_CONST && a.gw != nullptr) {
      if (!a.has_saliency) {
        sb += wb / (double)a.T;
      } else {
        // w_j = S_j / n, n = sum_j |S_j| (1e-10 if zero); the other classes' S_j are summed as the forward sums them
        double n = 0.0, dotw = 0.0;
        for (int j = 0; j < K; ++j) {
          const double* p0 = a.part + ((size_t)f * a.nch * K + j) * (NS + 1) + NS;
          double sj = 0.0;
          for (int c = 0; c < a.nch; ++c) sj += p0[(size_t)c * K * (NS + 1)];
          n += fabs(sj);
          dotw += a.gw[(size_t)f * K + j] * sj;
        }
        sb += n == 0.0 ? wb / 1e-10 : wb / n - dotw / (n * n);
      }
    }
    a.gS[(size_t)f * K + k] = sb;
  }
}

struct MstepBwdArgs {
  const void* y;           // (F, T, D) CT
  int F, T, D, K, nch;     // nch: frame chunks of kBwdFrames
  const double* aff;       // (F, K, T)
  const double* q;         // (F, K, T) or null (= 1)
  const double* saliency;  // (F, T) or null
  const double2* gpsi;     // (F, K, D, D)
  const double* gS;        // (F, K)
  double* gaff;            // (F, K, T) out
  double* gq;              // (F, K, T) out, or null
  double* gsal;            // (F, T) out, or null
  double2* ybar;           // (F, T, D) out
};

// Per frame: cbar_k = z^H Psibar_k z, c_k = gamma_k s / max(q_k, 10 tiny); zbar = sum_k 2 c_k Psibar_k z;
// gbar = cbar / max(q, 10 tiny) + Sbar; gammabar = gbar s, qbar = -cbar g / q^2, saliencybar = sum_k gbar gamma
template <typename CT>
__global__ void __launch_bounds__(kBwdFrames) cacgmm_mstep_bwd_kernel(const MstepBwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = a.D, K = a.K, T = a.T, NS = D * D;
  double2* z = reinterpret_cast<double2*>(smem_raw);
  double2* zb = z + (size_t)D * kBwdFrames;
  double2* M = zb + (size_t)D * kBwdFrames;
  double* nrm = reinterpret_cast<double*>(M + NS);
  double* proj = nrm + kBwdFrames;
  const int f = blockIdx.x, chunk = blockIdx.y, i = threadIdx.x;
  const int t0 = chunk * kBwdFrames, nt = min(kBwdFrames, T - t0), t = t0 + i;
  const bool valid = i < nt;
  bwd_load_frames(reinterpret_cast<const CT*>(a.y), f, T, D, t0, nt, z, nrm);
  for (int d = 0; d < D; ++d) zb[d * kBwdFrames + i] = make_double2(0.0, 0.0);
  const double sal = (a.saliency && valid) ? a.saliency[(size_t)f * T + t] : 1.0;
  double sbar = 0.0;
  for (int k = 0; k < K; ++k) {
    __syncthreads();
    const double2* __restrict__ P = a.gpsi + ((size_t)f * K + k) * NS;
    for (int j = threadIdx.x; j < NS; j += blockDim.x) M[j] = P[j];
    __syncthreads();
    if (valid) {
      const size_t ok = ((size_t)f * K + k) * T + t;
      const double g = a.aff[ok];
      const double gs = g * sal;
      const double qv = a.q ? a.q[ok] : 1.0;
      const double invq = a.q ? 1.0 / fmax(qv, 10.0 * kTiny) : 1.0;
      const double c = gs * invq;
      const double cb = bwd_quad(M, z, zb, D, i, c);
      const double gbar = cb * invq + a.gS[(size_t)f * K + k];
      a.gaff[ok] = gbar * sal;
      if (a.gq) a.gq[ok] = qv > 10.0 * kTiny ? -cb * gs * invq * invq : 0.0;
      sbar = fma(gbar, g, sbar);
    }
  }
  if (a.gsal && valid) a.gsal[(size_t)f * T + t] = sbar;
  __syncthreads();
  bwd_store_ybar(a.ybar, f, T, D, t0, nt, z, zb, nrm, proj);
}

}  // namespace pbb
