// EM kernels for the complex angular central Gaussian mixture model (cACGMM).
//
// Data layout in HBM (one fit):
//   z      (F, D, T) complex  unit-norm observation, frames contiguous
//   coef   (F, K, D*D) f64    B_k^{-1} in "slot" form (see common.cuh), so that
//                             q_kt = sum_s coef[k][s] * psi_t[s]
//   ld/w/ew (F, K) f64        log det, mixture weight, w * exp(ld_min - ld)
//   part   (F, NCH, K, D*D+1) per frame-chunk partial scatter sums + sum of gamma
//
// One EM iteration = em kernel (E-step of iteration i fused with the M-step
// accumulation) + update kernel (normalise, Hermitian Jacobi eigensolve, floor,
// rebuild coef).  The observation is read once per iteration; gamma and the
// quadratic form never round-trip through HBM.
#pragma once
#include "common.cuh"
#include "em_args.cuh"
#include "heig.cuh"

namespace pbb {

template <int N> __device__ __forceinline__ double ipow(double x) {
  if constexpr (N == 1) return x;
  else if constexpr (N % 2 == 0) { const double y = ipow<N / 2>(x); return y * y; }
  else return x * ipow<N - 1>(x);
}

// Posterior of one frame from the K quadratic forms.
//   reference: log_pdf = -D log q - log det                (cacg.py:200-201)
//              gamma = softmax_k(log_pdf) * w [* activity], renormalised with
//              the denominator floored at tiny, optional clip
//              (mixture_model_utils.py:7-55)
// fast != 0: gamma_k ~ w_k e^{-(ld_k - ld_min)} (q_min / q_k)^D, the same
// quantity without log/exp; every factor is <= 1 so nothing overflows, and
// the host only enables it when the largest term cannot underflow
// (2 D log10(1/floor) < 280, 'eigenvalue' normalisation).
// Outputs gam[k], invq[k] = 1 / max(q, 10 tiny) (cacg.py:310-314) and,
// if want_ll, logsumexp_k log_pdf (cacgmm.py:137).
template <int D, int K>
__device__ __forceinline__ void em_softmax(const double (&q)[K], const double* __restrict__ ld,
                                           const double* __restrict__ w, const double* __restrict__ ew,
                                           const uint8_t* __restrict__ act, size_t act_stride, bool fast,
                                           double eps, bool want_ll, double (&gam)[K], double (&invq)[K],
                                           double& ll) {
  double a[K];
  if (fast) {
    double qmin = q[0];
#pragma unroll
    for (int k = 1; k < K; ++k) qmin = fmin(qmin, q[k]);
    qmin = fmax(qmin, 10.0 * kTiny);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      invq[k] = 1.0 / fmax(q[k], 10.0 * kTiny);
      a[k] = ew[k] * ipow<D>(qmin * invq[k]);
    }
    ll = 0.0;
  } else {
    double lp[K];
    double m = -INFINITY;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      lp[k] = -(double)D * log(q[k]) - ld[k];
      m = fmax(m, lp[k]);
      invq[k] = 1.0 / fmax(q[k], 10.0 * kTiny);
    }
    double se = 0.0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double e = exp(lp[k] - m);
      se += e;
      a[k] = e * w[k];
    }
    ll = want_ll ? m + log(se) : 0.0;
  }
  double den = 0.0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (act != nullptr) a[k] = act[k * act_stride] ? a[k] : 0.0;
    den += a[k];
  }
  const double inv = 1.0 / fmax(den, kTiny);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double g = a[k] * inv;
    if (eps != 0.0) g = fmin(fmax(g, eps), 1.0 - eps);
    gam[k] = g;
  }
}

// Complex Watson posterior of one frame: log_pdf = kappa |m^H z|^2 - log c(kappa)
// (complex_watson.py:73-87), then the same softmax (mixture_model_utils.py:7-55,
// affiliation_eps = 0, cwmm.py:161).  q[k] = |m_k^H z|^2 arrives as the slot-form
// quadratic form of the rank-1 matrix m m^H.
// A non-zero eps clips the posterior to [eps, 1 - eps] (CBMM, cbmm.py:41-55).
template <int K>
__device__ __forceinline__ void watson_softmax(const double (&q)[K], const double* __restrict__ lognorm,
                                               const double* __restrict__ w, const double* __restrict__ kappa,
                                               double eps, double (&gam)[K]) {
  double lp[K];
  double m = -INFINITY;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    lp[k] = kappa[k] * q[k] - lognorm[k];
    m = fmax(m, lp[k]);
  }
  double den = 0.0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    gam[k] = exp(lp[k] - m) * w[k];
    den += gam[k];
  }
  const double inv = 1.0 / fmax(den, kTiny);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    gam[k] *= inv;
    if (eps != 0.0) gam[k] = fmin(fmax(gam[k], eps), 1.0 - eps);
  }
}

// --------------------------------------------------------------------------
// Fast path: D <= 8, K <= 4.  One CTA = 4 warps = one (bin, frame-chunk).
// The D*D slots are split into 4 groups, one per warp; lane = frame.  Each
// warp forms the outer-product slots of its group once per frame and uses
// them twice: for its share of the K quadratic forms (E-step; shares are
// combined through shared memory) and for its share of the K weighted scatter
// matrices (M-step, 3*16 fp64 accumulators per lane at D=8, K=3).  That is
// 2 D^2 (1 + K) fp64 FMA-pipe operations per frame -- the minimum for the
// B^{-1}-form of the cACG E-step plus the Hermitian M-step.
// --------------------------------------------------------------------------
constexpr int kEmGroups = 4;

template <int D, int K>
struct EmFastSmem {
  static constexpr int NS = D * D;
  static constexpr int NSG = (NS + kEmGroups - 1) / kEmGroups;
  static constexpr int NSGP = NSG + (NSG & 1);
  double coef[kEmGroups][K][NSGP];
  double xq[2][kEmGroups][K][32];
  double ld[K], w[K], ew[K];
};

template <int D, int K, typename CT, int GI>
__device__ __forceinline__ void em_fast_group(const EmArgs& a, EmFastSmem<D, K>& sm, int f, int chunk,
                                              int lane) {
  using S = EmFastSmem<D, K>;
  constexpr int NS = S::NS, NSG = S::NSG;
  constexpr unsigned need = slot_range_channels(D, GI * NSG, GI * NSG + NSG);
  const int T = a.T;
  const int zs = a.zs;
  const CT* __restrict__ zf = reinterpret_cast<const CT*>(a.z) + (size_t)f * D * zs;
  const int t_begin = chunk * a.frames_per_block;
  const int t_end = min(T, t_begin + a.frames_per_block);
  const int mode = a.mode;
  const bool fast = a.softmax_fast != 0;
  const bool want_ll = a.loglik_part != nullptr;

  double acc[K * NSG];
#pragma unroll
  for (int i = 0; i < K * NSG; ++i) acc[i] = 0.0;
  double sg[K];
#pragma unroll
  for (int k = 0; k < K; ++k) sg[k] = 0.0;
  double llsum = 0.0;
  int buf = 0;

  for (int t0 = t_begin; t0 < t_end; t0 += 32) {
    const int t = t0 + lane;
    const bool valid = t < t_end;
    double zr[D], zi[D];
    static_for<D>([&](auto dd) {
      constexpr int d = decltype(dd)::value;
      if constexpr ((need >> d) & 1u) {
        double2 v = make_double2(0.0, 0.0);
        if (valid) v = ld_cplx(zf + (size_t)d * zs + t);
        zr[d] = v.x; zi[d] = v.y;
      }
    });
    double psi[NSG];
    static_for<NSG>([&](auto ii) {
      constexpr int i = decltype(ii)::value;
      constexpr int s = GI * NSG + i;
      if constexpr (s < NS) {
        constexpr SlotInfo si = slot_info(D, s);
        if constexpr (si.kind == 0) psi[i] = zr[si.d] * zr[si.d] + zi[si.d] * zi[si.d];
        else if constexpr (si.kind == 1) psi[i] = zr[si.d] * zr[si.e] + zi[si.d] * zi[si.e];
        else psi[i] = zr[si.d] * zi[si.e] - zi[si.d] * zr[si.e];
      } else {
        psi[i] = 0.0;
      }
    });

    double gam[K], invq[K];
    if (mode != kModeM) {
      // ---- E-step: this group's share of the K quadratic forms -------------
#pragma unroll
      for (int k = 0; k < K; ++k) {
        double pq = 0.0;
#pragma unroll
        for (int i = 0; i < NSG; ++i) pq = fma(sm.coef[GI][k][i], psi[i], pq);
        sm.xq[buf][GI][k][lane] = pq;
      }
      __syncthreads();
      double q[K];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        double v = sm.xq[buf][0][k][lane];
#pragma unroll
        for (int g = 1; g < kEmGroups; ++g) v += sm.xq[buf][g][k][lane];
        q[k] = fmax(fabs(v), kTiny);  // cacg.py:185-199
      }
      buf ^= 1;
      double ll;
      const uint8_t* act = a.activity ? a.activity + ((size_t)f * K) * T + (valid ? t : 0) : nullptr;
      if (a.model_kind == 1) {
        if (a.w_time != nullptr) {  // frequency-tied weights, see below
          double wl[K];
#pragma unroll
          for (int k = 0; k < K; ++k) wl[k] = a.w_time[(size_t)k * (a.w_time_st ? T : 1) + (a.w_time_st && valid ? t : 0)];
          watson_softmax<K>(q, sm.ld, wl, sm.ew, a.aff_eps, gam);
        } else {
          watson_softmax<K>(q, sm.ld, sm.w, sm.ew, a.aff_eps, gam);
        }
#pragma unroll
        for (int k = 0; k < K; ++k) invq[k] = 1.0;
        ll = 0.0;
      } else if (a.w_time != nullptr) {
        // frequency-tied mixture weights (weight_constant_axis=-3, mixture_model_utils.py:187-190):
        // one weight per (class, frame) shared by all bins; log-domain softmax
        double wl[K];
#pragma unroll
        for (int k = 0; k < K; ++k) wl[k] = a.w_time[(size_t)k * (a.w_time_st ? T : 1) + (a.w_time_st && valid ? t : 0)];
        em_softmax<D, K>(q, sm.ld, wl, sm.ew, act, (size_t)T, false, a.aff_eps, want_ll, gam, invq, ll);
      } else {
        em_softmax<D, K>(q, sm.ld, sm.w, sm.ew, act, (size_t)T, fast, a.aff_eps, want_ll, gam, invq, ll);
      }
      if (GI == 0 && valid) {
        llsum += ll;
        if (a.aff_out) {
#pragma unroll
          for (int k = 0; k < K; ++k) a.aff_out[((size_t)f * K + k) * T + t] = gam[k];
        }
        if (a.q_out) {
#pragma unroll
          for (int k = 0; k < K; ++k) a.q_out[((size_t)f * K + k) * T + t] = q[k];
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const size_t o = ((size_t)f * K + k) * T + (valid ? t : 0);
        gam[k] = a.aff_in ? a.aff_in[o] : 1.0;
        invq[k] = a.q_in ? 1.0 / fmax(a.q_in[o], 10.0 * kTiny) : 1.0;
      }
    }
    if (mode != kModeE) {
      // ---- M-step: sum_t (gamma * saliency / q) * psi ----------------------
      const double sal = a.saliency ? a.saliency[(size_t)f * T + (valid ? t : 0)] : 1.0;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double gs = valid ? gam[k] * sal : 0.0;
        const double c = gs * invq[k];
        if (GI == 0) sg[k] += gs;
#pragma unroll
        for (int i = 0; i < NSG; ++i) acc[k * NSG + i] = fma(c, psi[i], acc[k * NSG + i]);
      }
    }
  }

  // ---- reduce over the 32 frames of the warp and publish ---------------------
  if (mode != kModeE) {
    double* __restrict__ prow = a.part + ((size_t)f * a.nch + chunk) * K * (NS + 1);
    warp_reduce_halving<K * NSG>(acc, lane);
    int lo, hi;
    reduce_range<K * NSG>(lane, lo, hi);
#pragma unroll
    for (int j = 0; j < HalvingSizes<K * NSG>::n5; ++j) {
      const int idx = lo + j;
      if (idx < hi) {
        const int k = idx / NSG, i = idx - k * NSG;
        const int s = GI * NSG + i;
        if (s < NS) prow[(size_t)k * (NS + 1) + s] = acc[j];
      }
    }
    if (GI == 0) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double v = warp_sum(sg[k]);
        if (lane == 0) prow[(size_t)k * (NS + 1) + NS] = v;
      }
    }
  }
  if (GI == 0 && want_ll) {
    const double v = warp_sum(llsum);
    if (lane == 0) a.loglik_part[(size_t)f * a.nch + chunk] = v;
  }
}

template <int D, int K, typename CT>
__global__ void __launch_bounds__(32 * kEmGroups, 3) em_fast_kernel(const EmArgs a) {
  using S = EmFastSmem<D, K>;
  __shared__ __align__(16) S sm;
  const int f = a.f0 + blockIdx.y, chunk = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (a.mode != kModeM) {
    const double* __restrict__ cf = a.coef + (size_t)f * K * S::NS;
    for (int i = threadIdx.x; i < kEmGroups * K * S::NSGP; i += blockDim.x) {
      const int g = i / (K * S::NSGP);
      const int r = i - g * (K * S::NSGP);
      const int k = r / S::NSGP, j = r - k * S::NSGP;
      const int s = g * S::NSG + j;
      sm.coef[g][k][j] = (j < S::NSG && s < S::NS) ? cf[(size_t)k * S::NS + s] : 0.0;
    }
    if (threadIdx.x < K) {
      sm.ld[threadIdx.x] = a.ld[(size_t)f * K + threadIdx.x];
      sm.w[threadIdx.x] = a.w[(size_t)f * K + threadIdx.x];
      sm.ew[threadIdx.x] = a.ew[(size_t)f * K + threadIdx.x];
    }
    __syncthreads();
  }
  switch (warp) {
    case 0: em_fast_group<D, K, CT, 0>(a, sm, f, chunk, lane); break;
    case 1: em_fast_group<D, K, CT, 1>(a, sm, f, chunk, lane); break;
    case 2: em_fast_group<D, K, CT, 2>(a, sm, f, chunk, lane); break;
    default: em_fast_group<D, K, CT, 3>(a, sm, f, chunk, lane); break;
  }
}

// --------------------------------------------------------------------------
// Generic path: any D < 35, K < 20 (the reference's own limits,
// cacgmm.py:249-250).  Phase 1: thread = frame, E-step with coef read through
// L1; phase 2: thread = (class, slot), loops over the chunk's frames.  No
// cross-thread reduction is needed, sums are deterministic.
// --------------------------------------------------------------------------
constexpr int kGenFrames = 128;  // frames per block of the generic kernel

template <typename CT>
__global__ void __launch_bounds__(kGenFrames) em_generic_kernel(const EmArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = a.D, K = a.K, T = a.T, NS = D * D;
  double* c_s = reinterpret_cast<double*>(smem_raw);          // [K][kGenFrames]
  double* g_s = c_s + (size_t)K * kGenFrames;                 // [K][kGenFrames] gamma*saliency
  int* tab = reinterpret_cast<int*>(g_s + (size_t)K * kGenFrames);  // [NS]
  __shared__ double red[kGenFrames / 32];
  const int f = a.f0 + blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x;
  const int t_begin = chunk * kGenFrames;
  const int t_end = min(T, t_begin + kGenFrames);
  const int t = t_begin + tid;
  const bool valid = t < t_end;
  const int zs = a.zs;
  const CT* __restrict__ zf = reinterpret_cast<const CT*>(a.z) + (size_t)f * D * zs;
  for (int s = tid; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();

  double gam[kMaxK], invq[kMaxK];
  double ll = 0.0;
  if (a.mode != kModeM) {
    double q[kMaxK];
    for (int k = 0; k < K; ++k) q[k] = 0.0;
    if (valid) {
      const double* __restrict__ cf = a.coef + (size_t)f * K * NS;
      for (int s = 0; s < NS; ++s) {
        const int pk = tab[s];
        const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
        const double2 zd = ld_cplx(zf + (size_t)d * zs + t);
        const double2 ze = ld_cplx(zf + (size_t)e * zs + t);
        const double psi = kind == 2 ? zd.x * ze.y - zd.y * ze.x : zd.x * ze.x + zd.y * ze.y;
        for (int k = 0; k < K; ++k) q[k] = fma(cf[(size_t)k * NS + s], psi, q[k]);
      }
    }
    double m = -INFINITY;
    double lp[kMaxK];
    for (int k = 0; k < K; ++k) {
      q[k] = fmax(fabs(q[k]), kTiny);
      if (a.model_kind == 1) {
        lp[k] = a.ew[(size_t)f * K + k] * q[k] - a.ld[(size_t)f * K + k];
        invq[k] = 1.0;
      } else {
        lp[k] = -(double)D * log(q[k]) - a.ld[(size_t)f * K + k];
        invq[k] = 1.0 / fmax(q[k], 10.0 * kTiny);
      }
      m = fmax(m, lp[k]);
    }
    double se = 0.0, den = 0.0;
    for (int k = 0; k < K; ++k) {
      const double e = exp(lp[k] - m);
      se += e;
      const double wk = a.w_time ? a.w_time[(size_t)k * (a.w_time_st ? T : 1) + (a.w_time_st && valid ? t : 0)]
                                : a.w[(size_t)f * K + k];
      double av = e * wk;
      if (a.activity && valid) av = a.activity[((size_t)f * K + k) * T + t] ? av : 0.0;
      gam[k] = av;
      den += av;
    }
    ll = valid ? m + log(se) : 0.0;
    const double inv = 1.0 / fmax(den, kTiny);
    for (int k = 0; k < K; ++k) {
      double g = gam[k] * inv;
      if (a.aff_eps != 0.0) g = fmin(fmax(g, a.aff_eps), 1.0 - a.aff_eps);
      gam[k] = g;
      if (valid) {
        if (a.aff_out) a.aff_out[((size_t)f * K + k) * T + t] = g;
        if (a.q_out) a.q_out[((size_t)f * K + k) * T + t] = q[k];
      }
    }
  } else {
    for (int k = 0; k < K; ++k) {
      const size_t o = ((size_t)f * K + k) * T + (valid ? t : 0);
      gam[k] = a.aff_in ? a.aff_in[o] : 1.0;
      invq[k] = a.q_in ? 1.0 / fmax(a.q_in[o], 10.0 * kTiny) : 1.0;
    }
  }
  if (a.loglik_part) {
    const double v = warp_sum(ll);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
      double sum = 0.0;
      for (int i = 0; i < kGenFrames / 32; ++i) sum += red[i];
      a.loglik_part[(size_t)f * a.nch + chunk] = sum;
    }
  }
  if (a.mode == kModeE) return;
  const double sal = (a.saliency && valid) ? a.saliency[(size_t)f * T + t] : 1.0;
  for (int k = 0; k < K; ++k) {
    const double gs = valid ? gam[k] * sal : 0.0;
    g_s[k * kGenFrames + tid] = gs;
    c_s[k * kGenFrames + tid] = gs * invq[k];
  }
  __syncthreads();
  const int nt = t_end - t_begin;
  double* __restrict__ prow = a.part + ((size_t)f * a.nch + chunk) * K * (NS + 1);
  for (int idx = tid; idx < K * (NS + 1); idx += blockDim.x) {
    const int k = idx / (NS + 1), s = idx - k * (NS + 1);
    double sum = 0.0;
    if (s == NS) {
      for (int i = 0; i < nt; ++i) sum += g_s[k * kGenFrames + i];
    } else {
      const int pk = tab[s];
      const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
      const CT* zd = zf + (size_t)d * zs + t_begin;
      const CT* ze = zf + (size_t)e * zs + t_begin;
      for (int i = 0; i < nt; ++i) {
        const double2 vd = ld_cplx(zd + i), ve = ld_cplx(ze + i);
        const double psi = kind == 2 ? vd.x * ve.y - vd.y * ve.x : vd.x * ve.x + vd.y * ve.y;
        sum = fma(c_s[k * kGenFrames + i], psi, sum);
      }
    }
    prow[idx] = sum;
  }
}

// --------------------------------------------------------------------------
// Model update: one CTA per bin, one warp per class (looping if K is larger
// than the warps that fit).  complex_angular_central_gaussian.py:306-338 +
// from_covariance :81-132 + estimate_mixture_weight
// (mixture_model_utils.py:133-203).
// --------------------------------------------------------------------------
struct UpdArgs {
  int F, T, D, K;
  int nch;
  const double* part;   // (F, NCH, K, NS + 1)
  int covariance_norm;  // PBB_NORM_*
  int weight_mode;      // PBB_WEIGHT_*
  int has_saliency;
  double eigenvalue_floor;
  double2* evec;        // (F, K, D, D) out
  double* eval;         // (F, K, D) out
  double* weight;       // (F, K) out
  double* coef;         // (F, K, NS) out
  double* ld;           // (F, K) out
  double* ew;           // (F, K) out
  int* status;
  int warps;            // warps per CTA
};

// coef / ld from eigenvectors V (columns, shared memory, ld = D) and floored
// eigenvalues lam[x] (shared).  B^{-1} = V diag(1/lam) V^H,
// complex_angular_central_gaussian.py:185-199 with the 'optimal' einsum path.
__device__ inline double model_from_eig_warp(const double2* __restrict__ V, const double* __restrict__ lam,
                                             const int* __restrict__ tab, int D, int lane,
                                             double* __restrict__ coef_out) {
  const int NS = D * D;
  for (int s = lane; s < NS; s += 32) {
    const int pk = tab[s];
    const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
    double re = 0.0, im = 0.0;
    for (int x = 0; x < D; ++x) {
      const double2 vd = V[d * D + x], ve = V[e * D + x];
      const double il = 1.0 / lam[x];
      // vd * conj(ve)
      re = fma(vd.x * ve.x + vd.y * ve.y, il, re);
      im = fma(vd.y * ve.x - vd.x * ve.y, il, im);
    }
    coef_out[s] = kind == 0 ? re : (kind == 1 ? 2.0 * re : -2.0 * im);
  }
  double l = 0.0;
  for (int x = lane; x < D; x += 32) l += log(lam[x]);
  return warp_sum(l);
}

__host__ __device__ inline size_t update_smem_per_warp(int D) {
  const size_t b = jacobi_smem_bytes(D) + (size_t)(D * D + D + 1) * sizeof(double);
  return (b + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t from_eig_smem_per_warp(int D) {
  const size_t b = (size_t)D * D * sizeof(double2) + (size_t)D * sizeof(double);
  return (b + 15) & ~(size_t)15;
}

__global__ void cacg_update_kernel(const UpdArgs u) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = u.D, K = u.K, NS = D * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x;
  // layout: per warp [A | V | rot | S(NS) | lam(D)], then shared [sumg(K) | ld(K) | tab(NS)]
  const size_t per_warp = update_smem_per_warp(D);
  unsigned char* mine = smem_raw + per_warp * warp;
  double2* A = reinterpret_cast<double2*>(mine);
  double2* V = A + NS;
  double* rot = reinterpret_cast<double*>(V + NS);
  double* S = rot + ((D + 1) / 2) * 6;
  double* lam = S + NS;
  double* sumg = reinterpret_cast<double*>(smem_raw + per_warp * u.warps);
  double* ld_s = sumg + K;
  int* tab = reinterpret_cast<int*>(ld_s + K);
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();

  for (int k = warp; k < K; k += u.warps) {
    // 1. sum the per-chunk partials in a fixed order
    const double* __restrict__ p0 = u.part + ((size_t)f * u.nch * K + k) * (NS + 1);
    for (int s = lane; s <= NS; s += 32) {
      double sum = 0.0;
      for (int c = 0; c < u.nch; ++c) sum += p0[(size_t)c * K * (NS + 1) + s];
      if (s < NS) S[s] = sum; else sumg[k] = sum;
    }
    __syncwarp();
    // 2. covariance = D * S / max(sum gamma, tiny)      (cacg.py:316-330); for sum gamma <= tiny as D S / tiny,
    // since D / tiny overflows for D >= 4 (2^-1022 is tiny, so the division is an exact power-of-two scaling)
    const bool live = sumg[k] > kTiny;
    const double scale = (double)D / fmax(sumg[k], kTiny);
    bool bad = false;
    double* Ad = reinterpret_cast<double*>(A);
    for (int s = lane; s < NS; s += 32) {
      const int pk = tab[s];
      const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
      const double v = live ? S[s] * scale : ((double)D * S[s]) * 0x1p1022;
      bad |= !isfinite(v);
      if (kind == 0) { Ad[2 * (d * D + d)] = v; Ad[2 * (d * D + d) + 1] = 0.0; }
      else if (kind == 1) { Ad[2 * (d * D + e)] = v; Ad[2 * (e * D + d)] = v; }
      else { Ad[2 * (d * D + e) + 1] = -v; Ad[2 * (e * D + d) + 1] = v; }  // Sigma_de = conj(psi_de)
    }
    __syncwarp();
    if (u.covariance_norm == PBB_NORM_TRACE) {  // cacg.py:88-90
      double tr = 0.0;
      for (int d = lane; d < D; d += 32) tr += A[d * D + d].x;
      tr = warp_sum(tr);
      const double it = 1.0 / fmax(tr, kTiny);
      for (int i = lane; i < NS; i += 32) { A[i].x *= it; A[i].y *= it; }
      __syncwarp();
    }
    // 3. eigendecomposition                                (cacg.py:95)
    warp_jacobi_any(A, V, rot, D, lane);
    // 4. normalise + floor                                 (cacg.py:111-126)
    double lmax = -INFINITY;
    for (int d = lane; d < D; d += 32) lmax = fmax(lmax, A[d * D + d].x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = fmax(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    for (int d = lane; d < D; d += 32) {
      double l = A[d * D + d].x;
      if (u.covariance_norm == PBB_NORM_EIGENVALUE) l = fmax(l / fmax(lmax, kTiny), u.eigenvalue_floor);
      else l = fmax(l, lmax * u.eigenvalue_floor);
      bad |= !isfinite(l);
      lam[d] = l;
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMax(u.status, f + 1);
    __syncwarp();
    // 5. outputs, ascending like np.linalg.eigh
    double2* __restrict__ Vo = u.evec + ((size_t)f * K + k) * NS;
    double* __restrict__ lo = u.eval + ((size_t)f * K + k) * D;
    for (int x = lane; x < D; x += 32) {
      const int r = eig_rank(A, D, x);
      lo[r] = lam[x];
      for (int d = 0; d < D; ++d) Vo[d * D + r] = V[d * D + x];
    }
    // 6. E-step form of the model (not needed after the last iteration of a fit: coef == nullptr)
    if (u.coef != nullptr) {
      const double ldk = model_from_eig_warp(V, lam, tab, D, lane, u.coef + ((size_t)f * K + k) * NS);
      if (lane == 0) ld_s[k] = ldk;
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < K) {
    const int k = threadIdx.x;
    double wk;
    if (u.weight_mode == PBB_WEIGHT_CONST) {
      wk = 1.0 / K;
    } else if (!u.has_saliency) {
      wk = sumg[k] / (double)u.T;  // np.mean over time
    } else {
      double n1 = 0.0;  // _unit_norm(ord=1, axis=-2, eps=1e-10, 'where')
      for (int j = 0; j < K; ++j) n1 += fabs(sumg[j]);
      wk = sumg[k] / (n1 == 0.0 ? 1e-10 : n1);
    }
    u.weight[(size_t)f * K + k] = wk;
    if (u.coef != nullptr) {
      double ldmin = ld_s[0];
      for (int j = 1; j < K; ++j) ldmin = fmin(ldmin, ld_s[j]);
      u.ld[(size_t)f * K + k] = ld_s[k];
      u.ew[(size_t)f * K + k] = wk * exp(ldmin - ld_s[k]);
    }
  }
}

// Model given as (eigenvectors, eigenvalues, weight) -> E-step form.  Used by
// predict and by a warm-started fit (cacgmm.py:229-234).
struct FromEigArgs {
  int F, D, K;
  const double2* evec;
  const double* eval;
  const double* weight;   // (F, K) or null (constant 1/K)
  double* coef; double* ld; double* w; double* ew;
  int warps;
};

__global__ void cacg_from_eig_kernel(const FromEigArgs u) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = u.D, K = u.K, NS = D * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x;
  const size_t per_warp = from_eig_smem_per_warp(D);
  unsigned char* mine = smem_raw + per_warp * warp;
  double2* V = reinterpret_cast<double2*>(mine);
  double* lam = reinterpret_cast<double*>(V + NS);
  double* ld_s = reinterpret_cast<double*>(smem_raw + per_warp * u.warps);
  int* tab = reinterpret_cast<int*>(ld_s + K);
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();
  for (int k = warp; k < K; k += u.warps) {
    const double2* __restrict__ Vi = u.evec + ((size_t)f * K + k) * NS;
    for (int i = lane; i < NS; i += 32) V[i] = Vi[i];
    for (int d = lane; d < D; d += 32) lam[d] = u.eval[((size_t)f * K + k) * D + d];
    __syncwarp();
    const double ldk = model_from_eig_warp(V, lam, tab, D, lane, u.coef + ((size_t)f * K + k) * NS);
    if (lane == 0) ld_s[k] = ldk;
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < K) {
    const int k = threadIdx.x;
    const double wk = u.weight ? u.weight[(size_t)f * K + k] : 1.0 / K;
    double ldmin = ld_s[0];
    for (int j = 1; j < K; ++j) ldmin = fmin(ldmin, ld_s[j]);
    u.w[(size_t)f * K + k] = wk;
    u.ld[(size_t)f * K + k] = ld_s[k];
    u.ew[(size_t)f * K + k] = wk * exp(ldmin - ld_s[k]);
  }
}

// --------------------------------------------------------------------------
// Complex Watson model update (complex_watson.py:300-315, pb_bss/utils.py:111-169):
// covariance = S / sum(gamma), mode = eigenvector of the largest eigenvalue,
// concentration = inverse hypergeometric ratio of that eigenvalue, evaluated on
// the quadratic B-spline the host built with the reference's own recipe
// (complex_watson.py:237-256): knots t[0..n+2], coefficients c[0..n-1].
// --------------------------------------------------------------------------
struct CwSpline {
  const double* t;   // n + 3 knots
  const double* c;   // n coefficients
  int n;
  double x_lo, x_hi;     // domain of the interpolant (first / last eigenvalue marker)
  double max_concentration;
};

__device__ inline double cw_spline_eval(const CwSpline& sp, double x) {
  if (!(x == x)) return x;                      // NaN in, NaN out
  // domain of the interpolant = first / last knot, read from the table (no host round trip)
  if (x < __ldg(sp.t)) return 0.0;               // fill_value = (0, max_concentration)
  if (x > __ldg(sp.t + sp.n + 2)) return sp.max_concentration;
  const int k = 2, n = sp.n;
  int lo = k, hi = n;  // find i in [k, n-1] with t[i] <= x < t[i+1]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sp.t[mid] <= x) lo = mid; else hi = mid;
  }
  const int i = lo;
  double d0 = sp.c[i - 2], d1 = sp.c[i - 1], d2 = sp.c[i];
  // de Boor, degree 2
  double a2 = (x - sp.t[i]) / (sp.t[i + 2] - sp.t[i]);
  double a1 = (x - sp.t[i - 1]) / (sp.t[i + 1] - sp.t[i - 1]);
  d2 = (1.0 - a2) * d1 + a2 * d2;
  d1 = (1.0 - a1) * d0 + a1 * d1;
  a2 = (x - sp.t[i]) / (sp.t[i + 1] - sp.t[i]);
  return (1.0 - a2) * d1 + a2 * d2;
}

struct CwUpdArgs {
  int F, T, D, K;
  int nch;
  const double* part;   // (F, NCH, K, NS + 1)
  int weight_mode;
  CwSpline spline;
  double2* mode;        // (F, K, D) out
  double* concentration;  // (F, K) out
  double* weight;       // (F, K) out
  double* coef; double* ld; double* ew;  // E-step form: slots of m m^H, log norm, kappa
  int* status;
  int warps;
};

// slots of the rank-1 matrix m m^H
__device__ inline void cw_coef_from_mode(const double2* __restrict__ m, const int* __restrict__ tab, int D, int lane,
                                         double* __restrict__ coef_out) {
  const int NS = D * D;
  for (int s = lane; s < NS; s += 32) {
    const int pk = tab[s];
    const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
    const double2 md = m[d], me = m[e];
    const double re = md.x * me.x + md.y * me.y, im = md.y * me.x - md.x * me.y;  // m_d conj(m_e)
    coef_out[s] = kind == 0 ? re : (kind == 1 ? 2.0 * re : -2.0 * im);
  }
}

__global__ void cw_update_kernel(const CwUpdArgs u) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = u.D, K = u.K, NS = D * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x;
  const size_t per_warp = update_smem_per_warp(D);
  unsigned char* mine = smem_raw + per_warp * warp;
  double2* A = reinterpret_cast<double2*>(mine);
  double2* V = A + NS;
  double* rot = reinterpret_cast<double*>(V + NS);
  double* S = rot + ((D + 1) / 2) * 6;
  double* sumg = reinterpret_cast<double*>(smem_raw + per_warp * u.warps);
  int* tab = reinterpret_cast<int*>(sumg + 2 * K);
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();
  for (int k = warp; k < K; k += u.warps) {
    const double* __restrict__ p0 = u.part + ((size_t)f * u.nch * K + k) * (NS + 1);
    for (int s = lane; s <= NS; s += 32) {
      double sum = 0.0;
      for (int c = 0; c < u.nch; ++c) sum += p0[(size_t)c * K * (NS + 1) + s];
      if (s < NS) S[s] = sum; else sumg[k] = sum;
    }
    __syncwarp();
    const double scale = 1.0 / sumg[k];  // complex_watson.py:311-312: no floor on the denominator
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
    __syncwarp();
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMax(u.status, f + 1);
    warp_jacobi_any(A, V, rot, D, lane);
    // largest eigenvalue; ties resolved like "last of the ascending order"
    int best = 0;
    double lmax = A[0].x;
    for (int d = 1; d < D; ++d) {
      const double l = A[d * D + d].x;
      if (l >= lmax) { lmax = l; best = d; }
    }
    const double kappa = cw_spline_eval(u.spline, lmax);
    double2* __restrict__ mo = u.mode + ((size_t)f * K + k) * D;
    double2* mloc = reinterpret_cast<double2*>(S);  // S is dead now: reuse for the mode vector
    for (int d = lane; d < D; d += 32) {
      const double2 v = V[d * D + best];
      mo[d] = v;
      mloc[d] = v;
    }
    __syncwarp();
    cw_coef_from_mode(mloc, tab, D, lane, u.coef + ((size_t)f * K + k) * NS);
    if (lane == 0) {
      u.concentration[(size_t)f * K + k] = kappa;
      u.ew[(size_t)f * K + k] = kappa;
      u.ld[(size_t)f * K + k] = cw_log_norm(kappa, D);
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x < K) {
    const int k = threadIdx.x;
    double wk;
    if (u.weight_mode == PBB_WEIGHT_CONST) {
      wk = 1.0 / K;
    } else {  // saliency branch of estimate_mixture_weight (cwmm.py:129-130 sets saliency = 1)
      double n1 = 0.0;
      for (int j = 0; j < K; ++j) n1 += fabs(sumg[j]);
      wk = sumg[k] / (n1 == 0.0 ? 1e-10 : n1);
    }
    u.weight[(size_t)f * K + k] = wk;
  }
}

// (mode, concentration, weight) -> E-step form, for CWMM.predict (cwmm.py:26-52)
struct CwFromModelArgs {
  int F, D, K;
  const double2* mode; const double* concentration; const double* weight;  // weight may be null (1/K)
  double* coef; double* ld; double* ew; double* w;
};

__global__ void cw_from_model_kernel(const CwFromModelArgs u) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = u.D, K = u.K, NS = D * D;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int f = blockIdx.x;
  int* tab = reinterpret_cast<int*>(smem_raw);
  for (int s = threadIdx.x; s < NS; s += blockDim.x) tab[s] = slot_pack(D, s);
  __syncthreads();
  for (int k = warp; k < K; k += nw) {
    cw_coef_from_mode(u.mode + ((size_t)f * K + k) * D, tab, D, lane, u.coef + ((size_t)f * K + k) * NS);
    if (lane == 0) {
      const double kappa = u.concentration[(size_t)f * K + k];
      u.ew[(size_t)f * K + k] = kappa;
      u.ld[(size_t)f * K + k] = cw_log_norm(kappa, D);
      u.w[(size_t)f * K + k] = u.weight ? u.weight[(size_t)f * K + k] : 1.0 / K;
    }
  }
}

// --------------------------------------------------------------------------
// Observation normalisation, (F, T, D) -> (F, D, T) [swap] or (F, T, D).
// One thread per frame; a 32 x D tile is transposed through shared memory so
// both the read and the write are coalesced.
// --------------------------------------------------------------------------
template <typename CT>
__global__ void normalize_kernel(const CT* __restrict__ y, CT* __restrict__ z, int F, int T, int D, int swap,
                                 int zs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* tile = reinterpret_cast<double2*>(smem_raw);  // [blockDim.x][D + 1]
  const int f = blockIdx.y;
  const int t0 = blockIdx.x * blockDim.x;
  const int nt = min((int)blockDim.x, T - t0);
  const CT* __restrict__ yf = y + ((size_t)f * T + t0) * D;
  const int ldt = D + 1;
  for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
    const int tt = i / D, d = i - tt * D;
    tile[tt * ldt + d] = ld_cplx(yf + i);
  }
  __syncthreads();
  if ((int)threadIdx.x < nt) {
    double n2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 v = tile[threadIdx.x * ldt + d];
      n2 += v.x * v.x + v.y * v.y;
    }
    // np.linalg.norm, then 'where' (cacg.py:49-54) or max(norm, tiny) (complex_watson.py:26-29):
    // both leave a zero vector at zero and divide every other vector by its norm.
    double nrm = sqrt(n2);
    if (nrm == 0.0) nrm = kTiny;
    nrm = fmax(nrm, kTiny);
    for (int d = 0; d < D; ++d) {
      double2 v = tile[threadIdx.x * ldt + d];
      // the reference divides (y / norm); keep a true division for bit parity of z
      v.x = v.x / nrm; v.y = v.y / nrm;
      tile[threadIdx.x * ldt + d] = v;
    }
  }
  __syncthreads();
  if (swap) {
    for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
      const int d = i / nt, tt = i - d * nt;
      const double2 v = tile[tt * ldt + d];
      st_cplx(z + ((size_t)f * D + d) * zs + t0 + tt, v.x, v.y);
    }
    if (t0 + (int)blockDim.x >= T) {  // zero the padding [T, zs) of every row
      const int npad = zs - T;
      for (int i = threadIdx.x; i < npad * D; i += blockDim.x) {
        const int d = i / npad, tt = i - d * npad;
        st_cplx(z + ((size_t)f * D + d) * zs + T + tt, 0.0, 0.0);
      }
    }
  } else {
    CT* __restrict__ zf = z + ((size_t)f * T + t0) * D;
    for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
      const int tt = i / D, d = i - tt * D;
      const double2 v = tile[tt * ldt + d];
      st_cplx(zf + i, v.x, v.y);
    }
  }
}

// Staged layout of the persistent kernels (the channel rows of one ring stage = one contiguous block):
//   out[f][c][d][i] = z[f][d][c * SF + i]; frames >= T are zero.  The repeated rows of a stage (common.cuh) are
//   added in shared memory only (stage_g2s, em_persistent.cuh).

// Normalisation into the staged layout.  One CTA per (frame tile, bin).
template <typename CT>
__global__ void normalize_staged_kernel(const CT* __restrict__ y, CT* __restrict__ z, int F, int T, int D, int SF,
                                        int nchunks, int* __restrict__ dead) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* tile = reinterpret_cast<double2*>(smem_raw);  // [blockDim.x][D + 1]
  const int f = blockIdx.y;
  const int t0 = blockIdx.x * blockDim.x;                // blockDim.x divides SF
  const int nt = max(0, min((int)blockDim.x, T - t0));
  const int ldt = D + 1;
  const CT* __restrict__ yf = y + ((size_t)f * T + t0) * D;
  for (int i = threadIdx.x; i < nt * D; i += blockDim.x) {
    const int tt = i / D, d = i - tt * D;
    tile[tt * ldt + d] = ld_cplx(yf + i);
  }
  __syncthreads();
  if ((int)threadIdx.x < nt) {
    double n2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double2 v = tile[threadIdx.x * ldt + d];
      n2 += v.x * v.x + v.y * v.y;
    }
    double nrm = sqrt(n2);
    // bins with an all-zero frame keep the reference's eigenvalue normalisation in every
    // iteration (see em_persistent.cuh): remember them
    if (nrm == 0.0 && dead != nullptr) dead[f] = 1;
    if (nrm == 0.0) nrm = kTiny;
    nrm = fmax(nrm, kTiny);
    for (int d = 0; d < D; ++d) {
      double2 v = tile[threadIdx.x * ldt + d];
      v.x = v.x / nrm; v.y = v.y / nrm;
      tile[threadIdx.x * ldt + d] = v;
    }
  }
  __syncthreads();
  const int c = t0 / SF, i0 = t0 - c * SF;
  CT* __restrict__ zc = z + ((size_t)f * nchunks + c) * D * SF;
  for (int i = threadIdx.x; i < D * (int)blockDim.x; i += blockDim.x) {
    // consecutive threads write consecutive addresses
    const int d = i / (int)blockDim.x;
    const int tt = i - d * (int)blockDim.x;
    double2 v = make_double2(0.0, 0.0);
    if (tt < nt) v = tile[tt * ldt + d];
    st_cplx(zc + d * SF + i0 + tt, v.x, v.y);
  }
}

// Streamed upload for the persistent fit: the observation (and the initial affiliations) live
// in PINNED HOST memory and are read here directly over PCIe while the EM kernel already runs
// on the bins that have arrived.  A few CTAs take bins from a counter (ascending order; any
// resident subset of the CTAs makes progress); per bin: normalise + stage the observation exactly
// like normalize_staged_kernel, copy the bin's initial affiliations to the device, then publish
// flags[bin] = 0 (release), which is what the bin's first EM task waits for (em_persistent.cuh).
// The link latency (~2 us) is covered by software pipelining: the 16-byte loads of the NEXT
// 128-frame chunk (of this bin or the next one) are in flight in registers while the current
// chunk is normalised and written, so every CTA always has a full chunk outstanding.
constexpr int kLoadThreads = 128;
constexpr int kLoadBatch = 8;  // 16-byte loads per thread and batch: 16 KB per CTA in flight

template <typename CT>
__global__ void __launch_bounds__(kLoadThreads, 3)
stream_load_kernel(const CT* __restrict__ y, CT* __restrict__ z, const double* __restrict__ aff_src,
                   double* __restrict__ aff_dst, int F, int T, int D, int K, int SF, int nchunks,
                   int* __restrict__ dead, int* __restrict__ flags, int* __restrict__ next_bin,
                   int* __restrict__ started) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* tile = reinterpret_cast<double2*>(smem_raw);  // [SF][D + 1]
  __shared__ int s_bin[2];
  // the host holds the EM kernel's launch back until every loader CTA is resident (cuStreamWaitValue32)
  if (threadIdx.x == 0) {
    atomicAdd(started, 1);
    __threadfence();
  }
  const int ldt = D + 1;
  const int tid = threadIdx.x;
  const int per_chunk = SF * D;                                   // complex elements of a full chunk
  const int nbatch = (per_chunk + kLoadThreads * kLoadBatch - 1) / (kLoadThreads * kLoadBatch);
  // the first batch of a chunk travels in registers across the pipeline; chunks with more than
  // one batch (D > 8) load the rest synchronously
  auto load_batch = [&](int f, int c, int b, double2 (&v)[kLoadBatch]) {
    const int t0 = c * SF;
    const int n = max(0, min(SF, T - t0)) * D;
    const CT* __restrict__ yf = y + ((size_t)f * T + t0) * D;
#pragma unroll
    for (int j = 0; j < kLoadBatch; ++j) {
      const int i = (b * kLoadBatch + j) * kLoadThreads + tid;
      if (i < n) v[j] = ld_cplx(yf + i);
    }
  };
  auto store_batch = [&](int c, int b, const double2 (&v)[kLoadBatch]) {
    const int n = max(0, min(SF, T - c * SF)) * D;
#pragma unroll
    for (int j = 0; j < kLoadBatch; ++j) {
      const int i = (b * kLoadBatch + j) * kLoadThreads + tid;
      if (i < n) {
        const int tt = i / D, d = i - tt * D;
        tile[tt * ldt + d] = v[j];
      }
    }
  };
  if (tid == 0) {
    s_bin[0] = atomicAdd(next_bin, 1);
    s_bin[1] = atomicAdd(next_bin, 1);
  }
  __syncthreads();
  int f = s_bin[0], nf = s_bin[1];
  double2 v[kLoadBatch];
  if (f < F) load_batch(f, 0, 0, v);
  while (f < F) {
    bool zero_frame = false;
    for (int c = 0; c < nchunks; ++c) {
      const int t0 = c * SF;
      const int nt = max(0, min(SF, T - t0));
      store_batch(c, 0, v);
      for (int b = 1; b < nbatch; ++b) {
        double2 u[kLoadBatch];
        load_batch(f, c, b, u);
        store_batch(c, b, u);
      }
      // next chunk of this bin, or the first chunk of the next bin: in flight from here on
      if (c + 1 < nchunks) load_batch(f, c + 1, 0, v);
      else if (nf < F) load_batch(nf, 0, 0, v);
      __syncthreads();
      for (int tt = tid; tt < nt; tt += kLoadThreads) {
        double n2 = 0.0;
        for (int d = 0; d < D; ++d) {
          const double2 x = tile[tt * ldt + d];
          n2 += x.x * x.x + x.y * x.y;
        }
        double nrm = sqrt(n2);
        zero_frame |= nrm == 0.0;
        if (nrm == 0.0) nrm = kTiny;
        nrm = fmax(nrm, kTiny);
        for (int d = 0; d < D; ++d) {
          double2 x = tile[tt * ldt + d];
          x.x = x.x / nrm; x.y = x.y / nrm;
          tile[tt * ldt + d] = x;
        }
      }
      __syncthreads();
      CT* __restrict__ zc = z + ((size_t)f * nchunks + c) * D * SF;
      // (rolled loops: with the next chunk's loads in flight, an unrolled store loop spills at 168 registers)
#pragma unroll 1
      for (int d = 0; d < D; ++d) {
#pragma unroll 1
        for (int tt = tid; tt < SF; tt += kLoadThreads) {
          double2 x = make_double2(0.0, 0.0);
          if (tt < nt) x = tile[tt * ldt + d];
          st_cplx(zc + d * SF + tt, x.x, x.y);
        }
      }
      __syncthreads();
    }
    if (aff_dst != nullptr) {
      const double2* __restrict__ src = reinterpret_cast<const double2*>(aff_src + (size_t)f * K * T);
      double2* __restrict__ dst = reinterpret_cast<double2*>(aff_dst + (size_t)f * K * T);
      const int n = K * T;
      if (((reinterpret_cast<size_t>(src) | reinterpret_cast<size_t>(dst)) & 15) == 0) {  // vector copies
        for (int i0 = 0; i0 < n / 2; i0 += kLoadThreads * kLoadBatch) {
          double2 u[kLoadBatch];
#pragma unroll
          for (int j = 0; j < kLoadBatch; ++j) {
            const int i = i0 + j * kLoadThreads + tid;
            if (i < n / 2) u[j] = __ldg(src + i);
          }
#pragma unroll
          for (int j = 0; j < kLoadBatch; ++j) {
            const int i = i0 + j * kLoadThreads + tid;
            if (i < n / 2) dst[i] = u[j];
          }
        }
        if ((n & 1) && tid == 0) aff_dst[(size_t)f * K * T + n - 1] = __ldg(aff_src + (size_t)f * K * T + n - 1);
      } else {
        const double* __restrict__ s1 = aff_src + (size_t)f * K * T;
        double* __restrict__ d1 = aff_dst + (size_t)f * K * T;
        for (int i0 = 0; i0 < n; i0 += kLoadThreads * kLoadBatch) {
          double u[kLoadBatch];
#pragma unroll
          for (int j = 0; j < kLoadBatch; ++j) {
            const int i = i0 + j * kLoadThreads + tid;
            if (i < n) u[j] = __ldg(s1 + i);
          }
#pragma unroll
          for (int j = 0; j < kLoadBatch; ++j) {
            const int i = i0 + j * kLoadThreads + tid;
            if (i < n) d1[i] = u[j];
          }
        }
      }
    }
    if (zero_frame && dead != nullptr) dead[f] = 1;
    if (tid == 0) s_bin[0] = atomicAdd(next_bin, 1);  // the bin after next
    __syncthreads();  // every thread's stores of this bin are ordered before the release below
    if (tid == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flags + f), "r"(0) : "memory");
    f = nf;
    nf = s_bin[0];
    __syncthreads();  // s_bin[0] is rewritten at the end of the next bin
  }
}

}  // namespace pbb
