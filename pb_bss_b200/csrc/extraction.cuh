// Kernels of the multi-source beamformers and the vector post-processing of pb_bss/extraction/beamformer.py:
// LCMV, WMWF, MERL MVDR, the reference-channel SNR, condition_covariance, distortionless_normalization,
// mvdr_snr_postfilter, zero_degree_normalization, phase_correction and apply_online_beamforming_vector.
// The linear solves are solve_kernel (linalg_kernels.cuh); everything here is elementwise or one thread per bin.
#pragma once
#include "common.cuh"
#include "linalg_kernels.cuh"

namespace pbb {

// a / b the way NumPy divides complex numbers (Smith's algorithm, npy_math's complex division)
__device__ __forceinline__ double2 cdiv_np(double2 a, double2 b) {
  if (fabs(b.x) >= fabs(b.y)) {
    if (b.x == 0.0 && b.y == 0.0) return make_double2(a.x / fabs(b.x), a.y / fabs(b.y));
    const double rat = b.y / b.x, scl = 1.0 / (b.x + b.y * rat);
    return make_double2((a.x + a.y * rat) * scl, (a.y - a.x * rat) * scl);
  }
  const double rat = b.x / b.y, scl = 1.0 / (b.y + b.x * rat);
  return make_double2((a.x * rat + a.y) * scl, (a.y * rat - a.x) * scl);
}

// principal square root (C99 csqrt, which np.sqrt uses for complex input)
__device__ __forceinline__ double2 csqrt_principal(double2 z) {
  if (z.x == 0.0 && z.y == 0.0) return make_double2(0.0, z.y);
  const double t = sqrt(0.5 * (fabs(z.x) + hypot(z.x, z.y)));
  if (z.x >= 0.0) return make_double2(t, z.y / (2.0 * t));
  return make_double2(fabs(z.y) / (2.0 * t), copysign(t, z.y));
}

// ---- LCMV (beamformer.py:414-456) ----------------------------------------------------------------------------
// rhs of the first solve: the K ATFs as columns, atf (K, F, D) -> H (F, D, K)
__global__ void lcmv_rhs_kernel(const double2* __restrict__ atf, int K, int F, int D, double2* __restrict__ H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * F * D) return;
  const int k = i % K, d = (i / K) % D, f = i / (K * D);
  H[i] = atf[((size_t)k * F + f) * D + d];
}

// G[f][k][l] = sum_d conj(atf[k][f][d]) X[f][d][l] with X = Phi_N^-1 H (:438-442); rhs[f][k] = response[k] rounded to
// complex64 like the reference's astype(np.complex64) (:444)
__global__ void lcmv_gram_kernel(const double2* __restrict__ atf, const double2* __restrict__ X,
                                 const double2* __restrict__ response, int K, int F, int D, double2* __restrict__ G,
                                 double2* __restrict__ rhs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * K * K) return;
  const int l = i % K, k = (i / K) % K, f = i / (K * K);
  double2 s = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) {
    const double2 a = atf[((size_t)k * F + f) * D + d];
    const double2 p = cmul(make_double2(a.x, -a.y), X[((size_t)f * D + d) * K + l]);
    s.x += p.x; s.y += p.y;
  }
  G[i] = s;
  if (l == 0) {
    const double2 r = response[k];
    rhs[(size_t)f * K + k] = make_double2((double)(float)r.x, (double)(float)r.y);
  }
}

// w[f][d] = sum_k X[f][d][k] y[f][k] (:450-454).  When any bin's K x K system was singular, the reference's
// stable_solve leaves the batched solve for a per-bin loop that writes into np.zeros_like(rhs), a complex64 array
// (math/solve.py:107-113): then y of EVERY bin is rounded to complex64, which *round_y reproduces.
__global__ void lcmv_combine_kernel(const double2* __restrict__ X, const double2* __restrict__ y,
                                    const int* __restrict__ round_y, int K, int F, int D, double2* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * D) return;
  const int f = i / D;
  const bool rnd = *round_y != 0;
  double2 s = make_double2(0.0, 0.0);
  for (int k = 0; k < K; ++k) {
    double2 yk = y[(size_t)f * K + k];
    if (rnd) yk = make_double2((double)(float)yk.x, (double)(float)yk.y);
    const double2 p = cmul(X[(size_t)i * K + k], yk);
    s.x += p.x; s.y += p.y;
  }
  w[i] = s;
}

// ---- WMWF filter (beamformer.py:735-742) ---------------------------------------------------------------------
// filter = phi / (mu + trace(phi)) or, frequency_dependent, phi / sqrt(target[0][0] * trace(phi)); one thread per
// matrix entry, each sums the trace itself (D <= 64 reads of one cached row)
__global__ void wmwf_filter_kernel(const double2* __restrict__ phi, const double2* __restrict__ target, int n, int D,
                                   int frequency_dependent, double mu, double2* __restrict__ filter) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * D * D) return;
  const size_t m = i / ((size_t)D * D);
  const double2* __restrict__ ph = phi + m * D * D;
  double2 lam = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) { lam.x += ph[d * D + d].x; lam.y += ph[d * D + d].y; }
  const double2 den = frequency_dependent ? csqrt_principal(cmul(target[m * D * D], lam))
                                          : make_double2(mu + lam.x, lam.y);
  filter[i] = cdiv_np(phi[i], den);
}

// out[m][r] = sum_c filter[m][r][c] * weight[m][r][c] (channel_selection_vector, :743-745)
__global__ void weighted_channel_sum_kernel(const double2* __restrict__ filter, const double2* __restrict__ weight,
                                            int n, int D, double2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * D) return;
  double2 s = make_double2(0.0, 0.0);
  for (int c = 0; c < D; ++c) {
    const double2 p = cmul(filter[i * D + c], weight[i * D + c]);
    s.x += p.x; s.y += p.y;
  }
  out[i] = s;
}

// ---- get_optimal_reference_channel (beamformer.py:601-624): per-bin SNR terms of every column R of w_mat ----
// (the same quadratic forms as souden_kernel; colsum_kernel sums them over the bins in a fixed order)
__global__ void reference_snr_kernel(const double2* __restrict__ w, const double2* __restrict__ target,
                                     const double2* __restrict__ noise, int n, int D, double2* __restrict__ num,
                                     double2* __restrict__ den) {
  const int m = blockIdx.x;
  const int R = threadIdx.x;
  if (R >= D) return;
  const double2* __restrict__ wm = w + (size_t)m * D * D;
  double2 qt, qn;
  quad_forms([&](int d) { return wm[d * D + R]; }, target + (size_t)m * D * D, noise + (size_t)m * D * D, D, qt, qn);
  num[(size_t)m * D + R] = qt;
  den[(size_t)m * D + R] = qn;
}

// ---- MERL MVDR (beamformer.py:263-289) ----------------------------------------------------------------------
// w = (G / trace G)[:, 0] with G = N^-1 T.  The reference sums its per-channel SNR over the channel axis too
// (np.sum of a 'c'-indexed einsum), so its argmax is always 0: column 0 is what it returns.
__global__ void merl_kernel(const double2* __restrict__ G, int n, int D, double2* __restrict__ w) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  const double2* __restrict__ g = G + (size_t)m * D * D;
  double2 lam = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) { lam.x += g[d * D + d].x; lam.y += g[d * D + d].y; }
  for (int d = 0; d < D; ++d) w[(size_t)m * D + d] = cdiv_np(g[d * D], lam);
}

// ---- vector post-processing (beamformer.py:491-514, 563-569) ---------------------------------------------------
// distortionless_normalization: out = (N w w^H / (w^H N w)) a, one thread per bin
__global__ void distortionless_kernel(const double2* __restrict__ vec, const double2* __restrict__ atf,
                                      const double2* __restrict__ noise, int n, int D, double2* __restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  const double2* __restrict__ w = vec + (size_t)m * D;
  const double2* __restrict__ a = atf + (size_t)m * D;
  const double2* __restrict__ N = noise + (size_t)m * D * D;
  // den = w^H N w ; wa = w^H a (the projection is rank one: sum_c u_r conj(w_c) a_c / den)
  double2 den = make_double2(0.0, 0.0), wa = make_double2(0.0, 0.0);
  for (int r = 0; r < D; ++r) {
    double2 u = make_double2(0.0, 0.0);
    for (int c = 0; c < D; ++c) {
      const double2 p = cmul(N[r * D + c], w[c]);
      u.x += p.x; u.y += p.y;
    }
    const double2 p = cmulc(u, w[r]);  // u_r conj(w_r)
    den.x += p.x; den.y += p.y;
    const double2 q = cmulc(a[r], w[r]);
    wa.x += q.x; wa.y += q.y;
  }
  for (int r = 0; r < D; ++r) {
    double2 u = make_double2(0.0, 0.0);
    for (int c = 0; c < D; ++c) {
      const double2 p = cmul(N[r * D + c], w[c]);
      u.x += p.x; u.y += p.y;
    }
    out[(size_t)m * D + r] = cmul(cdiv_np(u, den), wa);
  }
}

// mvdr_snr_postfilter: (w^H T w) / (w^H N w), one thread per bin
__global__ void snr_postfilter_kernel(const double2* __restrict__ vec, const double2* __restrict__ target,
                                      const double2* __restrict__ noise, int n, int D, double2* __restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  const double2* __restrict__ w = vec + (size_t)m * D;
  double2 qt, qn;
  quad_forms([&](int d) { return w[d]; }, target + (size_t)m * D * D, noise + (size_t)m * D * D, D, qt, qn);
  out[m] = cdiv_np(qt, qn);
}

// zero_degree_normalization: w * exp(-i angle(w[ref])), elementwise
__global__ void zero_degree_kernel(const double2* __restrict__ vec, int n, int D, int ref, double2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * D) return;
  const double2 r = vec[(i / D) * D + ref];
  double s, c;
  sincos(atan2(r.y, r.x), &s, &c);
  out[i] = cmul(vec[i], make_double2(c, -s));
}

// condition_covariance: (x + gamma trace(x) / D I) / (1 + gamma), elementwise
__global__ void condition_covariance_kernel(const double2* __restrict__ x, int n, int D, double gamma,
                                            double2* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * D * D) return;
  const double2* __restrict__ xm = x + (i / ((size_t)D * D)) * D * D;
  const int r = (int)(i % ((size_t)D * D)) / D, c = (int)(i % D);
  double2 tr = make_double2(0.0, 0.0);
  for (int d = 0; d < D; ++d) { tr.x += xm[d * D + d].x; tr.y += xm[d * D + d].y; }
  const double e = r == c ? 1.0 : 0.0;
  const double2 v = x[i];
  const double den = 1.0 + gamma;
  out[i] = make_double2((v.x + e * (gamma * tr.x / D)) / den, (v.y + e * (gamma * tr.y / D)) / den);
}

// ---- phase_correction (beamformer.py:517-560) ------------------------------------------------------------------
// The reference multiplies bin f >= 1 by the cumulative product, along AXIS 0 OF THE WHOLE ARRAY, of
// e = exp(i angle(sum_d conj(w_f) w_{f-1})).  For a 2-D (F, D) input axis 0 is the bin axis (scan_bins = 1): one
// thread scans the F - 1 factors.  For an (A, M, F, D) input (A = the reference's axis 0, M = the dims between)
// the product runs over A for every (m, f) on its own, not over the bins: one thread per (m, f), sequential in a.
// The sequential product keeps NumPy's cumprod rounding order (p_a = p_{a-1} e_a).  sincos(atan2(.)) gives the
// factor 1 for a zero inner product, as np.angle(0) = 0 does.
__global__ void phase_correction_kernel(const double2* __restrict__ vec, int A, int M, int F, int D, int scan_bins,
                                        double2* __restrict__ out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto factor = [&](const double2* cur, const double2* prev) {
    double2 s = make_double2(0.0, 0.0);
    for (int d = 0; d < D; ++d) {
      const double2 p = cmulc(prev[d], cur[d]);  // conj(w_f[d]) w_{f-1}[d]
      s.x += p.x; s.y += p.y;
    }
    double sn, cs;
    sincos(atan2(s.y, s.x), &sn, &cs);
    return make_double2(cs, sn);
  };
  if (scan_bins) {
    if (j != 0) return;
    for (int d = 0; d < D; ++d) out[d] = vec[d];
    double2 p = make_double2(1.0, 0.0);
    for (int f = 1; f < F; ++f) {
      const double2 e = factor(vec + (size_t)f * D, vec + (size_t)(f - 1) * D);
      p = f == 1 ? e : cmul(p, e);
      for (int d = 0; d < D; ++d) out[(size_t)f * D + d] = cmul(vec[(size_t)f * D + d], p);
    }
    return;
  }
  if (j >= (long long)M * F) return;
  const int mi = (int)(j / F), f = (int)(j % F);
  double2 p = make_double2(1.0, 0.0);
  for (int a = 0; a < A; ++a) {
    const size_t row = (((size_t)a * M + mi) * F + f) * D;
    if (f == 0) {
      for (int d = 0; d < D; ++d) out[row + d] = vec[row + d];
      continue;
    }
    const double2 e = factor(vec + row, vec + row - D);
    p = a == 0 ? e : cmul(p, e);
    for (int d = 0; d < D; ++d) out[row + d] = cmul(vec[row + d], p);
  }
}

// ---- apply_online_beamforming_vector (beamformer.py:586-598) ---------------------------------------------------
// out[b][f][t] = sum_d conj(v[t][f][d]) mix[b][f][d][t].  Bandwidth-bound.  The mix is contiguous along t and the
// vector along d, so one thread per (f, t) with t across the lanes coalesces the mix (and out), and each thread
// reads its own D contiguous vector entries (D * 16 bytes: for D = 8 exactly one 128-byte line, every byte used, so
// the uncoalesced vector reads fetch nothing twice).  A shared-memory transpose of the vector tile would add a
// barrier and shared traffic without saving any DRAM bytes.  The first kOnlineRegD entries stay in registers while
// the thread loops over the B leading indices of the mix, so the vector is read once, not once per index.
// Strides (elements): sv_t / sv_f = vector frame / bin strides (sv_f = 0: one vector bin broadcast over the bins),
// smb / smf = mix batch / bin strides (0 where the mix is broadcast); the vector's d stride is 1, the mix's d and t
// strides are T and 1.
constexpr int kOnlineRegD = 8;
template <typename CT>
__global__ void apply_online_kernel(const double2* __restrict__ v, const CT* __restrict__ mix, int B, int F, int D,
                                    int T, long long sv_t, long long sv_f, long long smb, long long smf,
                                    double2* __restrict__ out) {
  const int f = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const double2* __restrict__ vt = v + (size_t)t * sv_t + (size_t)f * sv_f;
  double2 vr[kOnlineRegD];
#pragma unroll
  for (int d = 0; d < kOnlineRegD; ++d)
    if (d < D) vr[d] = __ldg(vt + d);
  for (int b = 0; b < B; ++b) {
    const CT* __restrict__ y = mix + (size_t)b * smb + (size_t)f * smf + t;
    double2 s = make_double2(0.0, 0.0);
#pragma unroll
    for (int d = 0; d < kOnlineRegD; ++d) {
      if (d < D) {
        const double2 x = ld_cplx(y + (size_t)d * T);
        s.x += vr[d].x * x.x + vr[d].y * x.y;
        s.y += vr[d].x * x.y - vr[d].y * x.x;
      }
    }
    for (int d = kOnlineRegD; d < D; ++d) {
      const double2 w = __ldg(vt + d), x = ld_cplx(y + (size_t)d * T);
      s.x += w.x * x.x + w.y * x.y;
      s.y += w.x * x.y - w.y * x.x;
    }
    out[((size_t)b * F + f) * T + t] = s;
  }
}

}  // namespace pbb
