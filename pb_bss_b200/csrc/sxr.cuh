// SI-SDR, the invasive SxR and the mean square of pb_bss/evaluation/module_si_sdr.py and sxr_module.py
// (include/pbb.h, pbb_mean_square / pbb_si_sdr / pbb_input_sxr / pbb_output_sxr).
//
// fp64, no float atomics.  A row of n samples is cut into ceil(n / kSxrChunk) chunks; one CTA sums a chunk in a
// fixed order (each thread a strided sequence, then the warp butterfly, then the warps in order), and one CTA per
// row sums the chunk partials the same way.  The tree depends on n only, so a row's bits do not depend on its batch.
// Products and differences are rounded as NumPy rounds them (no FMA contraction); only the order of the length-n sums
// differs from NumPy's pairwise sum.  The ratio kernels work on at most 9 x 29 powers and follow the reference's order
// of operations exactly, with np.sum's summation order (np_sum below).
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kSxrThreads = 256;
constexpr long long kSxrChunk = 8192;  // samples per chunk partial
constexpr int kSxrPermCtas = 1024;     // CTAs of the permutation search (at most)

__host__ __device__ inline long long sxr_chunks(long long n) { return (n + kSxrChunk - 1) / kSxrChunk; }

__device__ __forceinline__ double sq_rn(double v) { return __dmul_rn(v, v); }

template <class T> struct SqLoad;
template <> struct SqLoad<float> { static __device__ double f(const float* p) { return sq_rn((double)__ldg(p)); } };
template <> struct SqLoad<double> { static __device__ double f(const double* p) { return sq_rn(__ldg(p)); } };
template <> struct SqLoad<short> { static __device__ double f(const short* p) { return sq_rn((double)__ldg(p)); } };
template <> struct SqLoad<int> { static __device__ double f(const int* p) { return sq_rn((double)__ldg(p)); } };
template <> struct SqLoad<long long> {
  static __device__ double f(const long long* p) { return sq_rn((double)__ldg(p)); }
};
template <> struct SqLoad<float2> {
  static __device__ double f(const float2* p) {
    const float2 v = __ldg(p);
    return abs2_rn(make_double2((double)v.x, (double)v.y));
  }
};
template <> struct SqLoad<double2> { static __device__ double f(const double2* p) { return abs2_rn(__ldg(p)); } };

// Sum of N values per thread over the CTA in a fixed order; the totals are valid in thread 0.
template <int N>
__device__ __forceinline__ void cta_sum(double (&v)[N]) {
  __shared__ double sh[N][kSxrThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < N; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] = __dadd_rn(v[j], __shfl_xor_sync(0xffffffffu, v[j], o));
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < N; ++j) sh[j][warp] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int j = 0; j < N; ++j) {
      double s = sh[j][0];
      for (int w = 1; w < kSxrThreads / 32; ++w) s = __dadd_rn(s, sh[j][w]);
      v[j] = s;
    }
}

// One chunk of |x|^2 per CTA: partial[blockIdx.x], blockIdx.x = row * chunks + chunk.
template <class T>
__global__ void __launch_bounds__(kSxrThreads) mean_square_chunk_kernel(const T* __restrict__ x, long long n,
                                                                        long long chunks, double* __restrict__ partial) {
  const long long row = blockIdx.x / chunks, c = blockIdx.x % chunks;
  const T* xr = x + row * n;
  const long long end = min(n, (c + 1) * kSxrChunk);
  double v[1] = {0.0};
#pragma unroll 4
  for (long long i = c * kSxrChunk + threadIdx.x; i < end; i += kSxrThreads) v[0] = __dadd_rn(v[0], SqLoad<T>::f(xr + i));
  cta_sum<1>(v);
  if (threadIdx.x == 0) partial[blockIdx.x] = v[0];
}

// Per row (one CTA): the N sums of its `chunks` partials (partial[(row * chunks + c) * N + j]).
template <int N>
__device__ __forceinline__ void row_totals(const double* __restrict__ partial, long long chunks, double (&v)[N]) {
  const double* p = partial + (size_t)blockIdx.x * chunks * N;
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = 0.0;
  for (long long c = threadIdx.x; c < chunks; c += kSxrThreads)
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = __dadd_rn(v[j], p[c * N + j]);
  cta_sum<N>(v);
}

__global__ void __launch_bounds__(kSxrThreads) mean_square_row_kernel(const double* __restrict__ partial, long long n,
                                                                      long long chunks, double* __restrict__ out) {
  double v[1];
  row_totals<1>(partial, chunks, v);
  if (threadIdx.x == 0) out[blockIdx.x] = __ddiv_rn(v[0], (double)n);  // n = 0: 0 / 0 = NaN, as np.mean
}

// SI-SDR pass 1: <r, r> and <r, e> of one chunk.  r and e are read at their row offsets (broadcast operands).
__global__ void __launch_bounds__(kSxrThreads) si_sdr_pass1_kernel(const double* __restrict__ r,
                                                                   const double* __restrict__ e,
                                                                   const long long* __restrict__ roff,
                                                                   const long long* __restrict__ eoff, long long n,
                                                                   long long chunks, double* __restrict__ partial) {
  const long long row = blockIdx.x / chunks, c = blockIdx.x % chunks;
  const double* rr = r + roff[row];
  const double* er = e + eoff[row];
  const long long end = min(n, (c + 1) * kSxrChunk);
  double v[2] = {0.0, 0.0};
#pragma unroll 4
  for (long long i = c * kSxrChunk + threadIdx.x; i < end; i += kSxrThreads) {
    const double a = __ldg(rr + i), b = __ldg(er + i);
    v[0] = __dadd_rn(v[0], __dmul_rn(a, a));
    v[1] = __dadd_rn(v[1], __dmul_rn(a, b));
  }
  cta_sum<2>(v);
  if (threadIdx.x == 0) {
    partial[2 * (size_t)blockIdx.x] = v[0];
    partial[2 * (size_t)blockIdx.x + 1] = v[1];
  }
}

// alpha = <r, e> / <r, r> per row (one CTA per row).
__global__ void __launch_bounds__(kSxrThreads) si_sdr_alpha_kernel(const double* __restrict__ partial,
                                                                   long long chunks, double* __restrict__ alpha) {
  double v[2];
  row_totals<2>(partial, chunks, v);
  if (threadIdx.x == 0) alpha[blockIdx.x] = __ddiv_rn(v[1], v[0]);
}

// SI-SDR pass 2: sum (alpha r)^2 and sum (e - alpha r)^2 of one chunk, from the rounded projection and residual.
__global__ void __launch_bounds__(kSxrThreads) si_sdr_pass2_kernel(const double* __restrict__ r,
                                                                   const double* __restrict__ e,
                                                                   const long long* __restrict__ roff,
                                                                   const long long* __restrict__ eoff, long long n,
                                                                   long long chunks, const double* __restrict__ alpha,
                                                                   double* __restrict__ partial) {
  const long long row = blockIdx.x / chunks, c = blockIdx.x % chunks;
  const double* rr = r + roff[row];
  const double* er = e + eoff[row];
  const double a = alpha[row];
  const long long end = min(n, (c + 1) * kSxrChunk);
  double v[2] = {0.0, 0.0};
#pragma unroll 4
  for (long long i = c * kSxrChunk + threadIdx.x; i < end; i += kSxrThreads) {
    const double p = __dmul_rn(a, __ldg(rr + i));
    const double q = __dsub_rn(__ldg(er + i), p);
    v[0] = __dadd_rn(v[0], __dmul_rn(p, p));
    v[1] = __dadd_rn(v[1], __dmul_rn(q, q));
  }
  cta_sum<2>(v);
  if (threadIdx.x == 0) {
    partial[2 * (size_t)blockIdx.x] = v[0];
    partial[2 * (size_t)blockIdx.x + 1] = v[1];
  }
}

__device__ __forceinline__ double db10(double ratio) { return __dmul_rn(10.0, log10(ratio)); }

// 10 log10(sum (alpha r)^2 / sum (e - alpha r)^2) per row (one CTA per row).
__global__ void __launch_bounds__(kSxrThreads) si_sdr_ratio_kernel(const double* __restrict__ partial,
                                                                   long long chunks, double* __restrict__ out) {
  double v[2];
  row_totals<2>(partial, chunks, v);
  if (threadIdx.x == 0) out[blockIdx.x] = db10(__ddiv_rn(v[0], v[1]));
}

// ---- SI-SDR backward (pbb_si_sdr_backward) ----
// With p = alpha r, q = e - p (rounded as pass 2 forms them), P = sum p^2 and Q = sum q^2 of a row and c = 20 / ln 10:
// ds/de = c (p / P - q / Q), ds/dr = c alpha (1 / P + 1 / Q) q.  Per row (one CTA): P, Q from the pass-2 partials,
// then coef = (c g / P, c g / Q) for the incoming gradient g of the row.
__global__ void __launch_bounds__(kSxrThreads) si_sdr_backward_row_kernel(const double* __restrict__ partial,
                                                                          long long chunks,
                                                                          const double* __restrict__ grad_out,
                                                                          double* __restrict__ coef) {
  double v[2];
  row_totals<2>(partial, chunks, v);
  if (threadIdx.x == 0) {
    const double cg = 20.0 / log(10.0) * grad_out[blockIdx.x];
    coef[2 * (size_t)blockIdx.x] = cg / v[0];
    coef[2 * (size_t)blockIdx.x + 1] = cg / v[1];
  }
}

// The gradient wrt one operand, one thread per element of its own (unbroadcast) rows: element (u, i) sums the rows
// index[start[u]] .. index[start[u + 1] - 1] that read own row u, in that order.  WRT_E: estimation, else reference.
template <bool WRT_E>
__global__ void __launch_bounds__(kSxrThreads) si_sdr_backward_kernel(
    const double* __restrict__ r, const double* __restrict__ e, const long long* __restrict__ roff,
    const long long* __restrict__ eoff, long long n, const double* __restrict__ alpha, const double* __restrict__ coef,
    long long own_rows, const long long* __restrict__ start, const long long* __restrict__ index,
    double* __restrict__ out) {
  const long long total = own_rows * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long u = idx / n, i = idx - u * n;
    double s = 0.0;
    for (long long j = start[u]; j < start[u + 1]; ++j) {
      const long long row = index[j];
      const double a = alpha[row], cp = coef[2 * row], cq = coef[2 * row + 1];
      const double p = __dmul_rn(a, __ldg(r + roff[row] + i));
      const double q = __dsub_rn(__ldg(e + eoff[row] + i), p);
      s += WRT_E ? cp * p - cq * q : a * (cp + cq) * q;
    }
    out[idx] = s;
  }
}

// np.sum of n values get(0) .. get(n - 1) (n <= 128 here): a left-to-right loop below 8 values, else NumPy's pairwise
// block of 8 accumulators, their fixed combination, then the remainder in order.
template <class F>
__device__ double np_sum(int n, F get) {
  if (n < 8) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, get(i));
    return s;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = get(j);
  int i = 8;
  for (; i < n - n % 8; i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], get(i + j));
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __dadd_rn(s, get(i));
  return s;
}

// _sxr: 10 log10(S / X), with IEEE inf / nan for zero powers
__device__ __forceinline__ double sxr_db(double s, double x) { return db10(__ddiv_rn(s, x)); }

// input_sxr (sxr_module.py:94-165) on S (K, D) and N (D), one thread.  The outputs have the reference's shapes:
// (K, D), (K), (D) or a scalar, depending on the averages.
__global__ void input_sxr_kernel(const double* __restrict__ S, const double* __restrict__ N, int K, int D,
                                 int average_sources, int average_channels, double* __restrict__ sdr,
                                 double* __restrict__ sir, double* __restrict__ snr) {
  __shared__ double I[PBB_SXR_MAX_K * PBB_SXR_MAX_D];
  __shared__ double res[3][PBB_SXR_MAX_K * PBB_SXR_MAX_D];
  __shared__ double Sm[PBB_SXR_MAX_K], Im[PBB_SXR_MAX_K];
  if (threadIdx.x != 0) return;
  for (int d = 0; d < D; ++d)
    for (int k = 0; k < K; ++k)  // np.sum(S[[n for n in range(K) if n != k], d])
      I[k * D + d] = np_sum(K - 1, [&](int i) { return S[(i < k ? i : i + 1) * D + d]; });
  int cols;  // the last axis of SDR / SIR / SNR before the source average
  if (average_channels) {
    for (int k = 0; k < K; ++k) {
      Sm[k] = __ddiv_rn(np_sum(D, [&](int d) { return S[k * D + d]; }), (double)D);
      Im[k] = __ddiv_rn(np_sum(D, [&](int d) { return I[k * D + d]; }), (double)D);
    }
    const double Nm = __ddiv_rn(np_sum(D, [&](int d) { return N[d]; }), (double)D);
    for (int k = 0; k < K; ++k) {
      res[0][k] = sxr_db(Sm[k], __dadd_rn(Im[k], Nm));
      res[1][k] = sxr_db(Sm[k], Im[k]);
      res[2][k] = sxr_db(Sm[k], Nm);
    }
    cols = 1;
  } else {
    for (int k = 0; k < K; ++k)
      for (int d = 0; d < D; ++d) {
        const int i = k * D + d;
        res[0][i] = sxr_db(S[i], __dadd_rn(I[i], N[d]));
        res[1][i] = sxr_db(S[i], I[i]);
        res[2][i] = sxr_db(S[i], N[d]);
      }
    cols = D;
  }
  double* out[3] = {sdr, sir, snr};
  for (int m = 0; m < 3; ++m) {
    const double* v = res[m];
    if (!average_sources) {
      for (int i = 0; i < K * cols; ++i) out[m][i] = v[i];
    } else if (cols == 1) {  // np.mean of a 1-D array: the pairwise sum
      out[m][0] = __ddiv_rn(np_sum(K, [&](int k) { return v[k]; }), (double)K);
    } else {  // np.mean(axis=0) of (K, D), D > 1: the rows added in order
      for (int d = 0; d < cols; ++d) {
        double s = 0.0;
        for (int k = 0; k < K; ++k) s = __dadd_rn(s, v[k * cols + d]);
        out[m][d] = __ddiv_rn(s, (double)K);
      }
    }
  }
}

// number of k-permutations of n
__host__ __device__ inline long long sxr_perm_count(int n, int k) {
  long long p = 1;
  for (int i = 0; i < k; ++i) p *= n - i;
  return p;
}

// The p-th tuple of itertools.permutations(range(Kt), Ks) (lexicographic order), packed 4 bits per position.
__device__ __forceinline__ unsigned long long sxr_unrank(long long p, int Ks, int Kt) {
  unsigned used = 0;
  unsigned long long sel = 0;
  for (int i = 0; i < Ks; ++i) {
    const long long block = sxr_perm_count(Kt - i - 1, Ks - i - 1);
    int digit = (int)(p / block);
    p -= digit * block;
    int t = 0;
    for (;; ++t)
      if (!(used >> t & 1u) && digit-- == 0) break;
    used |= 1u << t;
    sel |= (unsigned long long)t << (4 * i);
  }
  return sel;
}
__device__ __forceinline__ int sxr_sel(unsigned long long sel, int k) { return (int)(sel >> (4 * k) & 15u); }

// np.argmax's order: a NaN beats everything but an earlier NaN, else the larger value, then the smaller index
__device__ __forceinline__ bool sxr_better(double a, long long ia, double b, long long ib) {
  const bool na = isnan(a), nb = isnan(b);
  if (na != nb) return na;
  if (!na && a != b) return a > b;
  return ia < ib;
}

__device__ __forceinline__ void cta_argmax(double& v, long long& idx) {
  __shared__ double sv[kSxrThreads / 32];
  __shared__ long long si[kSxrThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (sxr_better(ov, oi, v, idx)) { v = ov; idx = oi; }
  }
  if (lane == 0) { sv[warp] = v; si[warp] = idx; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 0; w < kSxrThreads / 32; ++w)
      if (sxr_better(sv[w], si[w], v, idx)) { v = sv[w]; idx = si[w]; }
}

// The mutual power np.sum([S[k, sel[k]] for k]) of every selection; per CTA the first maximiser (best, best_idx).
__global__ void __launch_bounds__(kSxrThreads) output_sxr_search_kernel(const double* __restrict__ S, int Ks, int Kt,
                                                                        long long P, double* __restrict__ best,
                                                                        long long* __restrict__ best_idx) {
  double v = 0.0;
  long long idx = P;  // no candidate yet: loses every comparison with an index < P
  for (long long p = (long long)blockIdx.x * kSxrThreads + threadIdx.x; p < P; p += (long long)gridDim.x * kSxrThreads) {
    const unsigned long long sel = sxr_unrank(p, Ks, Kt);
    const double m = np_sum(Ks, [&](int k) { return S[k * Kt + sxr_sel(sel, k)]; });
    if (idx == P || sxr_better(m, p, v, idx)) { v = m; idx = p; }
  }
  if (idx == P) v = -INFINITY;  // idle threads: ordered after every real candidate by their index
  cta_argmax(v, idx);
  if (threadIdx.x == 0) {
    best[blockIdx.x] = v;
    best_idx[blockIdx.x] = idx;
  }
}

// output_sxr (sxr_module.py:168-274) after the search, one thread: the selection and SDR / SIR / SNR (Ks) or their
// means.
__global__ void output_sxr_kernel(const double* __restrict__ S, const double* __restrict__ N, int Ks, int Kt,
                                  const double* __restrict__ best, const long long* __restrict__ best_idx, int ctas,
                                  int average_sources, double* __restrict__ sdr, double* __restrict__ sir,
                                  double* __restrict__ snr, long long* __restrict__ selection) {
  __shared__ double res[3][PBB_SXR_MAX_K];
  if (threadIdx.x != 0) return;
  double v = best[0];
  long long idx = best_idx[0];
  for (int c = 1; c < ctas; ++c)
    if (sxr_better(best[c], best_idx[c], v, idx)) { v = best[c]; idx = best_idx[c]; }
  const unsigned long long sel = sxr_unrank(idx, Ks, Kt);
  for (int k = 0; k < Ks; ++k) {
    const int t = sxr_sel(sel, k);
    const double SS = S[k * Kt + t];
    // np.sum(np.delete(S[:, t], k))
    const double II = np_sum(Ks - 1, [&](int i) { return S[(i < k ? i : i + 1) * Kt + t]; });
    const double NN = N[t];
    res[0][k] = sxr_db(SS, __dadd_rn(II, NN));
    res[1][k] = sxr_db(SS, II);
    res[2][k] = sxr_db(SS, NN);
    selection[k] = t;
  }
  double* out[3] = {sdr, sir, snr};
  for (int m = 0; m < 3; ++m) {
    if (average_sources)
      out[m][0] = __ddiv_rn(np_sum(Ks, [&](int k) { return res[m][k]; }), (double)Ks);
    else
      for (int k = 0; k < Ks; ++k) out[m][k] = res[m][k];
  }
}

}  // namespace pbb
