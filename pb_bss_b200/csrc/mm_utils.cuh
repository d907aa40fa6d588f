// Kernels of the building blocks of pb_bss.distribution.mixture_model_utils / utils, pb_bss.utils and
// pb_bss.evaluation.sxr_module (include/pbb.h, csrc/api_mm_utils.cu).  Every operand is read through its own strides
// (pbb_nd_layout), the arithmetic is fp64 and each result is rounded once to its storage type.  All sums run in a
// fixed order, so a result does not change from call to call.
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kNdThreads = 256;
constexpr int kAffRegK = 8;  // classes held in registers by the affiliation kernel; larger K re-reads the column

// offsets of operands 0 .. NOPS-1 at the flat row-major index i of the layout
template <int NOPS>
__device__ __forceinline__ void nd_offsets(const pbb_nd_layout& L, long long i, long long (&off)[NOPS]) {
#pragma unroll
  for (int o = 0; o < NOPS; ++o) off[o] = 0;
  for (int d = L.nd - 1; d >= 0; --d) {
    const long long n = L.shape[d];
    const long long c = d == 0 ? i : i % n;  // i < shape[0] remains for the outermost dim: no division
    i /= d == 0 ? 1 : n;
#pragma unroll
    for (int o = 0; o < NOPS; ++o) off[o] += c * L.stride[o][d];
  }
}

// np.maximum: NaN propagates (fmax drops it)
__device__ __forceinline__ double nan_max(double a, double b) { return isnan(a) ? a : fmax(a, b); }

// ---- log_pdf_to_affiliation (mixture_model_utils.py:7-55), one thread per column, any K ----
template <class T>
__device__ __forceinline__ double aff_term(const T* lp, const double* w, const uint8_t* m, const long long (&off)[4],
                                           const long long* cs, int k, double mx) {
  double a = exp((double)lp[off[0] + k * cs[0]] - mx);
  if (w) a *= w[off[1] + k * cs[1]];
  if (m && !m[off[2] + k * cs[2]]) a *= 0.0;  // a * False, so inf * 0 gives NaN as in NumPy
  return a;
}

template <class T>
__global__ void __launch_bounds__(kNdThreads) affiliation_nd_kernel(const T* __restrict__ lp,
                                                                    const double* __restrict__ w,
                                                                    const uint8_t* __restrict__ m, pbb_nd_layout L,
                                                                    long long cols, int K, long long cs0,
                                                                    long long cs1, long long cs2, long long cs3,
                                                                    double tiny, double eps, T* __restrict__ out) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const long long cs[4] = {cs0, cs1, cs2, cs3};
  long long off[4];
  nd_offsets<4>(L, c, off);
  double mx = -INFINITY;  // np.amax: a NaN wins
  for (int k = 0; k < K; ++k) {
    const double v = (double)lp[off[0] + k * cs[0]];
    if (v > mx || isnan(v)) mx = isnan(mx) ? mx : v;
  }
  if (K <= kAffRegK) {
    double a[kAffRegK], s = 0.0;
#pragma unroll
    for (int k = 0; k < kAffRegK; ++k)
      if (k < K) { a[k] = aff_term(lp, w, m, off, cs, k, mx); s += a[k]; }
    s = nan_max(s, tiny);
#pragma unroll
    for (int k = 0; k < kAffRegK; ++k)
      if (k < K) {
        double v = a[k] / s;
        if (eps != 0.0 && !isnan(v)) v = fmin(fmax(v, eps), 1.0 - eps);
        out[off[3] + k * cs[3]] = (T)v;
      }
    return;
  }
  double s = 0.0;
  for (int k = 0; k < K; ++k) s += aff_term(lp, w, m, off, cs, k, mx);
  s = nan_max(s, tiny);
  for (int k = 0; k < K; ++k) {
    double v = aff_term(lp, w, m, off, cs, k, mx) / s;
    if (eps != 0.0 && !isnan(v)) v = fmin(fmax(v, eps), 1.0 - eps);
    out[off[3] + k * cs[3]] = (T)v;
  }
}

// ---- reductions over a set of axes (np.sum / np.mean, vector norms) ----
// The reduced index space [0, n) of every output is cut into chunks of red_chunk_len(outs, n) elements, sized so that
// the whole reduction gives about kRedWarps warps (one chunk when there are that many outputs already); a warp
// reduces one (output, chunk) -- lane l takes l, l + 32, ... of the chunk in order, then a fixed butterfly --
// or, for fewer than 32 elements, one thread its whole range in order.  With more than one chunk the partials are
// combined in chunk order by red_finish_kernel.  The partition depends on the shapes only, so results repeat bit
// for bit, and a long reduction with few outputs still spreads over the whole GPU.
constexpr long long kRedWarps = 16384;  // about 2 waves of 64 warps on each of the 132 SMs
constexpr long long kRedMinChunk = 256;

__host__ __device__ inline long long red_chunk_len(long long outs, long long n) {
  long long len = (outs * n + kRedWarps - 1) / kRedWarps;
  len = (len < kRedMinChunk ? kRedMinChunk : len + 31) / 32 * 32;
  return len >= n ? (n > 0 ? n : 1) : len;
}

enum RedTerm { kTermValue = 0, kTermSquare = 1, kTermAbs = 2, kTermNonzero = 3, kTermPow = 4, kTermMax = 5, kTermMin = 6 };
enum RedPost { kPostDivide = 0, kPostNorm = 1 };

struct RedOp {
  int term;        // RedTerm
  int post;        // RedPost
  double p;        // kTermPow: the norm order
  double divisor;  // kPostDivide
  double eps;      // kPostNorm: eps_style 0 plus, 1 max, 2 where
  int eps_style;
};

__device__ __forceinline__ double red_identity(int term) {
  return term == kTermMin ? INFINITY : 0.0;
}
// max / min: a NaN wins, as in np.max
__device__ __forceinline__ double red_combine(int term, double a, double b) {
  if (term == kTermMax || term == kTermMin) {
    if (isnan(a)) return a;
    if (isnan(b)) return b;
    return term == kTermMax ? fmax(a, b) : fmin(a, b);
  }
  return a + b;
}

template <class T, bool CPLX>
__device__ __forceinline__ double red_term(const T* __restrict__ x, const double* __restrict__ mul, long long ox,
                                           long long om, const RedOp& op) {
  const double re = (double)x[CPLX ? 2 * ox : ox];
  const double im = CPLX ? (double)x[2 * ox + 1] : 0.0;
  switch (op.term) {
    case kTermValue: return mul ? __dmul_rn(re, mul[om]) : re;
    case kTermSquare: return CPLX ? __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)) : __dmul_rn(re, re);
    case kTermNonzero: return (re != 0.0 || im != 0.0) ? 1.0 : 0.0;
    default: {
      const double a = CPLX ? hypot(re, im) : fabs(re);
      return op.term == kTermPow ? pow(a, op.p) : a;
    }
  }
}

// the value an output gets from its combined reduction
template <class TO>
__device__ __forceinline__ TO red_post(double s, const RedOp& op) {
  if (op.post == kPostDivide) return (TO)(s / op.divisor);
  double nrm = op.term == kTermSquare ? sqrt(s) : op.term == kTermPow ? pow(s, 1.0 / op.p) : s;
  if (op.eps_style == 0) nrm = nrm + op.eps;
  else if (op.eps_style == 1) nrm = nan_max(nrm, op.eps);
  else if (nrm == 0.0) nrm = op.eps;
  return (TO)nrm;
}

// offsets, in 32-bit arithmetic while the index fits (a 64-bit division costs several times as much)
template <int NOPS>
__device__ __forceinline__ void nd_offsets_fast(const pbb_nd_layout& L, long long i, long long (&off)[NOPS]) {
  if (i > 0x7fffffffll) {
    nd_offsets<NOPS>(L, i, off);
    return;
  }
  unsigned u = (unsigned)i;
#pragma unroll
  for (int o = 0; o < NOPS; ++o) off[o] = 0;
  for (int d = L.nd - 1; d >= 0; --d) {
    const long long nl = L.shape[d];  // a dim of 2^31 or more leaves u (< 2^31) as it is, as 2^31 does
    const unsigned n = nl > 0x7fffffffll ? 0x80000000u : (unsigned)nl;
    const unsigned c = d == 0 ? u : u % n;
    u = d == 0 ? 0u : u / n;
#pragma unroll
    for (int o = 0; o < NOPS; ++o) off[o] += (long long)c * L.stride[o][d];
  }
}

// out (operand 2 of O) or partial[o * chunks + c]
template <class T, bool CPLX, class TO, bool WARP>
__global__ void __launch_bounds__(kNdThreads) reduce_kernel(const T* __restrict__ x, const double* __restrict__ mul,
                                                            pbb_nd_layout O, pbb_nd_layout R, long long outs,
                                                            long long n, long long chunk_len, long long chunks,
                                                            RedOp op,
                                                            double* __restrict__ partial, TO* __restrict__ out) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long g = WARP ? gid >> 5 : gid;
  const int lane = WARP ? (int)(threadIdx.x & 31) : 0;
  if (g >= outs * chunks) return;  // a whole warp leaves together in the WARP form
  const long long o = g / chunks, c = g - o * chunks;
  long long oo[3];
  nd_offsets<3>(O, o, oo);
  const long long r0 = c * chunk_len, r1 = min(n, r0 + chunk_len);
  double s = red_identity(op.term);
  for (long long r = r0 + lane; r < r1; r += (WARP ? 32 : 1)) {
    long long ro[2];
    nd_offsets_fast<2>(R, r, ro);
    s = red_combine(op.term, s, red_term<T, CPLX>(x, mul, oo[0] + ro[0], oo[1] + ro[1], op));
  }
  if (WARP) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s = red_combine(op.term, s, __shfl_xor_sync(0xffffffffu, s, d));
    if (lane) return;
  }
  if (chunks == 1) out[oo[2]] = red_post<TO>(s, op);
  else partial[g] = s;
}

// one warp per output: the partials of its chunks, lane-strided in chunk order, then the fixed butterfly
template <class TO>
__global__ void __launch_bounds__(kNdThreads) red_finish_kernel(const double* __restrict__ partial, pbb_nd_layout O,
                                                                long long outs, long long chunks, RedOp op,
                                                                TO* __restrict__ out) {
  const long long o = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = (int)(threadIdx.x & 31);
  if (o >= outs) return;
  double s = red_identity(op.term);
  for (long long c = lane; c < chunks; c += 32) s = red_combine(op.term, s, partial[o * chunks + c]);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s = red_combine(op.term, s, __shfl_xor_sync(0xffffffffu, s, d));
  if (lane) return;
  long long oo[3];
  nd_offsets<3>(O, o, oo);
  out[oo[2]] = red_post<TO>(s, op);
}

// ---- force_hermitian (distribution/utils.py:318-330): one thread per entry ----
template <class T, bool CPLX>
__global__ void __launch_bounds__(kNdThreads) force_hermitian_kernel(const T* __restrict__ a, long long total, int D,
                                                                     T* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long mat = i / ((long long)D * D);
  const int r = (int)((i / D) % D), c = (int)(i % D);
  const long long j = mat * D * D + (long long)c * D + r;  // the transposed entry
  if (CPLX) {
    out[2 * i] = (T)(((double)a[2 * i] + (double)a[2 * j]) / 2.0);
    out[2 * i + 1] = (T)(((double)a[2 * i + 1] - (double)a[2 * j + 1]) / 2.0);
  } else {
    out[i] = (T)(((double)a[i] + (double)a[j]) / 2.0);
  }
}

// ---- abs_square (utils.py:314-336), in the precision of the input ----
template <class T, bool CPLX>
__global__ void __launch_bounds__(kNdThreads) abs_square_kernel(const T* __restrict__ x, long long n,
                                                                T* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if constexpr (CPLX) {
    const T re = x[2 * i], im = x[2 * i + 1];
    if constexpr (sizeof(T) == 4) out[i] = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
    else out[i] = __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im));
  } else {
    out[i] = x[i] * x[i];
  }
}

struct alignas(16) Bytes16 {
  unsigned long long lo, hi;
};

// ---- labels_to_one_hot (utils.py:234-311): one thread per output element, final layout ----
template <class E>
__global__ void __launch_bounds__(kNdThreads) one_hot_kernel(const long long* __restrict__ labels, long long outer,
                                                             long long inner, int C, E one, E* __restrict__ out,
                                                             int* __restrict__ status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= outer * C * inner) return;
  const long long in = i % inner, o = i / ((long long)C * inner);
  const int c = (int)((i / inner) % C);
  const long long li = o * inner + in;
  long long l = labels[li];
  if (l < -(long long)C || l >= C) {
    if (c == 0) {  // keep the smallest 1 + index; 0 = no error yet
      const int v = (int)min(li + 1, (long long)0x7fffffff);
      int old = *status;
      while (old == 0 || old > v) {
        const int seen = atomicCAS(status, old, v);
        if (seen == old) break;
        old = seen;
      }
    }
    l = -1 - (long long)C;  // matches no category
  } else if (l < 0) {
    l += C;
  }
  out[i] = l == c ? one : E{};
}

// ---- N *= factor of set_snr (sxr_module.py:72-78); x / norm of _unit_norm (DIVIDE) ----
template <class T, bool CPLX, bool DIVIDE>
__global__ void __launch_bounds__(kNdThreads) scale_nd_kernel(const T* x, const double* __restrict__ f,
                                                              pbb_nd_layout L, long long total, T* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long off[3];
  nd_offsets_fast<3>(L, i, off);
  const double s = f[off[1]];
  if (CPLX) {
    const double re = (double)x[2 * off[0]], im = (double)x[2 * off[0] + 1];
    out[2 * off[2]] = (T)(DIVIDE ? re / s : re * s);
    out[2 * off[2] + 1] = (T)(DIVIDE ? im / s : im * s);
  } else {
    const double v = (double)x[off[0]];
    out[off[2]] = (T)(DIVIDE ? v / s : v * s);
  }
}

}  // namespace pbb
