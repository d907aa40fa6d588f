// Oracle masks (pb_bss/extraction/mask_module.py) and array geometry (beamform_utils.py): kernels of api_mask.cu.
//
// Every mask kernel reads the signal in its own layout through a pbb_mask_layout (include/pbb.h): an index is
// decomposed row-major over the layout's shape and each coordinate adds its input and output stride.  Nothing is
// transposed or made contiguous on the way in.
//
// lorenz_mask and quantile_mask are per-row selections.  Both run as a radix select over the bit patterns of
// non-negative doubles (which order like the values): 8 digits of 8 bits, most significant first.  Each digit
// histograms the elements that still match the selected prefix, and one warp picks the bucket that holds the answer:
//   rank    (quantile)  the bucket holding the r-th largest element (r counted from the top, descending);
//   Lorenz  the lowest bucket whose largest element still has cumsum / sum < fraction, where the cumsum at that
//           element is (sum of everything above the bucket) + its own value.  The cumsum of non-negative values is
//           non-decreasing, so the qualifying elements form a prefix of the descending order and the threshold is
//           its last element; after the last digit the prefix is that element's value.
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kSelBuckets = 256;
constexpr int kSelPasses = 8;
constexpr int kSelWarps = 8;                 // warps of a short-row CTA, one row at a time per warp
constexpr int kSelTileValues = 8192;         // values of a short-row tile (64 KB)
constexpr int kSelHistBytes = kSelBuckets * (4 + 8 + 8);

// ---- element access ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double2 ld_elem(const double2* p, long long o) { return __ldg(p + o); }
__device__ __forceinline__ double2 ld_elem(const float2* p, long long o) {
  const float2 v = __ldg(p + o);
  return make_double2((double)v.x, (double)v.y);
}
__device__ __forceinline__ double2 ld_elem(const double* p, long long o) { return make_double2(__ldg(p + o), 0.0); }
__device__ __forceinline__ double2 ld_elem(const float* p, long long o) {
  return make_double2((double)__ldg(p + o), 0.0);
}
template <class T> struct IsComplex { static constexpr bool value = false; };
template <> struct IsComplex<double2> { static constexpr bool value = true; };
template <> struct IsComplex<float2> { static constexpr bool value = true; };

__device__ __forceinline__ void st_elem(double* p, double2 v) { *p = v.x; }
__device__ __forceinline__ void st_elem(float* p, double2 v) { *p = (float)v.x; }
__device__ __forceinline__ void st_elem(double2* p, double2 v) { *p = v; }
__device__ __forceinline__ void st_elem(float2* p, double2 v) { *p = make_float2((float)v.x, (float)v.y); }

// sqrt(a^2 + b^2) for a >= b > 0 with 2^e <= a < 2^(e+1), -1022 <= e <= 1000
__device__ __forceinline__ double abs_rn_scaled(double a, double b, int e) {
  // scale by 2^-e so that a lies in [1, 2): exact, and b >= 2^-1022 or it is negligible
  const double down = __longlong_as_double((long long)(1023 - e) << 52), up = __longlong_as_double((long long)(1023 + e) << 52);
  a = __dmul_rn(a, down);
  b = __dmul_rn(b, down);
  const double a2 = __dmul_rn(a, a), a2l = fma(a, a, -a2);
  const double b2 = __dmul_rn(b, b), b2l = fma(b, b, -b2);
  const double s = __dadd_rn(a2, b2);
  const double sl = __dadd_rn(__dadd_rn(__dsub_rn(a2, s), b2), __dadd_rn(a2l, b2l));
  double h = __dsqrt_rn(s);
  const double r = __dadd_rn(fma(-h, h, s), sl);
  h = __dadd_rn(h, __dmul_rn(r, __dmul_rn(0.5, __drcp_rn(h))));
  return __dmul_rn(h, up);
}

// the exponent edges of abs_rn, out of line: |a| >= 2^1001, or |a| < 2^-1000
__device__ __noinline__ double abs_rn_edge(double a, double b, int e) {
  if (e == -1023) {  // subnormal: a = A 2^-1074, b = B 2^-1074, |s| = round(sqrt(A^2 + B^2)) 2^-1074
    const unsigned long long A = (unsigned long long)__double_as_longlong(a), B = (unsigned long long)__double_as_longlong(b);
    const unsigned __int128 N4 = ((unsigned __int128)A * A + (unsigned __int128)B * B) * 4;
    unsigned long long k = (unsigned long long)__dsqrt_rn(__ull2double_rn(A) * (double)A + __ull2double_rn(B) * (double)B);
    while ((unsigned __int128)(2 * k + 1) * (2 * k + 1) < N4) ++k;
    while (k > 0 && (unsigned __int128)(2 * k - 1) * (2 * k - 1) > N4) --k;
    return __longlong_as_double((long long)k);  // k < 2^53: the double with the bits of k is k 2^-1074
  }
  // one exact power-of-two step into the range of abs_rn_scaled: 2^-128 for huge a (b may underflow, but then
  // b / a < 2^-1000 and b is negligible; the final product rounds to inf exactly when |s| does), 2^128 for small
  // normal a (exact both ways: the result is at least a >= 2^-1022)
  const double pre = e > 0 ? 0x1p-128 : 0x1p128, post = e > 0 ? 0x1p128 : 0x1p-128;
  return __dmul_rn(abs_rn_scaled(__dmul_rn(a, pre), __dmul_rn(b, pre), e > 0 ? e - 128 : e + 128), post);
}

// |s| (np.abs = C's hypot: an infinite part gives +inf even next to a NaN).  Normal |a| >= |b|: the square root of
// the sum of squares held exactly as a double-double, corrected by one Newton step on the residual, in a frame scaled
// by powers of two so that neither square over- or underflows.  The corrected value is within 2^-48 ulp of the exact
// one, so the result is the correctly rounded one unless |s| lies within that distance of a midpoint between two
// doubles; midpoints are reached exactly (a Pythagorean triple with an odd 54-bit hypotenuse, scaled by a power of
// two), and there the result is one of the two neighbours, not necessarily the even one.  Subnormal |a|: a and b are
// integer multiples of 2^-1074, and round(sqrt(A^2 + B^2)) is exact in 128-bit integers (the square root of an
// integer is never half way).
__device__ __forceinline__ double abs_rn(double2 v) {
  double a = fabs(v.x), b = fabs(v.y);
  if (a < b) { const double t = a; a = b; b = t; }
  if (b == 0.0 || !isfinite(a) || isnan(b))
    return isinf(a) || isinf(b) ? __longlong_as_double(0x7ff0000000000000ll) : a + b;
  const int e = (int)((__double_as_longlong(a) >> 52) & 0x7ff) - 1023;
  if (e < -1000 || e > 1000) return abs_rn_edge(a, b, e);
  return abs_rn_scaled(a, b, e);
}

// NumPy's complex division (umath loops: Smith's method, a zero divisor gives the inf / nan of the real divisions)
__device__ __forceinline__ double2 np_cdiv(double2 a, double2 b) {
  const double br = fabs(b.x), bi = fabs(b.y);
  if (br >= bi) {
    if (br == 0.0 && bi == 0.0) return make_double2(a.x / br, a.y / br);
    const double rat = b.y / b.x, scl = 1.0 / __dadd_rn(b.x, __dmul_rn(b.y, rat));
    return make_double2(__dmul_rn(__dadd_rn(a.x, __dmul_rn(a.y, rat)), scl),
                        __dmul_rn(__dsub_rn(a.y, __dmul_rn(a.x, rat)), scl));
  }
  const double rat = b.x / b.y, scl = 1.0 / __dadd_rn(b.y, __dmul_rn(b.x, rat));
  return make_double2(__dmul_rn(__dadd_rn(__dmul_rn(a.x, rat), a.y), scl),
                      __dmul_rn(__dsub_rn(__dmul_rn(a.y, rat), a.x), scl));
}

__device__ __forceinline__ void layout_offsets(const pbb_mask_layout& L, long long idx, long long& in,
                                               long long& out) {
  in = 0;
  out = 0;
  for (int a = L.nd - 1; a >= 0; --a) {
    const long long s = L.shape[a];
    const long long q = idx / s, c = idx - q * s;
    in += c * L.in_stride[a];
    out += c * L.out_stride[a];
    idx = q;
  }
}

// *status = 1 + row, keeping the smallest failing row
__device__ __forceinline__ void report_first_row(int* status, long long row) {
  const int v = (int)(row + 1);
  int old = *(volatile int*)status;
  while (old == 0 || old > v) {
    const int prev = atomicCAS(status, old, v);
    if (prev == old) break;
    old = prev;
  }
}

// ---- source-reduction masks -----------------------------------------------------------------------------------------
// One thread per index of `rest`: a first sweep over the sources reduces (argmax / sums), a second one re-reads the
// thread's own elements (an L1 hit) and writes the K mask values.  No per-source register array, so any K works.
template <class TI, class TO>
__global__ void __launch_bounds__(256) source_mask_kernel(const TI* __restrict__ x, int kind, int K, int D,
                                                          long long sK, long long sD, long long oK,
                                                          pbb_mask_layout rest, long long n, double eps,
                                                          TO* __restrict__ out) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    long long ib, ob;
    layout_offsets(rest, r, ib, ob);
    const TI* __restrict__ xr = x + ib;
    TO* __restrict__ o = out + ob;
    if (kind == PBB_MASK_IDEAL_BINARY || kind == PBB_MASK_WIENER_LIKE) {
      double best = 0.0, total = 0.0;
      int arg = 0;
      for (int k = 0; k < K; ++k) {
        double p = 0.0;
        for (int d = 0; d < D; ++d) p = __dadd_rn(p, abs2_rn(ld_elem(xr, k * sK + d * sD)));
        // np.argmax: the first maximum, and the first NaN over any number
        if (k == 0 || p > best || (p != p && best == best)) { best = p; arg = k; }
        total = __dadd_rn(total, p);
      }
      if (kind == PBB_MASK_IDEAL_BINARY) {
        for (int k = 0; k < K; ++k) st_elem(o + k * oK, make_double2(k == arg ? 1.0 : 0.0, 0.0));
      } else {
        const double den = __dadd_rn(total, eps);
        for (int k = 0; k < K; ++k) {
          double p = 0.0;
          for (int d = 0; d < D; ++d) p = __dadd_rn(p, abs2_rn(ld_elem(xr, k * sK + d * sD)));
          st_elem(o + k * oK, make_double2(p / den, 0.0));
        }
      }
      continue;
    }
    double2 obs = make_double2(0.0, 0.0);
    double mag_sum = 0.0;
    for (int k = 0; k < K; ++k) {
      const double2 s = ld_elem(xr, k * sK);
      obs.x = __dadd_rn(obs.x, s.x);
      obs.y = __dadd_rn(obs.y, s.y);
      if (kind == PBB_MASK_IDEAL_RATIO) mag_sum = __dadd_rn(mag_sum, abs_rn(s));
    }
    const double obs_mag = abs_rn(obs), obs_angle = atan2(obs.y, obs.x);
    for (int k = 0; k < K; ++k) {
      const double2 s = ld_elem(xr, k * sK);
      double2 m;
      if (kind == PBB_MASK_IDEAL_RATIO) {
        m = make_double2(abs_rn(s) / __dadd_rn(mag_sum, eps), 0.0);
      } else if (kind == PBB_MASK_IDEAL_AMPLITUDE) {
        m = make_double2(abs_rn(s) / __dadd_rn(obs_mag, eps), 0.0);
      } else if (kind == PBB_MASK_PHASE_SENSITIVE) {
        const double theta = __dsub_rn(atan2(s.y, s.x), obs_angle);
        m = make_double2(__dmul_rn(abs_rn(s) / __dadd_rn(obs_mag, eps), cos(theta)), 0.0);
      } else if (IsComplex<TI>::value) {
        m = np_cdiv(s, obs);
      } else {
        m = make_double2(s.x / obs.x, 0.0);
      }
      st_elem(o + k * oK, m);
    }
  }
}

// ---- row selection --------------------------------------------------------------------------------------------------
struct SelState {
  unsigned long long prefix;  // selected high bits
  double above;               // Lorenz: sum of the elements above the selected bucket
  double total;               // Lorenz: sum of the row
  long long rank;             // rank: 0-based position from the top among the elements matching the prefix
  int fail;
  int nan;                    // quantile, long rows: the row holds a NaN (set by row_gather_kernel in query 0's state)
};

struct RowSelParams {
  int lorenz;           // 1: Lorenz threshold, 0: two order statistics (quantile)
  int below;            // quantile: mask = x < threshold
  int f32;              // quantile: values and interpolation in float
  int pad;
  double fraction;
  long long k_lower, k_upper;
  double gamma, one_minus_gamma;
  double mask_low, mask_high;
};

__device__ __forceinline__ unsigned long long sel_high_mask(int pass) {
  const int shift = 56 - 8 * pass;
  return pass == 0 ? 0ull : (~0ull << (shift + 8));
}

__device__ __forceinline__ void sel_count(unsigned* cnt, double* sum, unsigned long long* mx, double v, int pass,
                                          unsigned long long prefix, bool lorenz) {
  const unsigned long long key = (unsigned long long)__double_as_longlong(v);
  const bool in = (key & sel_high_mask(pass)) == prefix;
  const int b = in ? (int)((key >> (56 - 8 * pass)) & 255ull) : -1;
  if (!lorenz) {
    // counts only: lanes of the warp that hit the same bucket add once, through their lowest lane
    const unsigned peers = __match_any_sync(__activemask(), b);
    if (in && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cnt + b, (unsigned)__popc(peers));
    return;
  }
  if (!in) return;
  atomicAdd(cnt + b, 1u);
  {
    atomicAdd(sum + b, v);
    atomicMax(mx + b, key);
  }
}

template <class T>
__device__ __forceinline__ T warp_incl_scan(T v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// One warp chooses the next digit from a 256-bucket histogram; every lane returns the same new state.  Lane l looks at
// the buckets 255 - 8 l .. 248 - 8 l, i.e. descending positions 8 l .. 8 l + 7.
__device__ inline void warp_decide(const unsigned* cnt, const double* sum, const unsigned long long* mx, int pass,
                                   bool lorenz, double fraction, SelState& st, int lane) {
  unsigned c[8];
  unsigned ctot = 0;
  double stot = 0.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int b = kSelBuckets - 1 - (lane * 8 + j);
    c[j] = cnt[b];
    ctot += c[j];
    if (lorenz) stot += sum[b];
  }
  int found = -1;
  if (lorenz) {
    if (pass == 0) st.total = warp_sum(stot);  // butterfly: the same value in every lane
    double run = st.above + (warp_incl_scan(stot, lane) - stot), keep = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int b = kSelBuckets - 1 - (lane * 8 + j);
      if (c[j] && __ddiv_rn(run + __longlong_as_double((long long)mx[b]), st.total) < fraction) {
        found = lane * 8 + j;
        keep = run;
      }
      run += sum[b];
    }
    const int best = __reduce_max_sync(0xffffffffu, found);
    if (best < 0) { st.fail = 1; return; }
    st.above = __shfl_sync(0xffffffffu, keep, best >> 3);
    st.prefix |= (unsigned long long)(kSelBuckets - 1 - best) << (56 - 8 * pass);
    return;
  }
  long long run = (long long)(warp_incl_scan(ctot, lane) - ctot), newrank = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (c[j] && run <= st.rank && st.rank < run + (long long)c[j]) {
      found = lane * 8 + j;
      newrank = st.rank - run;
    }
    run += c[j];
  }
  const int best = __reduce_max_sync(0xffffffffu, found);
  if (best < 0) { st.fail = 1; return; }
  st.rank = __shfl_sync(0xffffffffu, newrank, best >> 3);
  st.prefix |= (unsigned long long)(kSelBuckets - 1 - best) << (56 - 8 * pass);
}

__device__ __forceinline__ void sel_init(SelState& st, const RowSelParams& p, int query, long long n) {
  st.prefix = 0ull;
  st.above = 0.0;
  st.total = 0.0;
  st.fail = 0;
  st.nan = 0;
  // rank from the top of the k-th smallest element
  st.rank = p.lorenz ? 0 : n - 1 - (query == 0 ? p.k_lower : p.k_upper);
}

// np.percentile's _lerp in the input precision
__device__ __forceinline__ double quantile_lerp(double lo, double hi, const RowSelParams& p) {
  if (p.f32) {
    const float a = (float)lo, b = (float)hi, d = __fsub_rn(b, a);
    return p.gamma >= 0.5 ? (double)__fsub_rn(b, __fmul_rn(d, (float)p.one_minus_gamma))
                          : (double)__fadd_rn(a, __fmul_rn(d, (float)p.gamma));
  }
  const double d = __dsub_rn(hi, lo);
  return p.gamma >= 0.5 ? __dsub_rn(hi, __dmul_rn(d, p.one_minus_gamma)) : __dadd_rn(lo, __dmul_rn(d, p.gamma));
}

// value of a row element: Lorenz -> sum over the sensors of |s|^2; quantile -> |s| (rounded to float for float input)
template <class TI>
__device__ __forceinline__ double row_value(const TI* __restrict__ x, long long off, int D, long long sD,
                                            const RowSelParams& p) {
  if (p.lorenz) {
    double v = 0.0;
    for (int d = 0; d < D; ++d) v = __dadd_rn(v, abs2_rn(ld_elem(x, off + d * sD)));
    return v;
  }
  const double a = abs_rn(ld_elem(x, off));
  return p.f32 ? (double)(float)a : a;
}

template <class TO>
__device__ __forceinline__ void store_mask(TO* out, long long off, double v, double thr, const RowSelParams& p) {
  const bool m = p.lorenz ? v > thr : (p.below ? v < thr : v > thr);
  out[off] = (TO)(m ? p.mask_high : p.mask_low);
}

// Short rows: a CTA loads R rows (R n <= kSelTileValues) into shared memory, each warp selects its rows with a private
// histogram, and the CTA writes the mask.  rowfast: consecutive rows are adjacent in memory (the row layout's innermost
// input stride is 1), so the tile is walked row-fastest and the loads coalesce.
template <class TI, class TO>
__global__ void __launch_bounds__(kSelWarps * 32, 1) row_select_short_kernel(
    const TI* __restrict__ x, int D, long long sD, pbb_mask_layout rows, long long nrows, pbb_mask_layout elems, int n,
    int R, int rowfast, RowSelParams p, TO* __restrict__ out, int* status) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* vals = reinterpret_cast<double*>(smem);
  double* thr = vals + (size_t)R * n;
  unsigned char* hist = reinterpret_cast<unsigned char*>(thr + R) + (threadIdx.x >> 5) * kSelHistBytes;
  double* hsum = reinterpret_cast<double*>(hist);
  unsigned long long* hmax = reinterpret_cast<unsigned long long*>(hsum + kSelBuckets);
  unsigned* hcnt = reinterpret_cast<unsigned*>(hmax + kSelBuckets);
  const long long row0 = (long long)blockIdx.x * R;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int total = R * n;
  for (int j = threadIdx.x; j < total; j += blockDim.x) {
    const int rl = rowfast ? j % R : j / n, i = rowfast ? j / R : j % n;
    if (row0 + rl >= nrows) continue;
    long long ri, ro, ei, eo;
    layout_offsets(rows, row0 + rl, ri, ro);
    layout_offsets(elems, i, ei, eo);
    vals[rl * n + i] = row_value(x, ri + ei, D, sD, p);
  }
  __syncthreads();
  for (int rl = warp; rl < R; rl += kSelWarps) {
    if (row0 + rl >= nrows) break;
    const double* v = vals + (size_t)rl * n;
    double sel_lo = 0.0, sel_hi = 0.0;
    bool fail = false, nan = false;
    const int queries = p.lorenz ? 1 : 2;
#pragma unroll 1
    for (int q = 0; q < queries; ++q) {
      SelState st;
      sel_init(st, p, q, n);
      for (int pass = 0; pass < kSelPasses && !st.fail; ++pass) {
        for (int b = lane; b < kSelBuckets; b += 32) { hcnt[b] = 0u; hsum[b] = 0.0; hmax[b] = 0ull; }
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
          const double x = v[i];
          nan |= x != x;
          sel_count(hcnt, hsum, hmax, x, pass, st.prefix, p.lorenz);
        }
        __syncwarp();
        warp_decide(hcnt, hsum, hmax, pass, p.lorenz, p.fraction, st, lane);
        __syncwarp();
      }
      fail |= st.fail != 0;
      (q == 0 ? sel_lo : sel_hi) = __longlong_as_double((long long)st.prefix);
    }
    // np.percentile of a row with a NaN is NaN, whatever the rank: no element compares true, every one is mask_low
    double t = p.lorenz ? sel_lo : quantile_lerp(sel_lo, sel_hi, p);
    if (!p.lorenz && __any_sync(0xffffffffu, nan)) t = __longlong_as_double(0x7ff8000000000000ll);
    if (fail) {
      t = __longlong_as_double(0x7ff0000000000000ll);  // +inf: the mask is mask_low; the caller raises
      if (lane == 0 && status) report_first_row(status, row0 + rl);
    }
    if (lane == 0) thr[rl] = t;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < total; j += blockDim.x) {
    const int rl = rowfast ? j % R : j / n, i = rowfast ? j / R : j % n;
    if (row0 + rl >= nrows) continue;
    long long ri, ro, ei, eo;
    layout_offsets(rows, row0 + rl, ri, ro);
    layout_offsets(elems, i, ei, eo);
    store_mask(out, ro + eo, vals[rl * n + i], thr[rl], p);
  }
}

// Long rows, `chunks` CTAs per row (CTA c of row r is blockIdx.x = r chunks + c, so any number of rows fits the grid):
// the row values go to scratch once, then every digit is one histogram launch (shared-memory histogram per CTA, merged
// into the row's global histogram with atomics) and one decide launch (a warp per row, which also clears the histogram
// for the next digit).
template <class TI>
__global__ void __launch_bounds__(256) row_gather_kernel(const TI* __restrict__ x, int D, long long sD,
                                                         pbb_mask_layout rows, pbb_mask_layout elems, long long n,
                                                         int chunks, RowSelParams p, double* __restrict__ vals,
                                                         SelState* __restrict__ state) {
  const long long row = blockIdx.x / chunks, chunk = blockIdx.x - row * chunks;
  long long ri, ro;
  layout_offsets(rows, row, ri, ro);
  if (p.lorenz) {
    for (long long i = chunk * blockDim.x + threadIdx.x; i < n; i += (long long)chunks * blockDim.x) {
      long long ei, eo;
      layout_offsets(elems, i, ei, eo);
      vals[row * n + i] = row_value(x, ri + ei, D, sD, p);
    }
    return;
  }
  bool nan = false;
  for (long long i = chunk * blockDim.x + threadIdx.x; i < n; i += (long long)chunks * blockDim.x) {
    long long ei, eo;
    layout_offsets(elems, i, ei, eo);
    const double v = row_value(x, ri + ei, D, sD, p);
    nan |= v != v;
    vals[row * n + i] = v;
  }
  if (nan) state[row * 2].nan = 1;
}

__global__ void __launch_bounds__(256) row_hist_kernel(const double* __restrict__ vals, long long n, int chunks,
                                                       int pass, int query, int lorenz,
                                                       const SelState* __restrict__ state,
                                                       unsigned char* __restrict__ ghist) {
  // one sub-histogram per warp: the leading digits put almost every value into one or two buckets, and eight copies
  // cut the shared-memory atomic contention on them eightfold
  __shared__ unsigned cnt[8][kSelBuckets];
  __shared__ double sum[8][kSelBuckets];
  __shared__ unsigned long long mx[8][kSelBuckets];
  const long long row = blockIdx.x / chunks, chunk = blockIdx.x - row * chunks;
  const SelState st = state[row * 2 + query];
  if (st.fail) return;
  for (int b = threadIdx.x; b < 8 * kSelBuckets; b += blockDim.x) {
    cnt[0][b] = 0u;
    sum[0][b] = 0.0;
    mx[0][b] = 0ull;
  }
  __syncthreads();
  const int w = threadIdx.x >> 5;
  const double* __restrict__ v = vals + row * n;
  for (long long i = chunk * blockDim.x + threadIdx.x; i < n; i += (long long)chunks * blockDim.x)
    sel_count(cnt[w], sum[w], mx[w], v[i], pass, st.prefix, lorenz != 0);
  __syncthreads();
  unsigned char* h = ghist + row * kSelHistBytes;
  double* gsum = reinterpret_cast<double*>(h);
  unsigned long long* gmax = reinterpret_cast<unsigned long long*>(gsum + kSelBuckets);
  unsigned* gcnt = reinterpret_cast<unsigned*>(gmax + kSelBuckets);
  for (int b = threadIdx.x; b < kSelBuckets; b += blockDim.x) {
    unsigned c = 0;
    double s = 0.0;
    unsigned long long m = 0ull;
    for (int k = 0; k < 8; ++k) {
      c += cnt[k][b];
      s += sum[k][b];
      m = max(m, mx[k][b]);
    }
    if (!c) continue;
    atomicAdd(gcnt + b, c);
    if (lorenz) {
      atomicAdd(gsum + b, s);
      atomicMax(gmax + b, m);
    }
  }
}

__global__ void row_decide_kernel(long long n, int pass, int query, RowSelParams p, SelState* __restrict__ state,
                                  unsigned char* __restrict__ ghist) {
  const long long row = blockIdx.x;
  const int lane = threadIdx.x;
  SelState st = state[row * 2 + query];
  unsigned char* h = ghist + row * kSelHistBytes;
  double* gsum = reinterpret_cast<double*>(h);
  unsigned long long* gmax = reinterpret_cast<unsigned long long*>(gsum + kSelBuckets);
  unsigned* gcnt = reinterpret_cast<unsigned*>(gmax + kSelBuckets);
  if (!st.fail) warp_decide(gcnt, gsum, gmax, pass, p.lorenz, p.fraction, st, lane);
  __syncwarp();
  for (int b = lane; b < kSelBuckets; b += 32) { gcnt[b] = 0u; gsum[b] = 0.0; gmax[b] = 0ull; }
  if (lane == 0) state[row * 2 + query] = st;
}

// both queries' states, before row_gather_kernel flags the NaN rows and before pass 0 of the histogram reads them
__global__ void row_state_init_kernel(long long rows, long long n, RowSelParams p, SelState* state) {
  const long long row = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (row >= rows) return;
  for (int query = 0; query < 2; ++query) {
    SelState st;
    sel_init(st, p, query, n);
    state[row * 2 + query] = st;
  }
}

template <class TO>
__global__ void __launch_bounds__(256) row_apply_kernel(const double* __restrict__ vals, pbb_mask_layout rows,
                                                        pbb_mask_layout elems, long long n, int chunks, RowSelParams p,
                                                        const SelState* __restrict__ state, TO* __restrict__ out,
                                                        int* status) {
  const long long row = blockIdx.x / chunks, chunk = blockIdx.x - row * chunks;
  const SelState s0 = state[row * 2], s1 = state[row * 2 + 1];
  const bool fail = s0.fail || (!p.lorenz && s1.fail);
  const double a = __longlong_as_double((long long)s0.prefix), b = __longlong_as_double((long long)s1.prefix);
  double thr = fail ? __longlong_as_double(0x7ff0000000000000ll) : (p.lorenz ? a : quantile_lerp(a, b, p));
  if (!p.lorenz && s0.nan) thr = __longlong_as_double(0x7ff8000000000000ll);  // np.percentile: NaN, all mask_low
  if (fail && chunk == 0 && threadIdx.x == 0 && status) report_first_row(status, row);
  long long ri, ro;
  layout_offsets(rows, row, ri, ro);
  for (long long i = chunk * blockDim.x + threadIdx.x; i < n; i += (long long)chunks * blockDim.x) {
    long long ei, eo;
    layout_offsets(elems, i, ei, eo);
    store_mask(out, ro + eo, vals[row * n + i], thr, p);
  }
}

// ---- biased binary mask ---------------------------------------------------------------------------------------------
template <class TI>
__global__ void __launch_bounds__(256) biased_binary_kernel(const TI* __restrict__ x, long long sC, long long oC,
                                                            pbb_mask_layout rest, long long n, int L,
                                                            const double* __restrict__ speech_div,
                                                            const double* __restrict__ noise_div,
                                                            const unsigned char* __restrict__ force,
                                                            unsigned char* __restrict__ out) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    long long ib, ob;
    layout_offsets(rest, r, ib, ob);
    const int j = (int)(r % L);
    const double ps = abs2_rn(ld_elem(x, ib)), pn = abs2_rn(ld_elem(x, ib + sC));
    const double ts = ps / speech_div[j], tn = ps / noise_div[j];
    bool speech = ts > pn && ts > 0.005;
    bool noise = tn < pn || tn < 0.005;
    if (force[j]) { speech = false; noise = true; }
    out[ob] = speech;
    out[ob + oC] = noise;
  }
}

// ---- array geometry -------------------------------------------------------------------------------------------------
// one thread per (a, f): the M phases of column a, and their 2-norm over m when normalising
__global__ void steering_vector_kernel(const double* __restrict__ tdoa, int A, int M, const double* __restrict__ freq,
                                       int F, int normalize, double2* __restrict__ out) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)A * F) return;
  const int a = (int)(idx / F), f = (int)(idx % F);
  // NumPy: (-2j * pi) * f -> (+-0, -2 pi f); times tdoa -> (+-0, (-2 pi f) tdoa); exp of a zero real part
  const double w = __dmul_rn(-2.0 * 3.141592653589793, freq[f]);
  double scl = 1.0;
  if (normalize) {
    double s = 0.0;
    for (int m = 0; m < M; ++m) {
      double sn, cs;
      sincos(__dmul_rn(w, tdoa[(size_t)a * M + m]), &sn, &cs);
      s = __dadd_rn(s, abs2_rn(make_double2(cs, sn)));
    }
    scl = 1.0 / sqrt(s);  // in-place complex / real divides by (norm + 0j): Smith's method multiplies by 1 / norm
  }
  for (int m = 0; m < M; ++m) {
    double sn, cs;
    sincos(__dmul_rn(w, tdoa[(size_t)a * M + m]), &sn, &cs);
    out[((size_t)a * M + m) * F + f] = normalize ? make_double2(__dmul_rn(cs, scl), __dmul_rn(sn, scl))
                                                 : make_double2(cs, sn);
  }
}

__global__ void diffuse_coherence_kernel(const double* __restrict__ dist, int D, const double* __restrict__ freq,
                                         int F, double c, double* __restrict__ out) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)F * D * D) return;
  const int f = (int)(idx / ((long long)D * D)), de = (int)(idx % ((long long)D * D));
  double xv = __dmul_rn(__dmul_rn(2.0, freq[f]), dist[de]) / c;
  if (xv == 0.0) xv = 1.0e-20;  // np.sinc
  const double y = __dmul_rn(3.141592653589793, xv);
  out[idx] = sin(y) / y;
}

// mode 0: |source[:, s] - sensor[:, m]| / c -> out (S, M); mode 1: far-field TDOA -> out (M, S), S = angles
__global__ void array_geometry_kernel(int mode, const double* __restrict__ pts, int S, const double* __restrict__ sensor,
                                      int M, int ref, double c, double* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * M) return;
  if (mode == 0) {
    const int s = idx / M, m = idx % M;
    double acc = 0.0;
    for (int i = 0; i < 3; ++i) {
      const double d = __dsub_rn(pts[i * S + s], sensor[i * M + m]);
      acc = __dadd_rn(acc, __dmul_rn(d, d));
    }
    out[idx] = sqrt(acc) / c;
    return;
  }
  const int m = idx / S, k = idx % S;
  const double az = pts[k], el = pts[S + k];
  const double ca = cos(az), sa = sin(az), ce = cos(-el), se = sin(-el);
  const double u[3] = {-__dmul_rn(ce, ca), -sa, __dmul_rn(se, ca)};
  double acc = 0.0;
  for (int i = 0; i < 3; ++i) acc = fma(__dsub_rn(sensor[i * M + m], sensor[i * M + ref]), u[i], acc);
  out[idx] = acc / c;
}

}  // namespace pbb
