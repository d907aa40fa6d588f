// SRMR, the speech-to-reverberation modulation energy ratio (pbb_srmr_* in include/pbb.h).  All fp64 except the VAD's
// threshold compare, which is in the input precision as in the reference; no float atomics (bitwise reproducible).
//
//   VAD + normalisation   vad_tile_kernel<T, phase> over tiles of kVadTile samples (several CTAs per row) and
//                         vad_row_kernel<T, phase> over the tiles of a row (one CTA per row):
//                           max|x| -> threshold; first / last above-threshold index per tile -> the nearest above
//                           index before / after every tile; keep flags -> kept count per tile -> offsets and N_r;
//                           compaction into the zero-filled (rows, N) output with the partial sums -> mean;
//                           sum of squares -> std; (x - mean) / std in place
//   Hilbert envelope      the gammatone outputs (n, rows, N) in place: hypot(y, y conv g), g the discrete Hilbert
//                         kernel of length N_r, as one real FFT of M = 2P points per sequence through fft_large.cuh
//                         (kernel spectra once per row)
//   modulation energies   each (row, band, modulation filter) is a 2-state DF2T recurrence, scanned over hop blocks
//                         of S samples: srmr_block_kernel<false> (zero-start end states), srmr_carry_kernel,
//                         srmr_block_kernel<true> (rerun; the four quarter-window energies of every block), then
//                         srmr_mean_kernel: E_f = sum_q P[f + q][q] and the mean over the frames
//   ratio                 srmr_ratio_kernel, one thread per row
#pragma once
#include "fft_large.cuh"

namespace pbb {

// ---- VAD + normalisation ---------------------------------------------------------------------------------------
constexpr int kVadThreads = 512, kVadPer = 8, kVadTile = kVadThreads * kVadPer;
constexpr int kVadRowThreads = 1024;  // one tile per thread: rows of up to 1024 tiles (PBB_SRMR_MAX_SAMPLES)
static_assert(kVadTile == PBB_SRMR_VAD_TILE, "tile size");
static_assert((long long)kVadRowThreads * kVadTile >= PBB_SRMR_MAX_SAMPLES, "row kernel covers every tile");

enum { VAD_MAX, VAD_EDGES, VAD_COUNT, VAD_COMPACT, VAD_MOMENTS, VAD_NORMALISE };
enum { ROW_THRESHOLD, ROW_EDGES, ROW_OFFSETS, ROW_MEAN, ROW_STD };

struct VadParams {
  const void* x;        // (rows, N), T
  long long rows, N;
  int tiles;
  double gap;           // 0.05 * sample_rate: wider gaps between above-threshold samples are removed
  double* tmax;         // (rows, tiles): max|x| of the tile; then the row's threshold in [row * tiles]
  long long* first;     // (rows, tiles): first above index of the tile; then the nearest above index after it
  long long* last;      // (rows, tiles): last above index; then the nearest above index before it
  long long* count;     // (rows, tiles): kept samples; then the tile's offset in the output
  double* psum;         // (rows, tiles): partial sums
  double* stats;        // (rows, 2): mean, std
  long long* nr;        // (rows): N_r
  double* out;          // (rows, N), zero past N_r
};

// max that propagates NaN, as ndarray.max does
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

struct MaxOp { __device__ long long operator()(long long a, long long b) const { return a > b ? a : b; } };
struct MinOp { __device__ long long operator()(long long a, long long b) const { return a < b ? a : b; } };
struct AddOp { __device__ long long operator()(long long a, long long b) const { return a + b; } };

// Exclusive scan of one value per thread in thread order (kReverse: from the last thread down); *total gets the
// whole block's.  sh: 33 entries of shared memory.  Ends with a barrier, so sh can be reused.
template <bool kReverse, class Op>
__device__ long long block_scan(long long v, Op op, long long id, long long* sh, long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = kReverse ? __shfl_down_sync(0xffffffffu, v, o) : __shfl_up_sync(0xffffffffu, v, o);
    if (kReverse ? lane + o < 32 : lane >= o) v = op(v, t);
  }
  long long ex = kReverse ? __shfl_down_sync(0xffffffffu, v, 1) : __shfl_up_sync(0xffffffffu, v, 1);
  if (kReverse ? lane == 31 : lane == 0) ex = id;
  if (kReverse ? lane == 0 : lane == 31) sh[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long acc = id;
    for (int i = 0; i < nw; ++i) {
      const int w = kReverse ? nw - 1 - i : i;
      const long long t = sh[w];
      sh[w] = acc;
      acc = op(acc, t);
    }
    sh[32] = acc;
  }
  __syncthreads();
  const long long r = op(sh[warp], ex);
  *total = sh[32];
  __syncthreads();
  return r;
}

// Block sum in a fixed order: warp butterflies, then the warp totals in warp order.
__device__ double block_sum(double v, double* sh) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += sh[i];
  __syncthreads();
  return s;
}

__device__ double block_nan_max(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double m = sh[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = nan_max(m, sh[i]);
  __syncthreads();
  return m;
}

template <class T>
__device__ __forceinline__ T abs_t(T v) { return v < T(0) ? -v : v; }

// Keep flags of the thread's kVadPer samples (bit j: sample t0 + j < N) from the above-threshold flags and the nearest
// above indices before and after them.
__device__ __forceinline__ unsigned vad_keep(unsigned above, long long t0, long long prev, long long next,
                                             long long N, double gap) {
  long long nx[kVadPer];
#pragma unroll
  for (int j = kVadPer - 1; j >= 0; --j) {
    if (above >> j & 1) next = t0 + j;
    nx[j] = next;
  }
  unsigned keep = 0;
#pragma unroll
  for (int j = 0; j < kVadPer; ++j) {
    const bool a = above >> j & 1;
    if (a) prev = t0 + j;
    // removed: strictly between two above-threshold samples more than gap apart (L[i+1] - L[i] > 0.05 sr)
    const bool removed = !a && prev >= 0 && nx[j] < N && (double)(nx[j] - prev) > gap;
    if (!removed && t0 + j < N) keep |= 1u << j;
  }
  return keep;
}

// The sum of squares about the mean (VAD_MOMENTS) or the normalisation in place (VAD_NORMALISE) of the first N_r
// samples of the compacted rows.
template <int PHASE>
__global__ void __launch_bounds__(kVadThreads) vad_norm_kernel(const VadParams p) {
  __shared__ double shd[32];
  const long long row = blockIdx.x / p.tiles;
  const long long ti = row * p.tiles + blockIdx.x % p.tiles;
  const long long t0 = (long long)(blockIdx.x % p.tiles) * kVadTile + threadIdx.x * kVadPer;
  double* out = p.out + row * p.N;
  const long long L = p.nr[row];
  const double mean = p.stats[2 * row], sd = p.stats[2 * row + 1];
  double s2 = 0.0;
#pragma unroll
  for (int j = 0; j < kVadPer; ++j) {
    const long long t = t0 + j;
    if (t < L) {
      const double y = out[t] - mean;
      if (PHASE == VAD_MOMENTS) s2 += y * y;
      else out[t] = y / sd;
    }
  }
  if (PHASE == VAD_MOMENTS) {
    s2 = block_sum(s2, shd);
    if (threadIdx.x == 0) p.psum[ti] = s2;
  }
}

template <class T, int PHASE>
__global__ void __launch_bounds__(kVadThreads) vad_tile_kernel(const VadParams p) {
  __shared__ long long shl[33];
  __shared__ double shd[32];
  const long long row = blockIdx.x / p.tiles;
  const int tile = (int)(blockIdx.x % p.tiles);
  const long long ti = row * p.tiles + tile;
  const long long t0 = (long long)tile * kVadTile + threadIdx.x * kVadPer;
  const T* x = static_cast<const T*>(p.x) + row * p.N;
  double* out = p.out + row * p.N;
  T v[kVadPer];
#pragma unroll
  for (int j = 0; j < kVadPer; ++j) v[j] = t0 + j < p.N ? x[t0 + j] : T(0);
  if (PHASE == VAD_MAX) {
    double m = 0.0;
#pragma unroll
    for (int j = 0; j < kVadPer; ++j) m = nan_max(m, (double)abs_t(v[j]));
    m = block_nan_max(m, shd);
    if (threadIdx.x == 0) p.tmax[ti] = m;
    return;
  }
  const T thr = (T)p.tmax[row * p.tiles];
  unsigned above = 0;
#pragma unroll
  for (int j = 0; j < kVadPer; ++j)
    if (t0 + j < p.N && abs_t(v[j]) > thr) above |= 1u << j;
  const long long none_after = p.N;  // "no above index" sentinels: -1 before, N after
  const long long f = above ? t0 + __ffs(above) - 1 : none_after;
  const long long l = above ? t0 + 31 - __clz(above) : -1;
  long long tot;
  if (PHASE == VAD_EDGES) {
    block_scan<false>(l, MaxOp(), -1ll, shl, &tot);
    if (threadIdx.x == 0) p.last[ti] = tot;
    block_scan<false>(f, MinOp(), none_after, shl, &tot);
    if (threadIdx.x == 0) p.first[ti] = tot;
    return;
  }
  const long long prev = MaxOp()(block_scan<false>(l, MaxOp(), -1ll, shl, &tot), p.last[ti]);
  const long long next = MinOp()(block_scan<true>(f, MinOp(), none_after, shl, &tot), p.first[ti]);
  const unsigned keep = vad_keep(above, t0, prev, next, p.N, p.gap);
  const long long kept = __popc(keep);
  if (PHASE == VAD_COUNT) {
    block_scan<false>(kept, AddOp(), 0ll, shl, &tot);
    if (threadIdx.x == 0) p.count[ti] = tot;
    return;
  }
  // VAD_COMPACT
  long long pos = p.count[ti] + block_scan<false>(kept, AddOp(), 0ll, shl, &tot);
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < kVadPer; ++j)
    if (keep >> j & 1) {
      const double d = (double)v[j];
      out[pos++] = d;
      s += d;
    }
  s = block_sum(s, shd);
  if (threadIdx.x == 0) p.psum[ti] = s;
}

template <class T, int PHASE>
__global__ void __launch_bounds__(kVadRowThreads) vad_row_kernel(const VadParams p) {
  __shared__ long long shl[33];
  __shared__ double shd[32];
  const long long row = blockIdx.x;
  const int i = threadIdx.x;
  const bool mine = i < p.tiles;
  const long long ti = row * p.tiles + i;
  if (PHASE == ROW_THRESHOLD) {
    const double m = block_nan_max(mine ? p.tmax[ti] : 0.0, shd);
    if (i == 0) {
      const T mt = (T)m;
      p.tmax[row * p.tiles] = (double)((mt * mt) / (T)100000);  // (max_val ** 2) / (10 ** 5), in T
    }
    return;
  }
  long long tot;
  if (PHASE == ROW_EDGES) {
    const long long l = mine ? p.last[ti] : -1, f = mine ? p.first[ti] : p.N;
    const long long before = block_scan<false>(l, MaxOp(), -1ll, shl, &tot);
    const long long after = block_scan<true>(f, MinOp(), p.N, shl, &tot);
    if (mine) {
      p.last[ti] = before;
      p.first[ti] = after;
    }
    return;
  }
  if (PHASE == ROW_OFFSETS) {
    const long long off = block_scan<false>(mine ? p.count[ti] : 0ll, AddOp(), 0ll, shl, &tot);
    if (mine) p.count[ti] = off;
    if (i == 0) p.nr[row] = tot;
    return;
  }
  const double s = block_sum(mine ? p.psum[ti] : 0.0, shd);
  if (i == 0) {
    const double L = (double)p.nr[row];
    if (PHASE == ROW_MEAN) p.stats[2 * row] = s / L;
    else p.stats[2 * row + 1] = sqrt(s / L);
  }
}

// ---- Hilbert envelope ----------------------------------------------------------------------------------------------
// The discrete Hilbert kernel of length L at 1 <= n < L (hilbert(x).imag = x circularly convolved with g): even L:
// 2 cot(pi n / L) / L at odd n, else 0; odd L: cot(pi n / (2L)) / L at odd n, -tan(pi n / (2L)) / L at even n.
// Evaluated at e = min(n, L - n), with g[L - n] = -g[n], so that the angle near n = L keeps its digits.
__device__ __forceinline__ double hilbert_g(long long n, long long L) {
  const long long e = n < L - n ? n : L - n;
  const double sign = e == n ? 1.0 : -1.0;
  double s, c, g;
  if ((L & 1) == 0) {
    if ((e & 1) == 0) return 0.0;
    sincospi((double)e / (double)L, &s, &c);
    g = 2.0 * (c / s) / (double)L;
  } else {
    sincospi((double)e / (double)(2 * L), &s, &c);
    g = ((e & 1) ? c / s : -(s / c)) / (double)L;
  }
  return sign * g;
}

// Point j of the packed kernel of row g0 + seq: (k[2j], k[2j + 1]), k the length-M linear-convolution layout of g
// (lag d >= 0 at d, lag d < 0 at M + d).
struct HilbertKernelLoad {
  const long long* nr;
  long long g0, M;
  __device__ double k(long long t, long long L) const {
    if (t == 0) return 0.0;
    if (t < L) return hilbert_g(t, L);
    if (t > M - L) return -hilbert_g(M - t, L);
    return 0.0;
  }
  __device__ double2 operator()(long long seq, long long j) const {
    const long long L = nr[g0 + seq];
    return make_double2(k(2 * j, L), k(2 * j + 1, L));
  }
};

// Point j of the packed signal of sequence g0 + seq (band f, row r at s = f rows + r): (y[2j], y[2j + 1]), zero from
// N_r on.
struct HilbertSignalLoad {
  const double* y;
  const long long* nr;
  long long g0, rows, N;
  __device__ double2 operator()(long long seq, long long j) const {
    const long long s = g0 + seq, L = nr[s % rows], t = 2 * j;
    const double* p = y + s * N;
    return make_double2(t < L ? p[t] : 0.0, t + 1 < L ? p[t + 1] : 0.0);
  }
};

// Forward column pass: twiddle exp(-2 pi i n2 k1 / P) and store row k1 of the workspace.
struct FlForwardStore {
  double2* ws;
  int logP, logP2;
  __device__ void operator()(long long seq, int n2, int k1, double2 v) const {
    ws[(seq << logP) + ((long long)k1 << logP2) + n2] = cmul(v, fl_twiddle<-1>(n2, k1, logP));
  }
};

// Inverse column pass: z[j] = (Im[2j], Im[2j + 1]) of the analytic signal; the envelope over the signal in place.
struct EnvelopeStore {
  double* y;
  const long long* nr;
  long long g0, rows, N;
  int logP2;
  __device__ void operator()(long long seq, int n2, int n1, double2 v) const {
    const long long s = g0 + seq, L = nr[s % rows], t = 2 * (((long long)n1 << logP2) + n2);
    double* p = y + s * N;
    if (t < L) p[t] = hypot(p[t], v.x);
    if (t + 1 < L) p[t + 1] = hypot(p[t + 1], v.y);
  }
};

// Y[k] of the 2P-point real sequence from Z = DFT_P of its even/odd packing: (Z[k] + conj Z[P-k]) / 2 +
// W^k (Z[k] - conj Z[P-k]) / 2i, W = exp(-i pi / P); w = W^k.
__device__ __forceinline__ double2 real_split(double2 a, double2 b, double2 w) {
  const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
  const double2 fo = make_double2(0.5 * (a.y + b.y), -0.5 * (a.x - b.x));
  const double2 t = cmul(w, fo);
  return make_double2(fe.x + t.x, fe.y + t.y);
}

// Row pass of the kernel: Im K[k] per row (the kernel is real and odd, so K is imaginary), in the transposed order.
struct KernelSpectrumOp {
  static constexpr bool kInverse = false;
  double* ks;
  FlShape sh;
  long long g0;
  __device__ void operator()(long long seq, int kr, int k2, int, int, double2 a, double2 b, double2*) const {
    const long long k = kr + ((long long)k2 << sh.logP1);
    double s, c;
    sincospi(ldexp((double)k, -sh.logP), &s, &c);
    ks[((g0 + seq) << sh.logP) + ((long long)kr << sh.logP2) + k2] = real_split(a, b, make_double2(c, -s)).y;
  }
};

// Row pass of the signals: H = Y K at k and P - k, then the packed spectrum of the real inverse,
// Z'[k] = (H[k] + conj H[P-k]) / 2 + i (H[k] - conj H[P-k]) / 2 * conj W^k, scaled by 1 / P.
struct ConvolveOp {
  static constexpr bool kInverse = true;
  const double* ks;
  FlShape sh;
  long long g0, rows;
  __device__ void operator()(long long seq, int kr, int k2, int kp, int k2p, double2 a, double2 b, double2* o) const {
    const long long k = kr + ((long long)k2 << sh.logP1);
    const double* K = ks + (((g0 + seq) % rows) << sh.logP);
    double s, c;
    sincospi(ldexp((double)k, -sh.logP), &s, &c);
    const double2 yk = real_split(a, b, make_double2(c, -s));
    const double2 yp = real_split(b, a, make_double2(-c, -s));   // W^(P-k) = -conj W^-k
    const double kk = K[((long long)kr << sh.logP2) + k2];
    const double kq = k == 0 ? 0.0 : K[((long long)kp << sh.logP2) + k2p];  // K[P] = 0 for an odd kernel
    const double2 hk = make_double2(-yk.y * kk, yk.x * kk), hp = make_double2(-yp.y * kq, yp.x * kq);
    const double2 fe = make_double2(0.5 * (hk.x + hp.x), 0.5 * (hk.y - hp.y));
    const double2 fo = cmul(make_double2(0.5 * (hk.x - hp.x), 0.5 * (hk.y + hp.y)), make_double2(c, s));
    const double scale = ldexp(1.0, -sh.logP);
    *o = make_double2(scale * (fe.x - fo.y), scale * (fe.y + fo.x));
  }
};

// ---- modulation filters and energies ----------------------------------------------------------------------------------
struct ModParams {
  const double* env;      // (n * rows, N): sequence s = f rows + r
  const long long* nr;    // (rows)
  long long rows, N, seqs;  // seqs = n * rows
  int S, blocks;          // hop, blocks per sequence (ceil(N / S) + 3)
  const double* coef;     // (8, 3): b0, a1, a2 of b = [b0, 0, -b0], a = [1, a1, a2]
  const double* trans;    // (8, 4): the zero-input transition over S samples, row-major 2 x 2
  const double* window;   // (4 S): Hamming, sym
  double* state;          // (seqs * 8, blocks, 2): end states, then start states
  double* quarter;        // (seqs * 8, blocks, 4)
  double* means;          // (rows, n, 8)
  int n;
};

// One (sequence, modulation filter, block) per thread, the filter index fastest.
template <bool kEnergy>
__global__ void __launch_bounds__(256) srmr_block_kernel(const ModParams p) {
  const long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u >= p.seqs * 8 * p.blocks) return;
  const int k = (int)(u & 7);
  const long long sb = u >> 3, s = sb / p.blocks, b = sb - s * p.blocks, q = s * 8 + k;
  const long long L = p.nr[s % p.rows];
  const double b0 = p.coef[3 * k], na1 = -p.coef[3 * k + 1], na2 = -p.coef[3 * k + 2];
  double* st = p.state + (q * p.blocks + b) * 2;
  double z0 = kEnergy ? st[0] : 0.0, z1 = kEnergy ? st[1] : 0.0;
  const double* e = p.env + s * p.N;
  const long long t0 = b * p.S;
  double P[4] = {0.0, 0.0, 0.0, 0.0};
  // Only blocks before N_r run.  The end state of the block that holds N_r stops at N_r, which changes only the start
  // states of later blocks, whose samples are all past N_r and count for nothing.
  if (t0 < L) {
    const int len = (int)min((long long)p.S, L - t0);
    for (int j = 0; j < len; ++j) {
      const double x = e[t0 + j];
      const double y = fma(b0, x, z0);
      z0 = fma(na1, y, z1);
      z1 = fma(-b0, x, na2 * y);
      if (kEnergy) {
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
          const double wy = __ldg(p.window + qq * p.S + j) * y;
          P[qq] = fma(wy, wy, P[qq]);
        }
      }
    }
  }
  if (kEnergy) {
    double* o = p.quarter + (q * p.blocks + b) * 4;
#pragma unroll
    for (int qq = 0; qq < 4; ++qq) o[qq] = P[qq];
  } else {
    st[0] = z0;
    st[1] = z1;
  }
}

// s_{b+1} = A s_b + z_b over the blocks of every (sequence, filter), in place: the end states become start states.
__global__ void __launch_bounds__(256) srmr_carry_kernel(const ModParams p) {
  const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (q >= p.seqs * 8) return;
  const double* A = p.trans + 4 * (q & 7);
  const double a00 = A[0], a01 = A[1], a10 = A[2], a11 = A[3];
  double* st = p.state + q * p.blocks * 2;
  double s0 = 0.0, s1 = 0.0;
  for (int b = 0; b < p.blocks; ++b) {
    const double z0 = st[2 * b], z1 = st[2 * b + 1];
    st[2 * b] = s0;
    st[2 * b + 1] = s1;
    const double n0 = fma(a00, s0, fma(a01, s1, z0));
    s1 = fma(a10, s0, fma(a11, s1, z1));
    s0 = n0;
  }
}

// means[r][f][k] = (sum over the F_r frames of sum_q P[frame + q][q]) / F_r, in frame order.
__global__ void __launch_bounds__(256) srmr_mean_kernel(const ModParams p) {
  const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (q >= p.seqs * 8) return;
  const int k = (int)(q & 7);
  const long long s = q >> 3, r = s % p.rows, f = s / p.rows;
  const long long L = p.nr[r], W = 4ll * p.S;
  const long long F = L < W ? 1 : 1 + (L - W + p.S - 1) / p.S;
  const double* P = p.quarter + q * p.blocks * 4;
  double sum = 0.0;
  for (long long fr = 0; fr < F; ++fr) {
    const double e = ((P[fr * 4] + P[(fr + 1) * 4 + 1]) + P[(fr + 2) * 4 + 2]) + P[(fr + 3) * 4 + 3];
    sum += e;
  }
  p.means[(r * p.n + f) * 8 + k] = sum / (double)F;
}

// ---- ratio --------------------------------------------------------------------------------------------------------
// module_srmr.py:121-154: the first acoustic band at which the cumulative energy share exceeds 90 % sets BW; the
// denominator takes the modulation bands 4, 5 and then 6, 7 until BW lies between two consecutive cutoffs.
__global__ void srmr_ratio_kernel(const double* __restrict__ means, long long rows, int n,
                                  const double* __restrict__ erb, const double* __restrict__ cutoff,
                                  double* __restrict__ out) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const double* m = means + r * n * 8;
  double total = 0.0, col[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int f = 0; f < n; ++f)
    for (int k = 0; k < 8; ++k) {
      total += m[f * 8 + k];
      col[k] += m[f * 8 + k];
    }
  double sum = 0.0, bw = 0.0;
  for (int f = 0; f < n; ++f) {
    double ac = 0.0;
    for (int k = 0; k < 8; ++k) ac += m[f * 8 + k];
    sum += ac * 100.0 / total;
    if (sum > 90.0) {
      bw = erb[f];
      break;
    }
  }
  const double num = ((col[0] + col[1]) + col[2]) + col[3];
  double den = col[4];
  for (int i = 5; i < 8; ++i) {
    den += col[i];
    if (cutoff[i - 1] < bw && bw < cutoff[i]) break;
  }
  out[r] = num / den;
}

}  // namespace pbb
