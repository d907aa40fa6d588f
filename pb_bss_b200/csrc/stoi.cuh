// STOI, the short-time objective intelligibility of pb_bss/evaluation/module_stoi.py (pystoi.stoi, extended=False;
// Taal et al., IEEE TASLP 19(7), 2011), for a group of rows at once -- see include/pbb.h (pbb_stoi).  fp64, no float
// atomics: every reduction has a fixed order that depends on the shape only, so a row's bits do not depend on the
// batch it is in.
//
//   stoi_resample_kernel   polyphase resample_poly to 10 kHz of x and y (skipped at 10 kHz)
//   stoi_energy_kernel     20 log10(||w x_f|| + eps) of every 256-sample frame f, 128 f < L - 256
//   stoi_compact_kernel    per row: max E, keep mask, prefix sum -> kept-frame list, K_r, M_r = max(K_r - 1, 0)
//   stoi_bands_kernel      STFT frames of the overlap-added kept frames, windowed twice, 512-point real FFT,
//                          one-third octave band energies
//   stoi_segment_kernel    the correlation of every (segment, band), summed per block of segments
//   estoi_segment_kernel   ESTOI (pbb_estoi; Jensen and Taal, IEEE/ACM TASLP 24(11), 2016) in place of the above:
//                          the row- and column-normalised segments' inner products, summed per block of segments
//   stoi_value_kernel      per row: the sum of the block sums / (J 15), or / (J 30) for ESTOI, or 1e-5 below 30
//                          frames; the status word
#pragma once
#include "common.cuh"
#include "fft_stages.cuh"

namespace pbb {

constexpr int kStoiFrame = PBB_STOI_FRAME, kStoiHop = PBB_STOI_FRAME / 2;
constexpr int kStoiLogM = 8;  // the 512-point real FFT is one 256-point complex FFT
constexpr int kStoiBins = PBB_STOI_NFFT / 2 + 1, kStoiBands = PBB_STOI_BANDS, kStoiSeg = PBB_STOI_SEGMENT;
constexpr double kStoiEps = 2.220446049250313e-16;   // np.finfo(float).eps
constexpr double kStoiClip = 1.0 + 5.623413251903491;  // 1 + 10 ** (-BETA / 20), BETA = -15
constexpr int kStoiThreads = 256;
constexpr int kStoiFpc = 4;          // STFT frames per CTA of stoi_bands_kernel (32 KB of shared memory)
constexpr int kStoiSegBlock = 64;    // segments per CTA of stoi_segment_kernel
constexpr int kStoiCompactThreads = 1024;

struct StoiParams {
  const void* x;  // (rows, n) reference, input dtype
  const void* y;  // (rows, n) estimate
  long long rows, n, L;  // rows of the group, input length, length at 10 kHz
  int F, Mmax, blocks;   // frames of the silence detection, STFT frames at most (F - 1), segment blocks
  int up, down, tpp;     // rates in lowest terms, taps per phase
  long long pre_remove;
  const double* taps;    // (up, tpp): taps[ph][m] = h[ph + m up] of scipy's zero-padded, up-scaled filter
  const double* window;  // (256) hanning(258)[1:-1]
  const int* bands;      // (15, 2) [lo, hi) bins
  const double2* tw;     // (512) (cos, sin)(2 pi k / 512)
  double* sig;           // (rows, 2, L) resampled x, y; null at 10 kHz (the input is read in place)
  double* energy;        // (rows, F)
  int* kept;             // (rows, F) kept-frame indices, K_r of them
  long long* km;         // (rows, 2) K_r, M_r
  double* tob;           // (rows, 2, 15, Mmax) band energies
  double* partial;       // (rows, blocks) block sums of the correlations
  double* out;           // (rows)
  long long* status;     // (2) count of rows below 30 frames, first such row (-1: none)
  long long row0;        // index of the group's first row in the call
  int terms;             // products summed per segment: 15 (STOI, one per band) or 30 (ESTOI, d_m times 30)
};

// numpy's maximum / minimum: NaN if either operand is NaN
__device__ __forceinline__ double np_max(double a, double b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ double np_min(double a, double b) { return (a < b || a != a) ? a : b; }

// sample i of signal s (0: x, 1: y) of row r at 10 kHz
template <class T>
__device__ __forceinline__ double stoi_sample(const StoiParams& p, long long r, int s, long long i) {
  if (p.sig) return p.sig[(2 * r + s) * p.L + i];
  return (double)static_cast<const T*>(s ? p.y : p.x)[r * p.n + i];
}

// upfirdn(h, x, up, down)[j + pre_remove] = sum_i h[t - i up] x[i], t = (j + pre_remove) down: the taps of one phase
// against the samples i0, i0 - 1, ... (i0 = t / up), in increasing m.
template <class T>
__global__ void __launch_bounds__(kStoiThreads) stoi_resample_kernel(StoiParams p) {
  const long long total = p.rows * 2 * p.L;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long rs = i / p.L, j = i - rs * p.L;
    const T* src = static_cast<const T*>((rs & 1) ? p.y : p.x) + (rs >> 1) * p.n;
    const long long t = (j + p.pre_remove) * p.down, i0 = t / p.up;
    const double* h = p.taps + (t - i0 * p.up) * p.tpp;
    const long long m0 = i0 - (p.n - 1) > 0 ? i0 - (p.n - 1) : 0;
    const long long m1 = i0 + 1 < p.tpp ? i0 + 1 : p.tpp;
    double acc = 0.0;
    for (long long m = m0; m < m1; ++m) acc = fma(__ldg(h + m), (double)__ldg(src + i0 - m), acc);
    p.sig[i] = acc;
  }
}

// One warp per (row, frame) of the reference: lane l sums (w x)^2 over j = l + 32 k in increasing k, then a butterfly.
template <class T>
__global__ void __launch_bounds__(kStoiThreads) stoi_energy_kernel(StoiParams p) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= p.rows * p.F) return;
  const long long r = wid / p.F, f = wid - r * p.F;
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < kStoiFrame / 32; ++k) {
    const int j = lane + 32 * k;
    const double v = __ldg(p.window + j) * stoi_sample<T>(p, r, 0, f * kStoiHop + j);
    s = fma(v, v, s);
  }
  s = warp_sum(s);
  if (lane == 0) p.energy[wid] = 20.0 * log10(sqrt(s) + kStoiEps);
}

// One CTA per row: the NaN-propagating max of the energies, the keep mask (max - 40 - E_f < 0), and the kept-frame
// list by a block prefix sum over contiguous chunks of frames.
__global__ void __launch_bounds__(kStoiCompactThreads) stoi_compact_kernel(StoiParams p) {
  __shared__ double smax[kStoiCompactThreads / 32];
  __shared__ int scan[kStoiCompactThreads];
  const long long r = blockIdx.x;
  const double* e = p.energy + r * p.F;
  const int chunk = (p.F + kStoiCompactThreads - 1) / kStoiCompactThreads;
  const int f0 = min(p.F, (int)threadIdx.x * chunk), f1 = min(p.F, f0 + chunk);
  double m = -INFINITY;
  for (int f = f0; f < f1; ++f) m = np_max(e[f], m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = np_max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = m;
  __syncthreads();
  double emax = smax[0];
  for (int w = 1; w < kStoiCompactThreads / 32; ++w) emax = np_max(emax, smax[w]);
  const double thr = emax - (double)PBB_STOI_DYN_RANGE;
  int c = 0;
  for (int f = f0; f < f1; ++f) c += (thr - e[f]) < 0.0;
  scan[threadIdx.x] = c;
  __syncthreads();
  for (int o = 1; o < kStoiCompactThreads; o <<= 1) {
    const int v = threadIdx.x >= o ? scan[threadIdx.x - o] : 0;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  int k = scan[threadIdx.x] - c;
  int* kept = p.kept + r * p.F;
  for (int f = f0; f < f1; ++f)
    if ((thr - e[f]) < 0.0) kept[k++] = f;
  if (threadIdx.x == kStoiCompactThreads - 1) {
    const int K = scan[threadIdx.x];
    p.km[2 * r] = K;
    p.km[2 * r + 1] = K > 1 ? K - 1 : 0;
  }
}

// One CTA: kStoiFpc STFT frames of one (row, signal).  Sample j of STFT frame i of the overlap-added signal is the
// sum of the windowed kept frames i - 1 (second half) and i (j < 128), or i and i + 1 (first half, j >= 128): the
// two terms numpy's overlap-add adds, so the frame is bitwise numpy's before the FFT.
template <class T>
__global__ void __launch_bounds__(kStoiThreads) stoi_bands_kernel(StoiParams p) {
  constexpr int M = 1 << kStoiLogM;
  __shared__ double2 A[kStoiFpc * M], B[kStoiFpc * M];
  const int tiles = (p.Mmax + kStoiFpc - 1) / kStoiFpc;
  const long long rs = blockIdx.x / tiles, r = rs >> 1;
  const int s = (int)(rs & 1);
  const int t0 = (int)(blockIdx.x % tiles) * kStoiFpc;
  const int Mr = (int)p.km[2 * r + 1];
  if (t0 >= Mr) return;
  const int nf = min(kStoiFpc, Mr - t0);
  const int* kept = p.kept + r * p.F;
  for (int q = threadIdx.x; q < (nf << kStoiLogM); q += blockDim.x) {
    const int f = q >> kStoiLogM, c = q & (M - 1), i = t0 + f;
    double v[2] = {0.0, 0.0};
    if (c < kStoiFrame / 2) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = 2 * c + h;
        const long long a = (long long)__ldg(kept + i) * kStoiHop;
        double u = __ldg(p.window + j) * stoi_sample<T>(p, r, s, a + j);
        if (j < kStoiHop) {
          if (i > 0) {
            const long long b = (long long)__ldg(kept + i - 1) * kStoiHop;
            u = __ldg(p.window + j + kStoiHop) * stoi_sample<T>(p, r, s, b + j + kStoiHop) + u;
          }
        } else {
          const long long b = (long long)__ldg(kept + i + 1) * kStoiHop;
          u = u + __ldg(p.window + j - kStoiHop) * stoi_sample<T>(p, r, s, b + j - kStoiHop);
        }
        v[h] = __ldg(p.window + j) * u;
      }
    }
    A[q] = make_double2(v[0], v[1]);
  }
  __syncthreads();
  const double2* Z = fft_shared<-1>(A, B, kStoiLogM, nf, p.tw);
  double* pw = reinterpret_cast<double*>(Z == A ? B : A);  // |X_k|^2, (nf, 257)
  for (int q = threadIdx.x; q < nf * kStoiBins; q += blockDim.x) {
    const int f = q / kStoiBins, k = q - f * kStoiBins;
    const double2* z = Z + (f << kStoiLogM);
    double2 X;
    if (k == 0 || k == M) {
      const double2 z0 = z[0];
      X = make_double2(k == 0 ? z0.x + z0.y : z0.x - z0.y, 0.0);
    } else {
      // X_k = (Z_k + conj Z_{M-k}) / 2 + W^k (Z_k - conj Z_{M-k}) / 2i,  W = exp(-2 pi i / 512)
      const double2 a = z[k], b = z[M - k];
      const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
      const double2 fo = make_double2(0.5 * (a.y + b.y), -0.5 * (a.x - b.x));
      double2 w = __ldg(p.tw + k);
      w.y = -w.y;
      const double2 t = cmul(w, fo);
      X = make_double2(fe.x + t.x, fe.y + t.y);
    }
    pw[q] = X.x * X.x + X.y * X.y;
  }
  __syncthreads();
  if (threadIdx.x < nf * kStoiBands) {
    const int f = threadIdx.x / kStoiBands, band = threadIdx.x - f * kStoiBands;
    const int lo = __ldg(p.bands + 2 * band), hi = __ldg(p.bands + 2 * band + 1);
    double acc = 0.0;
    for (int k = lo; k < hi; ++k) acc += pw[f * kStoiBins + k];
    p.tob[((rs * kStoiBands) + band) * p.Mmax + t0 + f] = sqrt(acc);
  }
}

constexpr int kStoiSegFrames = kStoiSegBlock + kStoiSeg - 1;  // frames of a block of segments (the row stride W)

// The band energies of frames seg0 .. seg0 + nfr - 1 of row r into sx, sy (15, kStoiSegFrames).
__device__ __forceinline__ void stoi_stage_frames(const StoiParams& p, long long r, int seg0, int nfr, double* sx,
                                                  double* sy) {
  constexpr int W = kStoiSegFrames;
  const double* tx = p.tob + 2 * r * kStoiBands * p.Mmax;
  const double* ty = tx + kStoiBands * p.Mmax;
  for (int q = threadIdx.x; q < kStoiBands * nfr; q += blockDim.x) {
    const int b = q / nfr, f = q - b * nfr;
    sx[b * W + f] = tx[b * p.Mmax + seg0 + f];
    sy[b * W + f] = ty[b * p.Mmax + seg0 + f];
  }
}

// The CTA's sum of every thread's `local`, a fixed tree (warp butterfly, then the warps in order), into
// partial[blockIdx.x].  red holds kStoiThreads / 32 doubles.
__device__ __forceinline__ void stoi_block_sum(const StoiParams& p, double local, double* red) {
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = red[0];
    for (int w = 1; w < kStoiThreads / 32; ++w) t += red[w];
    p.partial[blockIdx.x] = t;
  }
}

// One CTA: kStoiSegBlock segments of one row.  The band energies of the block's frames are staged in shared memory;
// thread q takes the (segment, band) items q, q + 256, ... in order, and the CTA's sum is a fixed tree.
__global__ void __launch_bounds__(kStoiThreads) stoi_segment_kernel(StoiParams p) {
  constexpr int W = kStoiSegFrames;
  __shared__ double sx[kStoiBands * W], sy[kStoiBands * W];
  __shared__ double red[kStoiThreads / 32];
  const long long r = blockIdx.x / p.blocks;
  const int blk = (int)(blockIdx.x % p.blocks), seg0 = blk * kStoiSegBlock;
  const int J = (int)p.km[2 * r + 1] - kStoiSeg + 1;
  if (seg0 >= J) {
    if (threadIdx.x == 0) p.partial[blockIdx.x] = 0.0;
    return;
  }
  const int ns = min(kStoiSegBlock, J - seg0), nfr = ns + kStoiSeg - 1;
  stoi_stage_frames(p, r, seg0, nfr, sx, sy);
  __syncthreads();
  double local = 0.0;
  for (int q = threadIdx.x; q < ns * kStoiBands; q += blockDim.x) {
    const int j = q / kStoiBands, b = q - j * kStoiBands;
    const double* x = sx + b * W + j;
    const double* y = sy + b * W + j;
    double nx = 0.0, ny = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      nx = fma(x[k], x[k], nx);
      ny = fma(y[k], y[k], ny);
    }
    const double c = sqrt(nx) / (sqrt(ny) + kStoiEps);
    double my = 0.0, mx = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      my += np_min(y[k] * c, x[k] * kStoiClip);
      mx += x[k];
    }
    my /= kStoiSeg;
    mx /= kStoiSeg;
    double vy = 0.0, vx = 0.0, dot = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      const double a = np_min(y[k] * c, x[k] * kStoiClip) - my, e = x[k] - mx;
      vy = fma(a, a, vy);
      vx = fma(e, e, vx);
      dot = fma(a, e, dot);
    }
    local += dot / ((sqrt(vy) + kStoiEps) * (sqrt(vx) + kStoiEps));
  }
  stoi_block_sum(p, local, red);
}

// 1 / sqrt(s) of a centred sum of squares s, and 0 where s is zero up to rounding: at most 2^-92 = (64 eps)^2 times the
// sum of squares before centring, raw.  ESTOI without pystoi's N(0, eps^2) noise, whose expected contribution to such
// a row or column is zero: digital silence, and the columns of a segment with one non-zero frame, which are constant
// in exact arithmetic.  A NaN s fails the comparison and stays NaN.
constexpr double kEstoiTiny = 0x1p-92;
__device__ __forceinline__ double estoi_inv_norm(double s, double raw) {
  return s <= kEstoiTiny * raw ? 0.0 : 1.0 / sqrt(s);
}

// Dynamic shared memory of estoi_segment_kernel: the staged frames of x and y (15, kStoiSegFrames) and, per (segment,
// band) of the block, the row mean and inverse norm of x and y.  53 040 bytes: above the 48 KB static limit.
constexpr int kEstoiRows = kStoiSegBlock * kStoiBands;
constexpr size_t kEstoiSmemBytes = (2 * kStoiBands * kStoiSegFrames + 4 * kEstoiRows) * sizeof(double);

// One CTA: kStoiSegBlock segments of one row, the frames staged as in stoi_segment_kernel, so `partial` has the same
// layout.  Phase A: thread q takes the (segment, band) rows q, q + 256, ...: the mean over the 30 frames and the inverse
// root of the centred sum of squares, of x and of y.  Phase B: thread q takes the (segment, frame) columns q, q + 256,
// ...: the row-normalised column of x and of y over the 15 bands (recomputed from the staged frames and the phase-A
// scalars), its mean and inverse norm, and the inner product of the two normalised columns.  The CTA's sum is a fixed
// tree; the value kernel divides the row's total by 30 J.
__global__ void __launch_bounds__(kStoiThreads) estoi_segment_kernel(StoiParams p) {
  constexpr int W = kStoiSegFrames;
  extern __shared__ double smem[];
  double* sx = smem;
  double* sy = sx + kStoiBands * W;
  double* mx = sy + kStoiBands * W;  // (kStoiSegBlock, 15): row means and inverse norms of x and y
  double* ix = mx + kEstoiRows;
  double* my = ix + kEstoiRows;
  double* iy = my + kEstoiRows;
  __shared__ double red[kStoiThreads / 32];
  const long long r = blockIdx.x / p.blocks;
  const int blk = (int)(blockIdx.x % p.blocks), seg0 = blk * kStoiSegBlock;
  const int J = (int)p.km[2 * r + 1] - kStoiSeg + 1;
  if (seg0 >= J) {
    if (threadIdx.x == 0) p.partial[blockIdx.x] = 0.0;
    return;
  }
  const int ns = min(kStoiSegBlock, J - seg0), nfr = ns + kStoiSeg - 1;
  stoi_stage_frames(p, r, seg0, nfr, sx, sy);
  __syncthreads();
  for (int q = threadIdx.x; q < ns * kStoiBands; q += blockDim.x) {
    const int j = q / kStoiBands, b = q - j * kStoiBands;
    const double* x = sx + b * W + j;
    const double* y = sy + b * W + j;
    double ax = 0.0, ay = 0.0, rx = 0.0, ry = 0.0;
    // unrolled by 6, not fully: a full unroll holds the 60 staged values between the two passes in registers (155
    // per thread, one CTA per SM)
#pragma unroll 6
    for (int k = 0; k < kStoiSeg; ++k) {
      ax += x[k];
      ay += y[k];
      rx = fma(x[k], x[k], rx);
      ry = fma(y[k], y[k], ry);
    }
    ax /= kStoiSeg;
    ay /= kStoiSeg;
    double vx = 0.0, vy = 0.0;
#pragma unroll 6
    for (int k = 0; k < kStoiSeg; ++k) {
      const double e = x[k] - ax, a = y[k] - ay;
      vx = fma(e, e, vx);
      vy = fma(a, a, vy);
    }
    mx[q] = ax;
    ix[q] = estoi_inv_norm(vx, rx);
    my[q] = ay;
    iy[q] = estoi_inv_norm(vy, ry);
  }
  __syncthreads();
  double local = 0.0;
  for (int q = threadIdx.x; q < ns * kStoiSeg; q += blockDim.x) {
    const int j = q / kStoiSeg, n = q - j * kStoiSeg;
    const double* x = sx + j + n;
    const double* y = sy + j + n;
    const int s0 = j * kStoiBands;
    // the row-normalised values are recomputed from shared memory in the second pass rather than held in registers
    double cu = 0.0, cv = 0.0, ru = 0.0, rv = 0.0;
    for (int b = 0; b < kStoiBands; ++b) {
      const double e = (x[b * W] - mx[s0 + b]) * ix[s0 + b], a = (y[b * W] - my[s0 + b]) * iy[s0 + b];
      cu += e;
      cv += a;
      ru = fma(e, e, ru);
      rv = fma(a, a, rv);
    }
    cu /= kStoiBands;
    cv /= kStoiBands;
    double su = 0.0, sv = 0.0, dot = 0.0;
    for (int b = 0; b < kStoiBands; ++b) {
      const double e = (x[b * W] - mx[s0 + b]) * ix[s0 + b] - cu, a = (y[b * W] - my[s0 + b]) * iy[s0 + b] - cv;
      su = fma(e, e, su);
      sv = fma(a, a, sv);
      dot = fma(e, a, dot);
    }
    local += dot * estoi_inv_norm(su, ru) * estoi_inv_norm(sv, rv);
  }
  stoi_block_sum(p, local, red);
}

// One CTA for the group: the value of every row (block sums in order) and the status word.
__global__ void __launch_bounds__(kStoiThreads) stoi_value_kernel(StoiParams p) {
  __shared__ long long cnt[kStoiThreads], first[kStoiThreads];
  long long c = 0, fr = -1;
  for (long long r = threadIdx.x; r < p.rows; r += blockDim.x) {
    const long long M = p.km[2 * r + 1];
    double v;
    if (M < kStoiSeg) {
      v = 1e-5;
      ++c;
      if (fr < 0) fr = r;
    } else {
      const double* part = p.partial + r * p.blocks;
      double t = 0.0;
      for (int b = 0; b < p.blocks; ++b) t += part[b];
      v = t / (double)((M - kStoiSeg + 1) * p.terms);
    }
    p.out[r] = v;
  }
  cnt[threadIdx.x] = c;
  first[threadIdx.x] = fr;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long tc = 0, tf = -1;
    for (int t = 0; t < kStoiThreads; ++t) {
      tc += cnt[t];
      if (first[t] >= 0 && (tf < 0 || first[t] < tf)) tf = first[t];
    }
    p.status[0] += tc;
    if (p.status[1] < 0 && tf >= 0) p.status[1] = p.row0 + tf;
  }
}

}  // namespace pbb
