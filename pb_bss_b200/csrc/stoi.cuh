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

// STFT frames t0 .. t0 + nf - 1 of signal s of row r, FFT'd in shared memory; returns the buffer of A, B that holds
// the 256-point transforms Z (the other one is free).  Sample j of STFT frame i of the overlap-added signal is the
// sum of the windowed kept frames i - 1 (second half) and i (j < 128), or i and i + 1 (first half, j >= 128): the
// two terms numpy's overlap-add adds, so the frame is bitwise numpy's before the FFT.
template <class T>
__device__ __forceinline__ const double2* stoi_frames_fft(const StoiParams& p, long long r, int s, int t0, int nf,
                                                          double2* A, double2* B) {
  constexpr int M = 1 << kStoiLogM;
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
  return fft_shared<-1>(A, B, kStoiLogM, nf, p.tw);
}

// Bin k (0 <= k <= 256) of the 512-point real FFT from the 256-point complex transform z of its even / odd samples.
__device__ __forceinline__ double2 stoi_bin(const double2* z, int k, const double2* tw) {
  constexpr int M = 1 << kStoiLogM;
  if (k == 0 || k == M) {
    const double2 z0 = z[0];
    return make_double2(k == 0 ? z0.x + z0.y : z0.x - z0.y, 0.0);
  }
  // X_k = (Z_k + conj Z_{M-k}) / 2 + W^k (Z_k - conj Z_{M-k}) / 2i,  W = exp(-2 pi i / 512)
  const double2 a = z[k], b = z[M - k];
  const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
  const double2 fo = make_double2(0.5 * (a.y + b.y), -0.5 * (a.x - b.x));
  double2 w = __ldg(tw + k);
  w.y = -w.y;
  const double2 t = cmul(w, fo);
  return make_double2(fe.x + t.x, fe.y + t.y);
}

// One CTA: kStoiFpc STFT frames of one (row, signal): the frames' FFTs (stoi_frames_fft), then the band energies.
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
  const double2* Z = stoi_frames_fft<T>(p, r, s, t0, nf, A, B);
  double* pw = reinterpret_cast<double*>(Z == A ? B : A);  // |X_k|^2, (nf, 257)
  for (int q = threadIdx.x; q < nf * kStoiBins; q += blockDim.x) {
    const int f = q / kStoiBins, k = q - f * kStoiBins;
    const double2 X = stoi_bin(Z + (f << kStoiLogM), k, p.tw);
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

// ---- backward (pbb_stoi_backward) ------------------------------------------------------------------------------------
// The forward's resample / energy / compact / bands kernels run again on the same StoiParams layout, so the keep mask,
// the kept-frame list and the band energies are bitwise the forward's.  Then, one kernel per adjoint step, every sum
// a gather in a fixed order (no atomics):
//   stoi_rank_kernel            frame -> rank among the kept frames (-1: dropped)
//   stoi_segment_prep_kernel    STOI: per (segment, band) the scalars of the correlation's adjoint
//   estoi_segment_prep_kernel   ESTOI: per (segment, band) and per (segment, frame) the normalisations' scalars
//   stoi_segment_grad_kernel /  per (band, frame) of the band energies: the sum over the <= 30 segments that hold it,
//   estoi_segment_grad_kernel   in increasing segment order, of x and y
//   stoi_spectral_grad_kernel   per STFT frame: G_k = (gbar_b / e_b) X_k, Re sum_k G_k e^{+2 pi i j k / 512} by a
//                               256-point inverse FFT, times the second window: the gradient of the STFT frame
//   stoi_removal_grad_kernel    per 10 kHz sample: the kept frames over it, the STFT frames over its overlap-added
//                               position, times the first window
//   stoi_resample_grad_kernel   per input sample: the transpose of the polyphase filter (skipped at 10 kHz)
struct StoiGrad {
  const double* gout;  // (rows) dvalue
  int Jmax;            // segments at most, Mmax - 29 (>= 1)
  int chains;          // bit 0: x, bit 1: y
  int* rank;           // (rows, F)
  double* tbar;        // (rows, 2, 15, Mmax) gradient of the band energies
  double* seg;         // (rows, fields, 15 | 30, Jmax) per-segment scalars
  double* fbar;        // (rows, 2, Mmax, 256) gradient of the STFT frames (before the second window is undone)
  double* sbar;        // (rows, 2, L) gradient of the 10 kHz signals (the resampler's output); unused at 10 kHz
  double* gx;          // (rows, n) or null
  double* gy;          // (rows, n) or null
};

constexpr int kStoiFields = 10;                 // STOI: per (segment, band)
constexpr int kEstoiRowFields = 8;              // ESTOI: per (segment, band)
constexpr int kEstoiColFields = 7;              // ESTOI: per (segment, frame), after the row fields
constexpr int kEstoiSegDoubles = kEstoiRowFields * kStoiBands + kEstoiColFields * kStoiSeg;

// value = sum / (J terms): the gradient of one segment's term
__device__ __forceinline__ double stoi_seg_scale(const StoiParams& p, const StoiGrad& q, long long r, int J) {
  return q.gout[r] / (double)((long long)J * p.terms);
}

__global__ void stoi_rank_kernel(StoiParams p, StoiGrad q) {
  const long long total = p.rows * p.F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / p.F;
    const int k = (int)(i - r * p.F);
    if (k < p.km[2 * r]) q.rank[r * p.F + p.kept[i]] = k;
  }
}

// STOI, per (segment j, band b) with x_k, y_k the 30 band energies, as stoi_segment_kernel computes them:
//   c = ||x|| / (||y|| + eps), y'_k = min(c y_k, C x_k) (the x term on a tie), a = y' - mean y', e = x - mean x,
//   d = <a, e> / ((||a|| + eps)(||e|| + eps)).
// With g = dvalue / (15 J):  abar_k = A1 e_k - A2 a_k, ebar_k = A1 a_k - E2 e_k, A1 = g / (Da De), A2 = g d / (Da ||a||),
// E2 = g d / (De ||e||) (0 for a zero norm), Da = ||a|| + eps, De = ||e|| + eps;  y'bar_k = abar_k - mean abar;
// cbar = sum_{k: y' took c y} y'bar_k y_k.  Then
//   xbar_k = ebar_k - mean ebar + [x term] C y'bar_k + cbar x_k / (||x|| (||y|| + eps)),
//   ybar_k = [y term] c y'bar_k - cbar ||x|| y_k / ((||y|| + eps)^2 ||y||)   (0 terms for a zero norm).
// Fields: c, mean x, mean y', A1, A2, E2, mean abar, mean ebar, cbar / (||x|| (||y|| + eps)), cbar ||x|| / (...).
__global__ void __launch_bounds__(kStoiThreads) stoi_segment_prep_kernel(StoiParams p, StoiGrad q) {
  constexpr int W = kStoiSegFrames;
  __shared__ double sx[kStoiBands * W], sy[kStoiBands * W];
  const long long r = blockIdx.x / p.blocks;
  const int blk = (int)(blockIdx.x % p.blocks), seg0 = blk * kStoiSegBlock;
  const int J = (int)p.km[2 * r + 1] - kStoiSeg + 1;
  if (seg0 >= J) return;
  const int ns = min(kStoiSegBlock, J - seg0), nfr = ns + kStoiSeg - 1;
  stoi_stage_frames(p, r, seg0, nfr, sx, sy);
  __syncthreads();
  const double g = stoi_seg_scale(p, q, r, J);
  for (int t = threadIdx.x; t < ns * kStoiBands; t += blockDim.x) {
    const int j = t / kStoiBands, b = t - j * kStoiBands;
    const double* x = sx + b * W + j;
    const double* y = sy + b * W + j;
    double nx = 0.0, ny = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      nx = fma(x[k], x[k], nx);
      ny = fma(y[k], y[k], ny);
    }
    const double Nx = sqrt(nx), Ny = sqrt(ny);
    const double c = Nx / (Ny + kStoiEps);
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
    const double Sa = sqrt(vy), Se = sqrt(vx), Da = Sa + kStoiEps, De = Se + kStoiEps;
    const double d = dot / (Da * De);
    const double A1 = g / (Da * De);
    const double A2 = Sa > 0.0 ? g * d / (Da * Sa) : 0.0;
    const double E2 = Se > 0.0 ? g * d / (De * Se) : 0.0;
    double sa = 0.0, se = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      const double a = np_min(y[k] * c, x[k] * kStoiClip) - my, e = x[k] - mx;
      sa += A1 * e - A2 * a;
      se += A1 * a - E2 * e;
    }
    const double ma = sa / kStoiSeg, me = se / kStoiSeg;
    double cbar = 0.0;
    for (int k = 0; k < kStoiSeg; ++k) {
      const double u = y[k] * c, v = x[k] * kStoiClip;
      if (u < v || u != u) {
        const double e = x[k] - mx, a = u - my;
        cbar += (A1 * e - A2 * a - ma) * y[k];
      }
    }
    const double Dy = Ny + kStoiEps;
    const double f[kStoiFields] = {c, mx, my, A1, A2, E2, ma, me, Nx > 0.0 ? cbar / (Nx * Dy) : 0.0,
                                   Ny > 0.0 ? cbar * Nx / (Dy * Dy * Ny) : 0.0};
    double* o = q.seg + ((r * kStoiFields) * kStoiBands + b) * q.Jmax + seg0 + j;
#pragma unroll
    for (int i = 0; i < kStoiFields; ++i) o[(long long)i * kStoiBands * q.Jmax] = f[i];
  }
}

// One thread per (row, band, frame m) of the band energies: xbar, ybar summed over the segments j = m - k that hold
// frame m, in increasing j; zero for rows on the 1e-5 path and frames from M_r on.
__global__ void __launch_bounds__(kStoiThreads) stoi_segment_grad_kernel(StoiParams p, StoiGrad q) {
  const long long total = p.rows * kStoiBands * (long long)p.Mmax;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long rb = i / p.Mmax, r = rb / kStoiBands;
    const int m = (int)(i - rb * p.Mmax), b = (int)(rb - r * kStoiBands);
    const int Mr = (int)p.km[2 * r + 1], J = Mr - kStoiSeg + 1;
    double gxs = 0.0, gys = 0.0;
    if (J > 0 && m < Mr) {
      const double x = p.tob[(2 * r * kStoiBands + b) * p.Mmax + m];
      const double y = p.tob[((2 * r + 1) * kStoiBands + b) * p.Mmax + m];
      const double* f = q.seg + ((r * kStoiFields) * kStoiBands + b) * q.Jmax;
      const long long fs = (long long)kStoiBands * q.Jmax;
      for (int k = min(kStoiSeg - 1, m); k >= 0 && m - k < J; --k) {
        const int j = m - k;
        const double c = f[j], mx = f[fs + j], my = f[2 * fs + j], A1 = f[3 * fs + j], A2 = f[4 * fs + j],
                     E2 = f[5 * fs + j], ma = f[6 * fs + j], me = f[7 * fs + j], cx = f[8 * fs + j],
                     cy = f[9 * fs + j];
        const double u = y * c, v = x * kStoiClip;
        const bool ysel = u < v || u != u;
        const double a = (ysel ? u : v) - my, e = x - mx;
        const double ybar = A1 * e - A2 * a - ma;
        gxs += (A1 * a - E2 * e - me) + (ysel ? 0.0 : kStoiClip * ybar) + cx * x;
        gys += (ysel ? c * ybar : 0.0) - cy * y;
      }
    }
    q.tbar[(2 * r * kStoiBands + b) * p.Mmax + m] = gxs;
    q.tbar[((2 * r + 1) * kStoiBands + b) * p.Mmax + m] = gys;
  }
}

// ESTOI, per segment with X, Y (15 bands b x 30 frames n), as estoi_segment_kernel computes them:
//   row step   r_bn = (x_bn - mu_b) inv_b,  inv_b = 1 / ||x_b - mu_b|| (0 by the 2^-92 rule)
//   column     z_bn = (r_bn - nu_n) iv_n,   iv_n = 1 / ||r_n - nu_n||  (0 by the 2^-92 rule)
//   d = sum_bn z_bn z'_bn (primes: Y), g = dvalue / (30 J), D_n = sum_b z_bn z'_bn.
// Adjoint, for X (swap the roles for Y):  wbar_bn = g iv_n (z'_bn - z_bn D_n), rbar_bn = wbar_bn - mean_b wbar_bn,
// rho_b = sum_n r_bn rbar_bn, ubar_bn = inv_b (rbar_bn - r_bn rho_b), xbar_bn = ubar_bn - mean_n ubar_bn.  A zero inv or
// iv passes no gradient, as the constant zeros it normalises to.
// Row fields (segment, band): mu, inv of x and y, rho of x and y, mean_n ubar of x and y.
// Column fields (segment, frame): nu, iv of x and y, D, mean_b wbar of x and y.
__device__ __forceinline__ double* estoi_row_field(const StoiGrad& q, long long r, int i, int b) {
  return q.seg + ((r * kEstoiSegDoubles) + i * kStoiBands + b) * q.Jmax;
}
__device__ __forceinline__ double* estoi_col_field(const StoiGrad& q, long long r, int i, int n) {
  return q.seg + ((r * kEstoiSegDoubles) + kEstoiRowFields * kStoiBands + i * kStoiSeg + n) * q.Jmax;
}

// One CTA: kStoiSegBlock segments of one row, the frames staged as in estoi_segment_kernel.  Phase A per (segment,
// band) row: the forward's mean and inverse norm.  Phase B per (segment, frame) column: the forward's nu, iv, then D
// and the means of wbar.  Phase C per row: rho and the mean of ubar.  Scalars go to the workspace, which phases B and C
// read back after the CTA barrier.
__global__ void __launch_bounds__(kStoiThreads) estoi_segment_prep_kernel(StoiParams p, StoiGrad q) {
  constexpr int W = kStoiSegFrames;
  extern __shared__ double smem[];
  double* sx = smem;
  double* sy = sx + kStoiBands * W;
  double* mx = sy + kStoiBands * W;  // (kStoiSegBlock, 15)
  double* ix = mx + kEstoiRows;
  double* my = ix + kEstoiRows;
  double* iy = my + kEstoiRows;
  const long long r = blockIdx.x / p.blocks;
  const int blk = (int)(blockIdx.x % p.blocks), seg0 = blk * kStoiSegBlock;
  const int J = (int)p.km[2 * r + 1] - kStoiSeg + 1;
  if (seg0 >= J) return;
  const int ns = min(kStoiSegBlock, J - seg0), nfr = ns + kStoiSeg - 1;
  stoi_stage_frames(p, r, seg0, nfr, sx, sy);
  __syncthreads();
  const double g = stoi_seg_scale(p, q, r, J);
  for (int t = threadIdx.x; t < ns * kStoiBands; t += blockDim.x) {
    const int j = t / kStoiBands, b = t - j * kStoiBands;
    const double* x = sx + b * W + j;
    const double* y = sy + b * W + j;
    double ax = 0.0, ay = 0.0, rx = 0.0, ry = 0.0;
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
    mx[t] = ax;
    ix[t] = estoi_inv_norm(vx, rx);
    my[t] = ay;
    iy[t] = estoi_inv_norm(vy, ry);
    const int js = seg0 + j;
    estoi_row_field(q, r, 0, b)[js] = ax;
    estoi_row_field(q, r, 1, b)[js] = ix[t];
    estoi_row_field(q, r, 2, b)[js] = ay;
    estoi_row_field(q, r, 3, b)[js] = iy[t];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < ns * kStoiSeg; t += blockDim.x) {
    const int j = t / kStoiSeg, n = t - j * kStoiSeg;
    const double* x = sx + j + n;
    const double* y = sy + j + n;
    const int s0 = j * kStoiBands;
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
    const double iu = estoi_inv_norm(su, ru), iv = estoi_inv_norm(sv, rv);
    const double D = dot * iu * iv;
    double wx = 0.0, wy = 0.0;
    for (int b = 0; b < kStoiBands; ++b) {
      const double z = ((x[b * W] - mx[s0 + b]) * ix[s0 + b] - cu) * iu;
      const double zp = ((y[b * W] - my[s0 + b]) * iy[s0 + b] - cv) * iv;
      wx += g * iu * (zp - z * D);
      wy += g * iv * (z - zp * D);
    }
    const int js = seg0 + j;
    estoi_col_field(q, r, 0, n)[js] = cu;
    estoi_col_field(q, r, 1, n)[js] = iu;
    estoi_col_field(q, r, 2, n)[js] = cv;
    estoi_col_field(q, r, 3, n)[js] = iv;
    estoi_col_field(q, r, 4, n)[js] = D;
    estoi_col_field(q, r, 5, n)[js] = wx / kStoiBands;
    estoi_col_field(q, r, 6, n)[js] = wy / kStoiBands;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < ns * kStoiBands; t += blockDim.x) {
    const int j = t / kStoiBands, b = t - j * kStoiBands, js = seg0 + j;
    const double* x = sx + b * W + j;
    const double* y = sy + b * W + j;
    double rhox = 0.0, rhoy = 0.0;
    for (int pass = 0; pass < 2; ++pass) {
      double ux = 0.0, uy = 0.0;
      for (int n = 0; n < kStoiSeg; ++n) {
        const double cu = estoi_col_field(q, r, 0, n)[js], iu = estoi_col_field(q, r, 1, n)[js];
        const double cv = estoi_col_field(q, r, 2, n)[js], iv = estoi_col_field(q, r, 3, n)[js];
        const double D = estoi_col_field(q, r, 4, n)[js];
        const double rx = (x[n] - mx[t]) * ix[t], ry = (y[n] - my[t]) * iy[t];
        const double z = (rx - cu) * iu, zp = (ry - cv) * iv;
        const double rbx = g * iu * (zp - z * D) - estoi_col_field(q, r, 5, n)[js];
        const double rby = g * iv * (z - zp * D) - estoi_col_field(q, r, 6, n)[js];
        if (pass == 0) {
          rhox = fma(rx, rbx, rhox);
          rhoy = fma(ry, rby, rhoy);
        } else {
          ux += ix[t] * (rbx - rx * rhox);
          uy += iy[t] * (rby - ry * rhoy);
        }
      }
      if (pass == 1) {
        estoi_row_field(q, r, 4, b)[js] = rhox;
        estoi_row_field(q, r, 5, b)[js] = rhoy;
        estoi_row_field(q, r, 6, b)[js] = ux / kStoiSeg;
        estoi_row_field(q, r, 7, b)[js] = uy / kStoiSeg;
      }
    }
  }
}

// stoi_segment_grad_kernel's gather for ESTOI.
__global__ void __launch_bounds__(kStoiThreads) estoi_segment_grad_kernel(StoiParams p, StoiGrad q) {
  const long long total = p.rows * kStoiBands * (long long)p.Mmax;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long rb = i / p.Mmax, r = rb / kStoiBands;
    const int m = (int)(i - rb * p.Mmax), b = (int)(rb - r * kStoiBands);
    const int Mr = (int)p.km[2 * r + 1], J = Mr - kStoiSeg + 1;
    double gxs = 0.0, gys = 0.0;
    if (J > 0 && m < Mr) {
      const double x = p.tob[(2 * r * kStoiBands + b) * p.Mmax + m];
      const double y = p.tob[((2 * r + 1) * kStoiBands + b) * p.Mmax + m];
      const double g = stoi_seg_scale(p, q, r, J);
      const double *mux = estoi_row_field(q, r, 0, b), *inx = estoi_row_field(q, r, 1, b);
      const double *muy = estoi_row_field(q, r, 2, b), *iny = estoi_row_field(q, r, 3, b);
      const double *rhx = estoi_row_field(q, r, 4, b), *rhy = estoi_row_field(q, r, 5, b);
      const double *mux_ = estoi_row_field(q, r, 6, b), *muy_ = estoi_row_field(q, r, 7, b);
      for (int n = min(kStoiSeg - 1, m); n >= 0 && m - n < J; --n) {
        const int j = m - n;
        const double cu = estoi_col_field(q, r, 0, n)[j], iu = estoi_col_field(q, r, 1, n)[j];
        const double cv = estoi_col_field(q, r, 2, n)[j], iv = estoi_col_field(q, r, 3, n)[j];
        const double D = estoi_col_field(q, r, 4, n)[j];
        const double rx = (x - mux[j]) * inx[j], ry = (y - muy[j]) * iny[j];
        const double z = (rx - cu) * iu, zp = (ry - cv) * iv;
        const double rbx = g * iu * (zp - z * D) - estoi_col_field(q, r, 5, n)[j];
        const double rby = g * iv * (z - zp * D) - estoi_col_field(q, r, 6, n)[j];
        gxs += inx[j] * (rbx - rx * rhx[j]) - mux_[j];
        gys += iny[j] * (rby - ry * rhy[j]) - muy_[j];
      }
    }
    q.tbar[(2 * r * kStoiBands + b) * p.Mmax + m] = gxs;
    q.tbar[((2 * r + 1) * kStoiBands + b) * p.Mmax + m] = gys;
  }
}

// One CTA: kStoiFpc STFT frames of one (row, signal), as stoi_bands_kernel.  With the forward's transform Z of the
// frames and e_b their band energies (tob), G_k = (tbar_b / e_b) X_k in band b (0 outside the bands and where e_b = 0)
// is packed as istft_frames_body<ISTFT_STFT_BACKWARD> packs it (inner bins halved), so 2 Re of the 256-point inverse
// FFT is Re sum_{k=0}^{256} G_k e^{+2 pi i j k / 512}, the gradient of the frame before the rfft; times the second
// window, the gradient of STFT frame i of the overlap-added signal (j < 256).
template <class T>
__global__ void __launch_bounds__(kStoiThreads) stoi_spectral_grad_kernel(StoiParams p, StoiGrad q) {
  constexpr int M = 1 << kStoiLogM;
  __shared__ double2 A[kStoiFpc * M], B[kStoiFpc * M];
  __shared__ double coef[kStoiFpc * kStoiBands];
  __shared__ int edge[2 * kStoiBands];
  const int tiles = (p.Mmax + kStoiFpc - 1) / kStoiFpc;
  const long long rs = blockIdx.x / tiles, r = rs >> 1;
  const int s = (int)(rs & 1);
  if (!(q.chains >> s & 1)) return;
  const int t0 = (int)(blockIdx.x % tiles) * kStoiFpc;
  const int Mr = (int)p.km[2 * r + 1];
  if (Mr < kStoiSeg || t0 >= Mr) return;
  const int nf = min(kStoiFpc, Mr - t0);
  if (threadIdx.x < 2 * kStoiBands) edge[threadIdx.x] = __ldg(p.bands + threadIdx.x);
  if (threadIdx.x < nf * kStoiBands) {
    const int f = threadIdx.x / kStoiBands, b = threadIdx.x - f * kStoiBands;
    const long long o = (rs * kStoiBands + b) * p.Mmax + t0 + f;
    const double e = p.tob[o];
    coef[threadIdx.x] = e == 0.0 ? 0.0 : q.tbar[o] / e;
  }
  const double2* Z = stoi_frames_fft<T>(p, r, s, t0, nf, A, B);  // its barriers publish coef and edge
  double2* P = const_cast<double2*>(Z == A ? B : A);
  auto weight = [&](int f, int k) {
    for (int b = 0; b < kStoiBands; ++b)
      if (edge[2 * b] <= k && k < edge[2 * b + 1]) return coef[f * kStoiBands + b];
    return 0.0;
  };
  for (int t = threadIdx.x; t < (nf << kStoiLogM); t += blockDim.x) {
    const int f = t >> kStoiLogM, k = t & (M - 1);
    const double2* z = Z + (f << kStoiLogM);
    double2 a = stoi_bin(z, k, p.tw), b = stoi_bin(z, k == 0 ? M : M - k, p.tw);
    const double wa = weight(f, k), wb = weight(f, k == 0 ? M : M - k);
    a = make_double2(wa * a.x, wa * a.y);
    b = make_double2(wb * b.x, wb * b.y);
    double2 Zp;
    if (k == 0) {
      Zp = make_double2(0.5 * (a.x + b.x), 0.5 * (a.x - b.x));
    } else {
      a = make_double2(0.5 * a.x, 0.5 * a.y);
      b = make_double2(0.5 * b.x, 0.5 * b.y);
      const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
      const double2 fo = cmul(make_double2(0.5 * (a.x - b.x), 0.5 * (a.y + b.y)), __ldg(p.tw + k));
      Zp = make_double2(fe.x - fo.y, fe.y + fo.x);
    }
    P[t] = Zp;
  }
  __syncthreads();
  const double2* z = fft_shared<1>(P, const_cast<double2*>(Z), kStoiLogM, nf, p.tw);
  double* out = q.fbar + (rs * p.Mmax + t0) * kStoiFrame;
  for (int t = threadIdx.x; t < nf * kStoiFrame; t += blockDim.x) {
    const int f = t / kStoiFrame, j = t - f * kStoiFrame;
    const double2 v = z[(f << kStoiLogM) + (j >> 1)];
    out[t] = __ldg(p.window + j) * (2.0 * ((j & 1) ? v.y : v.x));
  }
}

// One thread per 10 kHz sample i of one (row, signal): the kept frames f in {i / 128 - 1, i / 128} over it, each at
// its rank k in the overlap-added signal, position 128 k + (i - 128 f); there the STFT frames over that position in
// increasing order; times w[i - 128 f].  Rows on the 1e-5 path get zeros.  At 10 kHz the result is the input's
// gradient (rows, n); else the resampler's output gradient sbar (rows, 2, L).
__global__ void __launch_bounds__(kStoiThreads) stoi_removal_grad_kernel(StoiParams p, StoiGrad q) {
  const long long total = p.rows * 2 * p.L;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long rs = i / p.L, smp = i - rs * p.L, r = rs >> 1;
    const int s = (int)(rs & 1);
    if (!(q.chains >> s & 1)) continue;
    const int Mr = (int)p.km[2 * r + 1];
    double acc = 0.0;
    if (Mr >= kStoiSeg) {
      const long long fq = smp / kStoiHop;
      for (long long f = fq - 1; f <= fq; ++f) {
        if (f < 0 || f >= p.F) continue;
        const int k = q.rank[r * p.F + f];
        if (k < 0) continue;
        const int t = (int)(smp - f * kStoiHop);
        const long long pos = (long long)k * kStoiHop + t, i1 = pos / kStoiHop;
        const double* fb = q.fbar + rs * p.Mmax * kStoiFrame;
        double zb = 0.0;
        if (i1 >= 1 && i1 - 1 < Mr) zb += fb[(i1 - 1) * kStoiFrame + (pos - (i1 - 1) * kStoiHop)];
        if (i1 < Mr) zb += fb[i1 * kStoiFrame + (pos - i1 * kStoiHop)];
        acc = fma(__ldg(p.window + t), zb, acc);
      }
    }
    if (p.sig) q.sbar[i] = acc;
    else (s ? q.gy : q.gx)[r * p.n + smp] = acc;
  }
}

// One thread per input sample i of one (row, signal): the transpose of stoi_resample_kernel, the outputs j whose tap
// index (j + pre_remove) down - i up lies in [0, up tpp), in increasing j.
__global__ void __launch_bounds__(kStoiThreads) stoi_resample_grad_kernel(StoiParams p, StoiGrad q) {
  const long long total = p.rows * 2 * p.n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long rs = i / p.n, smp = i - rs * p.n, r = rs >> 1;
    const int s = (int)(rs & 1);
    if (!(q.chains >> s & 1)) continue;
    const double* sb = q.sbar + rs * p.L;
    const long long lo = smp * p.up, span = (long long)p.up * p.tpp;
    long long j0 = (lo + p.down - 1) / p.down - p.pre_remove;
    if (j0 < 0) j0 = 0;
    long long j1 = (lo + span + p.down - 1) / p.down - p.pre_remove;
    if (j1 > p.L) j1 = p.L;
    double acc = 0.0;
    for (long long j = j0; j < j1; ++j) {
      const long long t = (j + p.pre_remove) * p.down - lo;
      acc = fma(__ldg(p.taps + (t % p.up) * p.tpp + t / p.up), sb[j], acc);
    }
    (s ? q.gy : q.gx)[r * p.n + smp] = acc;
  }
}

}  // namespace pbb
