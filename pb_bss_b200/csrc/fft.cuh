// Real FFTs of STFT frames in shared memory (fp64) for the transforms of pb_bss_b200/transform: a size-point real
// transform is one size/2-point complex transform of the even/odd-packed frame (radix-4 Stockham stages, one radix-2
// stage when log2(size/2) is odd) plus the real split step.  Twiddles come from a host-built table
// tw[k] = (cos 2 pi k / size, sin 2 pi k / size), k < size.
#pragma once
#include "common.cuh"
#include "fft_stages.cuh"

namespace pbb {

constexpr int kFftThreads = 256;
constexpr int kFftMinSize = 64, kFftMaxSize = 4096;
// frames per CTA: fpc * size <= kFftFrameBudget, i.e. two ping-pong buffers of fpc * size / 2 double2 = 64 KB
constexpr int kFftFrameBudget = 4096;

// ---- forward transform ----------------------------------------------------------------------------------------------
// STFT_ISTFT_BACKWARD: the gradient of the iSTFT wrt its spectrum, the STFT of the incoming gradient g (x = g,
// window = synthesis window, offset = crop) scaled to (2 / size) X_k for 0 < k < size/2 and (1 / size) X_k at k = 0 and
// size/2 (pbb_istft_backward)
enum { STFT_PLAIN = 0, STFT_GRIFFIN_LIM = 1, STFT_MISI = 2, STFT_ISTFT_BACKWARD = 3 };

struct StftParams {
  const void* x;        // (rows, n) real signal; MISI: x_hat (K, n) float64
  long long rows, n;
  int logM, shift, wl, offset, frames, fpc, tiles;  // offset = leading zeros of fading; tiles = CTAs per row
  const double* window;  // analysis window (wl)
  const double2* tw;     // size entries
  const double2* X;      // Griffin-Lim / MISI: the target spectrum (rows, frames, size/2 + 1) complex128
  const double* y;       // MISI: the mixture (n)
  double2* out;          // (rows, frames, size/2 + 1); Griffin-Lim: X_dash_dash
  double2* out_dash;     // Griffin-Lim: X_dash = |X| exp(i angle(X_dash_dash))
};

// One CTA: fpc consecutive frames of one row.  The sample span of those frames is loaded once into shared memory
// (zero outside [0, n): fading and end padding are never materialised), windowed and packed into M complex points per
// frame, transformed, split into M + 1 bins and written as contiguous rows.
template <class TI, int MODE>
__device__ __forceinline__ void stft_body(const StftParams& p) {
  extern __shared__ double2 smem[];
  const int M = 1 << p.logM, F = M + 1;
  const long long row = blockIdx.x / p.tiles;
  const int t0 = (int)(blockIdx.x % p.tiles) * p.fpc;
  const int nf = min(p.fpc, p.frames - t0);
  double2* A = smem;
  double2* B = smem + (p.fpc << p.logM);
  double* span = reinterpret_cast<double*>(B);  // dead once the frames are packed into A
  const int S = (nf - 1) * p.shift + p.wl;
  const long long s0 = (long long)t0 * p.shift - p.offset;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const long long s = s0 + i;
    double v = 0.0;
    if (s >= 0 && s < p.n) {
      if (MODE == STFT_MISI) {
        // x_hat + (y - sum_k x_hat) / K, the sum over k in row order (NumPy's axis-0 sum)
        const double* xh = static_cast<const double*>(p.x);
        double sum = xh[s];
        for (long long k = 1; k < p.rows; ++k) sum += xh[k * p.n + s];
        v = xh[row * p.n + s] + (__ldg(p.y + s) - sum) / (double)p.rows;
      } else {
        v = (double)static_cast<const TI*>(p.x)[row * p.n + s];
      }
    }
    span[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (nf << p.logM); i += blockDim.x) {
    const int f = i >> p.logM, j = 2 * (i & (M - 1));
    const double* fr = span + f * p.shift;
    const double re = j < p.wl ? fr[j] * __ldg(p.window + j) : 0.0;
    const double im = j + 1 < p.wl ? fr[j + 1] * __ldg(p.window + j + 1) : 0.0;
    A[i] = make_double2(re, im);
  }
  __syncthreads();
  const double2* Z = fft_shared<-1>(A, B, p.logM, nf, p.tw);
  const long long obase = (row * p.frames + t0) * F;
  for (int i = threadIdx.x; i < nf * F; i += blockDim.x) {
    const int f = i / F, k = i - f * F;
    const double2* z = Z + (f << p.logM);
    double2 X;
    if (k == 0 || k == M) {
      const double2 z0 = z[0];
      X = make_double2(k == 0 ? z0.x + z0.y : z0.x - z0.y, 0.0);
    } else {
      // X_k = (Z_k + conj Z_{M-k}) / 2 + W^k (Z_k - conj Z_{M-k}) / 2i,  W = exp(-2 pi i / size)
      const double2 a = z[k], b = z[M - k];
      const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
      const double2 fo = make_double2(0.5 * (a.y + b.y), -0.5 * (a.x - b.x));
      double2 w = __ldg(p.tw + k);
      w.y = -w.y;
      const double2 t = cmul(w, fo);
      X = make_double2(fe.x + t.x, fe.y + t.y);
    }
    if (MODE == STFT_ISTFT_BACKWARD) {
      // powers of two: exact
      const double sc = (k == 0 || k == M) ? 0.5 / M : 1.0 / M;
      X = make_double2(X.x * sc, X.y * sc);
    }
    p.out[obase + i] = X;
    if (MODE == STFT_GRIFFIN_LIM || MODE == STFT_MISI) {
      const double2 T = __ldg(p.X + obase + i);
      // exp(i angle(X)) as X / |X| (within rounding of cos / sin of atan2, without their reduction stack frame);
      // exp(i angle(0)) = 1
      const double mag = hypot(T.x, T.y), h = hypot(X.x, X.y);
      const double c = h > 0.0 ? X.x / h : 1.0, s = h > 0.0 ? X.y / h : 0.0;
      p.out_dash[obase + i] = make_double2(mag * c, mag * s);
    }
  }
}

template <class TI, int MODE>
__global__ void __launch_bounds__(kFftThreads) stft_kernel(StftParams p) { stft_body<TI, MODE>(p); }

__global__ void __launch_bounds__(kFftThreads) istft_backward_kernel(StftParams p) {
  stft_body<double, STFT_ISTFT_BACKWARD>(p);
}

// ---- inverse transform ----------------------------------------------------------------------------------------------
struct IstftParams {
  const double2* X;  // (rows, frames, size/2 + 1)
  long long rows;
  int logM, wl, frames, fpc, tiles;
  const double* synthesis;  // (wl)
  const double2* tw;
  double* framebuf;  // (rows, frames, wl): windowed frames
};

// ISTFT_PLAIN: irfft(X_t, n=size)[:wl] * synthesis window for fpc frames of one row.  The imaginary parts of the DC
// and Nyquist bins are ignored, as np.fft.irfft does.
// ISTFT_STFT_BACKWARD: the per-frame gradient of the STFT wrt its windowed frame, size irfft(G^)_j with G^_k = G_k / 2
// for 0 < k < size/2 and G^_k = G_k at k = 0 and size/2, times the analysis window (`synthesis` holds it), X = G
// (pbb_stft_backward)
enum { ISTFT_PLAIN = 0, ISTFT_STFT_BACKWARD = 1 };
template <int MODE>
__device__ __forceinline__ void istft_frames_body(const IstftParams& p) {
  extern __shared__ double2 smem[];
  const int M = 1 << p.logM, F = M + 1;
  const long long row = blockIdx.x / p.tiles;
  const int t0 = (int)(blockIdx.x % p.tiles) * p.fpc;
  const int nf = min(p.fpc, p.frames - t0);
  double2* A = smem;
  double2* B = smem + (p.fpc << p.logM);
  const double2* Xb = p.X + (row * p.frames + t0) * F;
  for (int i = threadIdx.x; i < (nf << p.logM); i += blockDim.x) {
    const int f = i >> p.logM, k = i & (M - 1);
    const double2* x = Xb + (long long)f * F;
    double2 Z;
    if (k == 0) {
      const double x0 = __ldg(&x[0].x), xm = __ldg(&x[M].x);
      Z = make_double2(0.5 * (x0 + xm), 0.5 * (x0 - xm));
    } else {
      // Fe = (X_k + conj X_{M-k}) / 2, Fo = (X_k - conj X_{M-k}) / 2 * conj W^k, Z_k = Fe + i Fo
      double2 a = __ldg(x + k), b = __ldg(x + M - k);
      if (MODE == ISTFT_STFT_BACKWARD) {
        a = make_double2(0.5 * a.x, 0.5 * a.y);
        b = make_double2(0.5 * b.x, 0.5 * b.y);
      }
      const double2 fe = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
      const double2 fo = cmul(make_double2(0.5 * (a.x - b.x), 0.5 * (a.y + b.y)), __ldg(p.tw + k));
      Z = make_double2(fe.x - fo.y, fe.y + fo.x);
    }
    A[i] = Z;
  }
  __syncthreads();
  const double2* z = fft_shared<1>(A, B, p.logM, nf, p.tw);
  const double m = (double)M;
  double* out = p.framebuf + (row * p.frames + t0) * p.wl;
  for (int i = threadIdx.x; i < nf * p.wl; i += blockDim.x) {
    const int f = i / p.wl, j = i - f * p.wl;
    const double2 v = z[(f << p.logM) + (j >> 1)];
    if (MODE == ISTFT_PLAIN) out[i] = __ldg(p.synthesis + j) * (((j & 1) ? v.y : v.x) / m);
    else out[i] = __ldg(p.synthesis + j) * (2.0 * ((j & 1) ? v.y : v.x));  // size irfft = 2 M (v / M)
  }
}

__global__ void __launch_bounds__(kFftThreads) istft_frames_kernel(IstftParams p) { istft_frames_body<ISTFT_PLAIN>(p); }

__global__ void __launch_bounds__(kFftThreads) stft_backward_kernel(IstftParams p) {
  istft_frames_body<ISTFT_STFT_BACKWARD>(p);
}

// out[r][m] = sum over the frames t covering sample m + crop of frame_t[m + crop - t shift], in increasing t from 0.0:
// the summation order of np.add.at, without atomics (bitwise reproducible).
__global__ void overlap_add_kernel(const double* __restrict__ frames, long long rows, int T, int wl, int shift,
                                   int crop, long long n_out, double* __restrict__ out) {
  const long long total = rows * n_out;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / n_out, m = i - r * n_out + crop;
    const long long lo = m >= wl ? (m - wl) / shift + 1 : 0;
    const long long hi = min((long long)T - 1, m / shift);
    const double* fr = frames + r * T * wl;
    double s = 0.0;
    for (long long t = lo; t <= hi; ++t) s += __ldg(fr + t * wl + (m - t * shift));
    out[i] = s;
  }
}

}  // namespace pbb
