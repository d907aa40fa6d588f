// The shared-memory FFT stages (fp64) shared by the STFT kernels of fft.cuh and the global-memory FFT of
// fft_large.cuh: radix-4 Stockham stages, one radix-2 stage when log2 of the length is odd.  Twiddles come from a
// table tw[k] = (cos 2 pi k / S, sin 2 pi k / S), k < S, S twice the complex length.
#pragma once
#include "common.cuh"

namespace pbb {

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// DIR = -1: forward (exp(-i ...)), +1: inverse (unnormalised)
template <int DIR>
__device__ __forceinline__ void dft_r(double2 (&v)[2]) {
  const double2 a = v[0], b = v[1];
  v[0] = make_double2(a.x + b.x, a.y + b.y);
  v[1] = make_double2(a.x - b.x, a.y - b.y);
}
template <int DIR>
__device__ __forceinline__ void dft_r(double2 (&v)[4]) {
  const double2 s02 = make_double2(v[0].x + v[2].x, v[0].y + v[2].y);
  const double2 d02 = make_double2(v[0].x - v[2].x, v[0].y - v[2].y);
  const double2 s13 = make_double2(v[1].x + v[3].x, v[1].y + v[3].y);
  const double2 d13 = make_double2(v[1].x - v[3].x, v[1].y - v[3].y);
  v[0] = make_double2(s02.x + s13.x, s02.y + s13.y);
  v[2] = make_double2(s02.x - s13.x, s02.y - s13.y);
  if (DIR < 0) {  // X1 = d02 - i d13, X3 = d02 + i d13
    v[1] = make_double2(d02.x + d13.y, d02.y - d13.x);
    v[3] = make_double2(d02.x - d13.y, d02.y + d13.x);
  } else {
    v[1] = make_double2(d02.x - d13.y, d02.y + d13.x);
    v[3] = make_double2(d02.x + d13.y, d02.y - d13.x);
  }
}

// One radix-R Stockham stage of nfft transforms of M = 2^logM points, src -> dst; Ns = 2^logNs is the product of the
// earlier radices.  Butterfly j reads src[j + r M/R], twiddles by exp(DIR 2 pi i r (j mod Ns) / (Ns R)) and writes
// dst[(j - j mod Ns) R + j mod Ns + r Ns].
template <int R, int DIR>
__device__ __forceinline__ void fft_stage(const double2* __restrict__ src, double2* __restrict__ dst, int logM,
                                          int logNs, int nfft, const double2* __restrict__ tw) {
  constexpr int logR = R == 4 ? 2 : 1;
  const int lognb = logM - logR, nb = 1 << lognb, Ns = 1 << logNs;
  const int tshift = logM + 1 - logNs - logR;  // table index step 2M / (Ns R)
  for (int b = threadIdx.x; b < (nfft << lognb); b += blockDim.x) {
    const int f = b >> lognb, j = b & (nb - 1), jm = j & (Ns - 1);
    const double2* s = src + (f << logM) + j;
    double2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = s[r << lognb];
    const int step = jm << tshift;
#pragma unroll
    for (int r = 1; r < R; ++r) {
      double2 w = __ldg(tw + r * step);
      if (DIR < 0) w.y = -w.y;
      v[r] = cmul(v[r], w);
    }
    dft_r<DIR>(v);
    double2* d = dst + (f << logM) + (j - jm) * R + jm;
#pragma unroll
    for (int r = 0; r < R; ++r) d[r << logNs] = v[r];
  }
}

// All stages of nfft M-point transforms; the input is in a (written before a __syncthreads), b is scratch of the
// same size.  Returns the buffer that holds the result (visible to the whole CTA).
template <int DIR>
__device__ double2* fft_shared(double2* a, double2* b, int logM, int nfft, const double2* __restrict__ tw) {
  int logNs = 0;
  for (; logNs + 2 <= logM; logNs += 2) {
    fft_stage<4, DIR>(a, b, logM, logNs, nfft, tw);
    __syncthreads();
    double2* t = a; a = b; b = t;
  }
  if (logNs < logM) {
    fft_stage<2, DIR>(a, b, logM, logNs, nfft, tw);
    __syncthreads();
    a = b;
  }
  return a;
}

}  // namespace pbb
