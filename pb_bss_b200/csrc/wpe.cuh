// WPE dereverberation (nara_wpe.wpe.wpe_v8, get_power, get_power_inverse, build_y_tilde) -- see include/pbb.h.
//
// Per bin (one (D, T) problem), n = taps D <= PBB_WPE_MAX_N, and per iteration:
//   1. wpe_corr_kernel: the real Gram matrix S S^T of the weighted statistics on fp64 m8n8k4 mma.sync.  S has
//      M = 2 (n + D) rows: the real parts of the n rows of Yt (row k D + d at frame t is Y_{d, t - delay - k}) and of
//      the D rows of Y, then their imaginary parts.  The complex Gram C = E E^H of E = [Yt; Y] is
//      (S_re S_re^T + S_im S_im^T) + i (S_im S_re^T - S_re S_im^T), and its blocks are R (n x n) and P (n x D).  Only
//      the lower triangle of 8 x 8 tiles is accumulated; it holds every entry of R and P.  Yt is never stored: a
//      chunk of kWpeChunk frames of Y plus the taps - 1 halo frames of the delayed window is staged in shared memory
//      and every row of S is an offset into it.  The weight enters once per frame and product: the column operand
//      of each mma is w_t S[j][t], the row operand is S[i][t] unweighted.  Long T splits the frames over `parts`
//      CTAs (a function of T only); each writes its own partial tiles.
//   2. wpe_solve_kernel: one CTA per bin sums the partials in part order, assembles R and P in shared memory and
//      solves R G = P by LU with partial pivoting (LAPACK's izamax pivot, |re| + |im|, first maximum), the
//      arithmetic of solve_kernel (linalg_kernels.cuh) for n up to 96.  A bin whose pivot is exactly zero (where
//      np.linalg.solve raises) is flagged; wpe_lstsq_kernel gives it the minimum-norm solution of np.linalg.lstsq
//      through the Hermitian eigendecomposition of R (warp_jacobi), eigenvalues at most eps n max|lambda| counted as
//      zero, the eigenvectors kept in the bin's (then unused) partial tiles in global memory.
//   3. wpe_filter_kernel: X = Y - G^H Yt, and in the same pass the next iteration's lambda_t = mean_d |X_dt|^2, its
//      psd_context mean and the per-bin max, giving w_t = 1 / max(lambda_t, 1e-10 max lambda).  X itself is only
//      stored by the last iteration (in the output's dtype and strides); the statistics of the next iteration need
//      Y and w only.  The first w comes from the same kernel with G = 0 (X = Y exactly).
//   4. the backward passes of a step (pbb_wpe_backward: R again by wpe_corr_kernel, wpe_gbar_kernel,
//      wpe_solve_rhs_kernel, wpe_step_backward_kernel) and of the power chain (wpe_power_backward_kernel,
//      wpe_power_inverse_backward_kernel); the closed forms are in include/pbb.h.
// Every sum runs in a fixed order and there are no float atomics: repeated calls are bitwise identical.  Status
// bits (PBB_WPE_NONFINITE, PBB_WPE_LSTSQ) are set on the device and read by the caller after the last iteration.
#pragma once
#include <math_constants.h>

#include "common.cuh"
#include "heig.cuh"
#include "cplx.cuh"

namespace pbb {

constexpr int kWpeMaxN = PBB_WPE_MAX_N;      // 96
constexpr int kWpeChunk = 64;                // frames per staged chunk of wpe_corr_kernel
constexpr int kWpeCorrWarps = 16;
constexpr int kWpePartFrames = 1024;         // frames per part of wpe_corr_kernel (at most kWpeMaxParts parts)
constexpr int kWpeMaxParts = 64;
constexpr int kWpeFilterChunk = 128;         // frames per staged chunk of wpe_filter_kernel

struct WpeShape {
  long long T;
  int D, taps, delay, n;
  int N2, T8, ntiles;   // n + D complex rows, 8-row blocks of the 2 N2 real rows, lower-triangle tiles
  int parts;            // frame parts of wpe_corr_kernel
  long long tb, span;   // first frame of the statistics ('valid': delay + taps - 1), frames per part
  long long psd_context;  // < 0: inf
};

// element strides of a (bins, D, T) operand
struct WpeStrides {
  long long b, d, t;
};

__device__ __forceinline__ double2 wpe_load(const double2* p, long long i) { return p[i]; }
__device__ __forceinline__ double2 wpe_load(const float2* p, long long i) {
  const float2 v = p[i];
  return make_double2(v.x, v.y);
}
__device__ __forceinline__ void wpe_store(double2* p, long long i, double2 v) { p[i] = v; }
__device__ __forceinline__ void wpe_store(float2* p, long long i, double2 v) {
  p[i] = make_float2((float)v.x, (float)v.y);
}

__device__ __forceinline__ void wpe_dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

// ---- 1. weighted statistics -------------------------------------------------------------------------------------
// Shared layout (doubles): [0, kWpeChunk) zeros (padding rows), then per part (re, im) and channel d the delayed
// window (kWpeChunk + taps - 1 frames from t0 - delay - taps + 1), then per part and channel the current window
// (kWpeChunk frames from t0).
__device__ __forceinline__ int wpe_row_offset(const WpeShape& s, int e) {
  const int lw = kWpeChunk + s.taps - 1;
  if (e >= 2 * s.N2) return 0;
  const int part = e >= s.N2, ee = e - part * s.N2;
  if (ee < s.n) {
    const int k = ee / s.D, d = ee - k * s.D;
    return kWpeChunk + (part * s.D + d) * lw + s.taps - 1 - k;
  }
  return kWpeChunk + 2 * s.D * lw + (part * s.D + ee - s.n) * kWpeChunk;
}

__host__ __device__ inline int wpe_corr_smem_doubles(int D, int taps) {
  return kWpeChunk + 2 * D * (kWpeChunk + taps - 1) + 2 * D * kWpeChunk + kWpeChunk;  // + the chunk's weights
}

// lower-triangle tile index -> (I, J), J <= I
__device__ __forceinline__ void wpe_tile(int t, int& I, int& J) {
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((i + 1) * (i + 2) / 2 <= t) ++i;
  while (i * (i + 1) / 2 > t) --i;
  I = i;
  J = t - i * (i + 1) / 2;
}

// grid (parts, bins, passes), kWpeCorrWarps warps; pass z covers tiles [16 TPW z, 16 TPW (z + 1)), warp v of it the
// tiles 16 TPW z + v + 16 i (i < TPW slots).  Shapes with more tiles than one pass holds run several passes, each
// staging the frames again.  part (bins, parts, ntiles, 64): tile element (r, c) at r * 8 + c.
template <int TPW, class TIn>
__global__ void __launch_bounds__(32 * kWpeCorrWarps) wpe_corr_kernel(const TIn* __restrict__ y, WpeStrides ys,
                                                                     WpeShape s, const double* __restrict__ w,
                                                                     double* __restrict__ part) {
  extern __shared__ __align__(16) double wsm[];
  const int p = blockIdx.x;
  const long long bin = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, q = lane & 3;
  const int lw = kWpeChunk + s.taps - 1;
  const int tile0 = blockIdx.z * kWpeCorrWarps * TPW + warp;
  double* wch = wsm + wpe_corr_smem_doubles(s.D, s.taps) - kWpeChunk;
  // per slot: the lane's row-operand and column-operand offsets, packed 16 + 16 bits
  unsigned offs[TPW];
  double acc[TPW][2];
#pragma unroll
  for (int i = 0; i < TPW; ++i) {
    const int t = tile0 + kWpeCorrWarps * i;
    int I = 0, J = 0;
    if (t < s.ntiles) wpe_tile(t, I, J);
    offs[i] = (unsigned)wpe_row_offset(s, 8 * I + r) | (unsigned)wpe_row_offset(s, 8 * J + r) << 16;
    acc[i][0] = acc[i][1] = 0.0;
  }
  for (int i = threadIdx.x; i < kWpeChunk; i += blockDim.x) wsm[i] = 0.0;
  const TIn* yb = y + bin * ys.b;
  const double* wb = w + bin * s.T;
  const long long f0 = s.tb + p * s.span, f1 = min(s.T, f0 + s.span);
  for (long long t0 = f0; t0 < f1; t0 += kWpeChunk) {
    __syncthreads();
    const long long ws = t0 - s.delay - s.taps + 1;
    for (int i = threadIdx.x; i < s.D * lw; i += blockDim.x) {
      const int d = i / lw, j = i - d * lw;
      const long long f = ws + j;
      const double2 v = f >= 0 && f < s.T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
      wsm[kWpeChunk + d * lw + j] = v.x;
      wsm[kWpeChunk + (s.D + d) * lw + j] = v.y;
    }
    for (int i = threadIdx.x; i < s.D * kWpeChunk; i += blockDim.x) {
      const int d = i / kWpeChunk, j = i - d * kWpeChunk;
      const long long f = t0 + j;
      const double2 v = f < f1 ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
      wsm[kWpeChunk + 2 * s.D * lw + d * kWpeChunk + j] = v.x;
      wsm[kWpeChunk + 2 * s.D * lw + (s.D + d) * kWpeChunk + j] = v.y;
    }
    for (int j = threadIdx.x; j < kWpeChunk; j += blockDim.x) wch[j] = t0 + j < f1 ? wb[t0 + j] : 0.0;
    __syncthreads();
#pragma unroll 2
    for (int k = 0; k < kWpeChunk; k += 4) {
      const double wv = wch[k + q];
#pragma unroll
      for (int i = 0; i < TPW; ++i) {
        if (tile0 + kWpeCorrWarps * i < s.ntiles) {
          const double a = wsm[(offs[i] & 0xffffu) + k + q];
          const double b = wsm[(offs[i] >> 16) + k + q] * wv;
          wpe_dmma(acc[i], a, b);
        }
      }
    }
  }
  double* out = part + (bin * s.parts + p) * (long long)s.ntiles * 64;
#pragma unroll
  for (int i = 0; i < TPW; ++i) {
    const int t = tile0 + kWpeCorrWarps * i;
    if (t < s.ntiles) {
      out[t * 64 + r * 8 + 2 * q] = acc[i][0];
      out[t * 64 + r * 8 + 2 * q + 1] = acc[i][1];
    }
  }
}

// entry (a, b) of the real Gram matrix of one bin, summed over the parts in order
__device__ __forceinline__ double wpe_gram(const double* __restrict__ pb, const WpeShape& s, int a, int b) {
  if (a < b) { const int t = a; a = b; b = t; }
  const int I = a >> 3, J = b >> 3;
  const long long off = (long long)(I * (I + 1) / 2 + J) * 64 + (a & 7) * 8 + (b & 7);
  const long long per = (long long)s.ntiles * 64;
  double v = 0.0;
  for (int p = 0; p < s.parts; ++p) v += pb[p * per + off];
  return v;
}

// C[i][j] of E E^H (i, j < n + D)
__device__ __forceinline__ double2 wpe_complex(const double* __restrict__ pb, const WpeShape& s, int i, int j) {
  const double rr = wpe_gram(pb, s, i, j), ii = wpe_gram(pb, s, s.N2 + i, s.N2 + j);
  const double ir = wpe_gram(pb, s, s.N2 + i, j), ri = wpe_gram(pb, s, i, s.N2 + j);
  return make_double2(rr + ii, ir - ri);
}

// ---- 2. the per-bin solve ---------------------------------------------------------------------------------------
__host__ __device__ inline size_t wpe_solve_smem_bytes(int n, int D) {
  return ((size_t)n * n + (size_t)n * D + n) * sizeof(double2) + 64 * sizeof(double);
}

__device__ __forceinline__ double wpe_block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) v = fmax(v, red[i]);
  return v;
}

// LU with partial pivoting of A (n x n, shared) applied to the right-hand sides X (n x D, shared); f: n scratch.
// state on entry: 0, or non-zero to skip the elimination.  Returns 1 on an exactly zero pivot (A, X then partly
// eliminated), else the entry state.  Every thread of the CTA calls it.
__device__ __forceinline__ int wpe_lu_eliminate(double2* A, double2* X, double2* f, int n, int D, int state,
                                                int& piv_s, int& state_s) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int j = 0; j < n && state == 0; ++j) {
    if (tid < 32) {
      double best = -1.0;
      int bi = n;
      for (int i = j + tid; i < n; i += 32) {
        const double2 v = A[i * n + j];
        const double mag = fabs(v.x) + fabs(v.y);
        if (mag > best) { best = mag; bi = i; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (tid == 0) {
        piv_s = bi;
        state_s = best > 0.0 ? 0 : 1;
      }
    }
    __syncthreads();
    state = state_s;
    if (state != 0) break;
    const int piv = piv_s;
    if (piv != j) {
      for (int c = tid; c < n + D; c += nt) {
        double2* a = c < n ? A + j * n + c : X + j * D + c - n;
        double2* b = c < n ? A + piv * n + c : X + piv * D + c - n;
        const double2 t = *a;
        *a = *b;
        *b = t;
      }
      __syncthreads();
    }
    const double2 pv = A[j * n + j];
    for (int i = j + 1 + tid; i < n; i += nt) f[i] = cdiv(A[i * n + j], pv);
    __syncthreads();
    const int w = n - j - 1 + D;
    for (int idx = tid; idx < (n - j - 1) * w; idx += nt) {
      const int i = j + 1 + idx / w, cc = idx % w;
      const double2 fi = f[i];
      if (cc < n - j - 1) {
        const int c = j + 1 + cc;
        const double2 qv = cmul(fi, A[j * n + c]);
        A[i * n + c].x -= qv.x; A[i * n + c].y -= qv.y;
      } else {
        const int c = cc - (n - j - 1);
        const double2 qv = cmul(fi, X[j * D + c]);
        X[i * D + c].x -= qv.x; X[i * D + c].y -= qv.y;
      }
    }
    __syncthreads();
  }
  return state;
}

// back substitution of the eliminated system: X <- U^-1 X
__device__ __forceinline__ void wpe_lu_back(const double2* A, double2* X, int n, int D) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = n - 1; i >= 0; --i) {
    if (tid < D) X[i * D + tid] = cdiv(X[i * D + tid], A[i * n + i]);
    __syncthreads();
    for (int idx = tid; idx < i * D; idx += nt) {
      const int rr = idx / D, c = idx - rr * D;
      const double2 qv = cmul(A[rr * n + i], X[i * D + c]);
      X[rr * D + c].x -= qv.x; X[rr * D + c].y -= qv.y;
    }
    __syncthreads();
  }
}

// one CTA (256 threads) per bin.  G (bins, n, D) complex; lstsq (bins) = 1 where the pivot was exactly zero.
__global__ void __launch_bounds__(256) wpe_solve_kernel(const double* __restrict__ part, WpeShape s,
                                                        double2* __restrict__ G, int* __restrict__ lstsq,
                                                        int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = s.n, D = s.D, tid = threadIdx.x, nt = blockDim.x;
  double2* A = reinterpret_cast<double2*>(smem_raw);
  double2* X = A + n * n;
  double2* f = X + n * D;
  double* red = reinterpret_cast<double*>(f + n);
  __shared__ int piv_s, state_s;   // state: 0 running, 1 singular (zero pivot), 2 non-finite
  const long long bin = blockIdx.x;
  const double* pb = part + bin * s.parts * (long long)s.ntiles * 64;
  double amax = 0.0;
  bool bad = false;
  for (int i = tid; i < n * (n + D); i += nt) {
    const int row = i / (n + D), col = i - row * (n + D);
    const double2 v = wpe_complex(pb, s, row, col);
    if (col < n) {
      A[row * n + col] = v;
      amax = cabs_max(amax, v);
      bad |= !isfinite(v.x) || !isfinite(v.y);
    } else {
      X[row * D + col - n] = v;
    }
  }
  bad = __syncthreads_or(bad);
  amax = wpe_block_max(amax, red);
  // solve with 2^-escale R (exact), as solve_kernel does: G = 2^-escale times that solution
  const int escale = !(amax > 0.0) || !isfinite(amax) ? 0 : ilogb(amax) & ~1;
  for (int i = tid; i < n * n; i += nt) A[i] = cscalbn(A[i], -escale);
  int state = wpe_lu_eliminate(A, X, f, n, D, bad ? 2 : 0, piv_s, state_s);
  double2* g = G + bin * (long long)n * D;
  if (tid == 0) {
    lstsq[bin] = state == 1;
    if (state) atomicOr(status, state == 1 ? PBB_WPE_LSTSQ : PBB_WPE_NONFINITE);
  }
  if (state == 2) {
    for (int i = tid; i < n * D; i += nt) g[i] = make_double2(CUDART_NAN, CUDART_NAN);
    return;
  }
  if (state == 1) return;   // wpe_lstsq_kernel writes this bin's G
  wpe_lu_back(A, X, n, D);
  for (int i = tid; i < n * D; i += nt) g[i] = cscalbn(X[i], -escale);
}

// The backward's solve: B <- R^-1 B in place (B (bins, n, D)), R assembled from the partial tiles exactly as
// wpe_solve_kernel does (the same scaling and pivots).  A zero pivot or a non-finite R gives NaN in that bin: the
// backward has no lstsq branch (the strict = 2 rule of solve_kernel).  One CTA (256 threads) per bin.
__global__ void __launch_bounds__(256) wpe_solve_rhs_kernel(const double* __restrict__ part, WpeShape s,
                                                            double2* __restrict__ B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = s.n, D = s.D, tid = threadIdx.x, nt = blockDim.x;
  double2* A = reinterpret_cast<double2*>(smem_raw);
  double2* X = A + n * n;
  double2* f = X + n * D;
  double* red = reinterpret_cast<double*>(f + n);
  __shared__ int piv_s, state_s;
  const long long bin = blockIdx.x;
  const double* pb = part + bin * s.parts * (long long)s.ntiles * 64;
  double2* b = B + bin * (long long)n * D;
  double amax = 0.0;
  bool bad = false;
  for (int i = tid; i < n * n; i += nt) {
    const int row = i / n, col = i - row * n;
    const double2 v = wpe_complex(pb, s, row, col);
    A[i] = v;
    amax = cabs_max(amax, v);
    bad |= !isfinite(v.x) || !isfinite(v.y);
  }
  for (int i = tid; i < n * D; i += nt) X[i] = b[i];
  bad = __syncthreads_or(bad);
  amax = wpe_block_max(amax, red);
  const int escale = !(amax > 0.0) || !isfinite(amax) ? 0 : ilogb(amax) & ~1;
  for (int i = tid; i < n * n; i += nt) A[i] = cscalbn(A[i], -escale);
  const int state = wpe_lu_eliminate(A, X, f, n, D, bad ? 2 : 0, piv_s, state_s);
  if (state) {
    for (int i = tid; i < n * D; i += nt) b[i] = make_double2(CUDART_NAN, CUDART_NAN);
    return;
  }
  wpe_lu_back(A, X, n, D);
  for (int i = tid; i < n * D; i += nt) b[i] = cscalbn(X[i], -escale);
}

__host__ __device__ inline size_t wpe_lstsq_smem_bytes(int n, int D) {
  return ((size_t)n * n + 2 * (size_t)n * D) * sizeof(double2) + (size_t)((n + 1) / 2) * 6 * sizeof(double);
}

// one warp per bin with an exactly zero pivot: G = V diag(1 / lambda) V^H P over the eigenvalues of R above
// eps n max|lambda| (np.linalg.lstsq's default rcond on the singular values of the Hermitian R).  V lives in the
// bin's first partial tiles (16 ntiles 32 >= n^2 complex), which are no longer needed once R is in shared memory.
__global__ void __launch_bounds__(32) wpe_lstsq_kernel(double* __restrict__ part, WpeShape s,
                                                       const int* __restrict__ lstsq, double2* __restrict__ G) {
  const long long bin = blockIdx.x;
  if (!lstsq[bin]) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = s.n, D = s.D, lane = threadIdx.x;
  double2* A = reinterpret_cast<double2*>(smem_raw);
  double2* P = A + n * n;
  double2* Tm = P + n * D;
  double* rot = reinterpret_cast<double*>(Tm + n * D);
  double* pb = part + bin * s.parts * (long long)s.ntiles * 64;
  double amax = 0.0;
  for (int i = lane; i < n * (n + D); i += 32) {
    const int row = i / (n + D), col = i - row * (n + D);
    const double2 v = wpe_complex(pb, s, row, col);
    if (col < n) { A[row * n + col] = v; amax = cabs_max(amax, v); }
    else P[row * D + col - n] = v;
  }
  const int escale = even_exponent(amax);
  for (int i = lane; i < n * n; i += 32) A[i] = cscalbn(A[i], -escale);
  __syncwarp();
  double2* V = reinterpret_cast<double2*>(pb);
  warp_jacobi(A, V, rot, n, lane);
  __syncwarp();
  double lmax = 0.0;
  for (int i = 0; i < n; ++i) lmax = fmax(lmax, fabs(A[i * n + i].x));
  const double cut = DBL_EPSILON * n * lmax;
  for (int i = lane; i < n * D; i += 32) {
    const int e = i / D, c = i - e * D;
    const double l = A[e * n + e].x;
    double2 t = make_double2(0.0, 0.0);
    if (fabs(l) > cut) {
      for (int k = 0; k < n; ++k) {
        const double2 qv = cmulc(P[k * D + c], V[k * n + e]);
        t.x += qv.x; t.y += qv.y;
      }
      t.x /= l; t.y /= l;
    }
    Tm[i] = t;
  }
  __syncwarp();
  double2* g = G + bin * (long long)n * D;
  for (int i = lane; i < n * D; i += 32) {
    const int rr = i / D, c = i - rr * D;
    double2 o = make_double2(0.0, 0.0);
    for (int e = 0; e < n; ++e) {
      const double2 qv = cmul(V[rr * n + e], Tm[e * D + c]);
      o.x += qv.x; o.y += qv.y;
    }
    g[i] = cscalbn(o, -escale);
  }
}

// ---- 3. filter and power ----------------------------------------------------------------------------------------
enum { kWpePowerInverse = 0, kWpePowerPlain = 1, kWpePowerNone = 2 };

__host__ __device__ inline size_t wpe_filter_smem_bytes(int D, int taps) {
  const int n = D * taps;
  return ((size_t)n * D + (size_t)D * (kWpeFilterChunk + taps - 1) + (size_t)D * kWpeFilterChunk) * sizeof(double2) +
         (size_t)D * kWpeFilterChunk * sizeof(double) + 256 * sizeof(double);
}

// One CTA (256 threads) per bin.  X = Y - G^H Yt (G null: X = Y), stored to out (null: not stored).  power mode:
// kWpePowerInverse writes w = 1 / max(lambda_c, 1e-10 max_t lambda_c) to pw, kWpePowerPlain writes lambda_c, where
// lambda_c is the psd_context mean of lambda_t = mean_d |X_dt|^2 (lam: bins x T scratch); kWpePowerNone skips it.
// Chunks run from the last frame to the first, so out may alias y: a chunk only reads frames at or before its own.
template <class TIn>
__global__ void __launch_bounds__(256) wpe_filter_kernel(const TIn* y, WpeStrides ys, WpeShape s,
                                                         const double2* __restrict__ G, TIn* out, WpeStrides os,
                                                         int power, double* __restrict__ lam, double* __restrict__ pw,
                                                         int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = s.D, taps = s.taps, n = s.n, tid = threadIdx.x, nt = blockDim.x;
  const int lw = kWpeFilterChunk + taps - 1;
  const long long T = s.T, bin = blockIdx.x;
  double2* Gs = reinterpret_cast<double2*>(smem_raw);
  double2* Yd = Gs + n * D;                 // delayed window (D, lw)
  double2* Yc = Yd + D * lw;                // current window (D, chunk)
  double* sq = reinterpret_cast<double*>(Yc + D * kWpeFilterChunk);   // |X|^2 (D, chunk)
  double* red = sq + D * kWpeFilterChunk;
  const TIn* yb = y + bin * ys.b;
  if (G != nullptr)
    for (int i = tid; i < n * D; i += nt) Gs[i] = G[bin * n * D + i];
  double* lb = lam + bin * T;
  int bad = 0;
  const long long nchunks = (T + kWpeFilterChunk - 1) / kWpeFilterChunk;
  for (long long ci = nchunks - 1; ci >= 0; --ci) {
    const long long t0 = ci * kWpeFilterChunk, ws = t0 - s.delay - taps + 1;
    __syncthreads();
    if (G != nullptr)
      for (int i = tid; i < D * lw; i += nt) {
        const int d = i / lw, j = i - d * lw;
        const long long f = ws + j;
        Yd[i] = f >= 0 && f < T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
      }
    for (int i = tid; i < D * kWpeFilterChunk; i += nt) {
      const int d = i / kWpeFilterChunk, j = i - d * kWpeFilterChunk;
      const long long f = t0 + j;
      Yc[i] = f < T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
    }
    __syncthreads();
    for (int i = tid; i < D * kWpeFilterChunk; i += nt) {
      const int d = i / kWpeFilterChunk, j = i - d * kWpeFilterChunk;
      double2 x = Yc[i];
      if (G != nullptr) {
        double2 acc = make_double2(0.0, 0.0);
        for (int k = 0; k < taps; ++k)
          for (int e = 0; e < D; ++e) {
            // conj(G[k D + e][d]) * Y_{e, t - delay - k}
            const double2 qv = cmulc(Yd[e * lw + j + taps - 1 - k], Gs[(k * D + e) * D + d]);
            acc.x += qv.x; acc.y += qv.y;
          }
        x.x -= acc.x;
        x.y -= acc.y;
      }
      const long long t = t0 + j;
      if (t < T) {
        if (out != nullptr) {
          wpe_store(out + bin * os.b, d * os.d + t * os.t, x);
          bad |= !isfinite(x.x) || !isfinite(x.y);
        }
        sq[i] = x.x * x.x + x.y * x.y;
      }
    }
    if (power == kWpePowerNone) continue;
    __syncthreads();
    for (int j = tid; j < kWpeFilterChunk; j += nt) {
      if (t0 + j >= T) continue;
      double v = 0.0;
      for (int d = 0; d < D; ++d) v += sq[d * kWpeFilterChunk + j];
      lb[t0 + j] = v / D;
    }
  }
  if (__syncthreads_or(bad) && tid == 0) atomicOr(status, PBB_WPE_NONFINITE);
  if (power == kWpePowerNone) return;
  double* pwb = pw + bin * T;
  const long long c = s.psd_context;
  if (c < 0) {
    // the mean over all frames: per-thread sums in frame order, then the threads in order
    double v = 0.0;
    for (long long t = tid; t < T; t += nt) v += lb[t];
    __syncthreads();
    red[tid] = v;
    __syncthreads();
    v = 0.0;
    for (int i = 0; i < nt; ++i) v += red[i];
    const double m = v / T;
    for (long long t = tid; t < T; t += nt) pwb[t] = m;
  } else if (c == 0) {
    for (long long t = tid; t < T; t += nt) pwb[t] = lb[t];
  } else {
    for (long long t = tid; t < T; t += nt) {
      const long long lo = t - c < 0 ? 0 : t - c, hi = t + c >= T ? T - 1 : t + c;
      double v = 0.0;
      for (long long u = lo; u <= hi; ++u) v += lb[u];
      pwb[t] = v / (double)(hi - lo + 1);
    }
  }
  if (power == kWpePowerPlain) return;
  double mx = 0.0;
  __syncthreads();
  for (long long t = tid; t < T; t += nt) mx = fmax(mx, pwb[t]);
  mx = wpe_block_max(mx, red);
  const double eps = 1e-10 * mx;
  for (long long t = tid; t < T; t += nt) pwb[t] = 1.0 / fmax(pwb[t], eps);
}

// get_power_inverse of a whole array: 1 / max(p, 1e-10 max p) over all `count` values of p, in place (one CTA)
__global__ void __launch_bounds__(1024) wpe_power_inverse_kernel(double* __restrict__ p, long long count) {
  __shared__ double red[32];
  double mx = 0.0;
  for (long long i = threadIdx.x; i < count; i += blockDim.x) mx = fmax(mx, p[i]);
  mx = wpe_block_max(mx, red);
  const double eps = 1e-10 * mx;
  for (long long i = threadIdx.x; i < count; i += blockDim.x) p[i] = 1.0 / fmax(p[i], eps);
}

// ---- 4. backward passes (pbb_wpe_backward, pbb_wpe_power_backward; the closed forms are in include/pbb.h) -------
constexpr int kWpeBackChunk = 64;            // frames per chunk of the backward's per-bin kernels

// caller weights (element (b, t) at b wsb + t wst) -> w (bins, T) contiguous
__global__ void wpe_weight_copy_kernel(const double* __restrict__ src, long long wsb, long long wst, long long bins,
                                       long long T, double* __restrict__ w) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < bins * T;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / T, t = i - b * T;
    w[i] = src[b * wsb + t * wst];
  }
}

__host__ __device__ inline size_t wpe_gbar_smem_bytes(int D, int taps) {
  return ((size_t)D * taps * D + (size_t)D * (kWpeBackChunk + taps - 1) + (size_t)D * kWpeBackChunk) *
         sizeof(double2);
}

// Gbar = -sum_t Yt_t xbar_t^H over every frame: Gbar[k D + e][d] = -sum_t Y_{e, t - delay - k} conj(xbar_{d, t}).
// One CTA (256 threads) per bin; each entry is owned by one thread and summed in frame order (the running sums stay
// in shared memory between chunks).  xbar (bins, D, T) contiguous; Gbar (bins, n, D).
template <class TIn>
__global__ void __launch_bounds__(256) wpe_gbar_kernel(const TIn* __restrict__ y, WpeStrides ys, WpeShape s,
                                                       const double2* __restrict__ xbar, double2* __restrict__ Gbar) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = s.D, taps = s.taps, n = s.n, tid = threadIdx.x, nt = blockDim.x;
  const int lw = kWpeBackChunk + taps - 1;
  const long long T = s.T, bin = blockIdx.x;
  double2* acc = reinterpret_cast<double2*>(smem_raw);
  double2* Yd = acc + n * D;                // delayed window (D, lw)
  double2* Xb = Yd + D * lw;                // xbar chunk (D, chunk)
  const TIn* yb = y + bin * ys.b;
  const double2* xb = xbar + bin * D * T;
  for (int i = tid; i < n * D; i += nt) acc[i] = make_double2(0.0, 0.0);
  for (long long t0 = 0; t0 < T; t0 += kWpeBackChunk) {
    const long long ws = t0 - s.delay - taps + 1;
    __syncthreads();
    for (int i = tid; i < D * lw; i += nt) {
      const int d = i / lw, j = i - d * lw;
      const long long f = ws + j;
      Yd[i] = f >= 0 && f < T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
    }
    for (int i = tid; i < D * kWpeBackChunk; i += nt) {
      const int d = i / kWpeBackChunk, j = i - d * kWpeBackChunk;
      Xb[i] = t0 + j < T ? xb[d * T + t0 + j] : make_double2(0.0, 0.0);
    }
    __syncthreads();
    for (int i = tid; i < n * D; i += nt) {
      const int row = i / D, d = i - row * D, k = row / D, e = row - k * D;
      const double2* yr = Yd + e * lw + taps - 1 - k;
      const double2* xr = Xb + d * kWpeBackChunk;
      double2 a = acc[i];
      for (int j = 0; j < kWpeBackChunk; ++j) {
        const double2 qv = cmulc(yr[j], xr[j]);   // Y conj(xbar)
        a.x += qv.x; a.y += qv.y;
      }
      acc[i] = a;
    }
  }
  __syncthreads();
  double2* g = Gbar + bin * (long long)n * D;
  for (int i = tid; i < n * D; i += nt) g[i] = make_double2(-acc[i].x, -acc[i].y);
}

__host__ __device__ inline size_t wpe_step_backward_smem_bytes(int D, int taps) {
  const int lw = kWpeBackChunk + taps - 1;
  return (2 * (size_t)D * taps * D + 3 * (size_t)D * lw) * sizeof(double2) + (size_t)D * kWpeBackChunk * sizeof(double);
}

// One stage of the step backward for one bin per CTA (256 threads), given G, Pbar = R^-1 Gbar and w, per frame:
//   x_t = y_t - G^H yt_t, c_t = Pbar^H yt_t, m_t = [t in S], u_t = xbar_t + m_t w_t c_t, b_t = m_t w_t x_t,
//   wbar_t = m_t Re(c_t^H x_t), ybar_t += u_t + sum_k (-G_k u_{t + delay + k} + Pbar_k b_{t + delay + k})
// with G_k, Pbar_k the D x D blocks of rows k D .. k D + D - 1.  The last term is the shift-add of
// Ytbar_t = -G u_t + Pbar b_t back onto Y, written as a gather over later frames: chunks run from the last frame to
// the first, u and b of every chunk go to ub (bins, 2, D, T) before the chunk gathers from it, and a chunk reads
// only frames at or after its own.  ybar, xbar (bins, D, T) contiguous; ybar accumulated, wbar (bins, T) written.
template <class TIn>
__global__ void __launch_bounds__(256) wpe_step_backward_kernel(const TIn* __restrict__ y, WpeStrides ys, WpeShape s,
                                                                const double2* __restrict__ G,
                                                                const double2* __restrict__ Pbar,
                                                                const double* __restrict__ w,
                                                                const double2* __restrict__ xbar, double2* ub,
                                                                double2* __restrict__ ybar,
                                                                double* __restrict__ wbar) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = s.D, taps = s.taps, n = s.n, tid = threadIdx.x, nt = blockDim.x;
  const int lw = kWpeBackChunk + taps - 1;
  const long long T = s.T, bin = blockIdx.x;
  double2* Gs = reinterpret_cast<double2*>(smem_raw);
  double2* Ps = Gs + n * D;
  double2* Yd = Ps + n * D;                 // delayed window of y (D, lw), frames from t0 - delay - taps + 1
  double2* Uf = Yd + D * lw;                // u over frames t0 + delay .. (D, lw)
  double2* Bf = Uf + D * lw;                // b likewise
  double* pr = reinterpret_cast<double*>(Bf + D * lw);   // Re(c^H x) terms (D, chunk)
  const TIn* yb = y + bin * ys.b;
  const double2* xb = xbar + bin * D * T;
  const double* wb = w + bin * T;
  double2* ubu = ub + bin * 2 * D * T;
  double2* ubb = ubu + D * T;
  double2* yo = ybar + bin * D * T;
  for (int i = tid; i < n * D; i += nt) {
    Gs[i] = G[bin * n * D + i];
    Ps[i] = Pbar[bin * n * D + i];
  }
  const long long nchunks = (T + kWpeBackChunk - 1) / kWpeBackChunk;
  for (long long ci = nchunks - 1; ci >= 0; --ci) {
    const long long t0 = ci * kWpeBackChunk, ws = t0 - s.delay - taps + 1;
    __syncthreads();
    for (int i = tid; i < D * lw; i += nt) {
      const int d = i / lw, j = i - d * lw;
      const long long f = ws + j;
      Yd[i] = f >= 0 && f < T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
    }
    __syncthreads();
    for (int i = tid; i < D * kWpeBackChunk; i += nt) {
      const int d = i / kWpeBackChunk, j = i - d * kWpeBackChunk;
      const long long t = t0 + j;
      if (t >= T) {
        pr[i] = 0.0;
        continue;
      }
      double2 x = wpe_load(yb, d * ys.d + t * ys.t), c = make_double2(0.0, 0.0);
      for (int k = 0; k < taps; ++k)
        for (int e = 0; e < D; ++e) {
          const double2 yv = Yd[e * lw + j + taps - 1 - k];
          const double2 qg = cmulc(yv, Gs[(k * D + e) * D + d]), qp = cmulc(yv, Ps[(k * D + e) * D + d]);
          x.x -= qg.x; x.y -= qg.y;
          c.x += qp.x; c.y += qp.y;
        }
      const double mw = t >= s.tb ? wb[t] : 0.0;
      const double2 xv = xb[d * T + t];
      ubu[d * T + t] = make_double2(xv.x + mw * c.x, xv.y + mw * c.y);
      ubb[d * T + t] = make_double2(mw * x.x, mw * x.y);
      pr[i] = t >= s.tb ? c.x * x.x + c.y * x.y : 0.0;
    }
    __syncthreads();
    for (int j = tid; j < kWpeBackChunk; j += nt) {
      if (t0 + j >= T) continue;
      double v = 0.0;
      for (int d = 0; d < D; ++d) v += pr[d * kWpeBackChunk + j];
      wbar[bin * T + t0 + j] = v;
    }
    // u and b over the frames t0 + delay + j (j < lw) that exist; later chunks wrote theirs in earlier iterations
    for (int i = tid; i < D * lw; i += nt) {
      const int d = i / lw, j = i - d * lw;
      const long long f = t0 + s.delay + j;
      const bool in = f < T;
      Uf[i] = in ? ubu[d * T + f] : make_double2(0.0, 0.0);
      Bf[i] = in ? ubb[d * T + f] : make_double2(0.0, 0.0);
    }
    __syncthreads();
    for (int i = tid; i < D * kWpeBackChunk; i += nt) {
      const int d = i / kWpeBackChunk, j = i - d * kWpeBackChunk;
      const long long t = t0 + j;
      if (t >= T) continue;
      double2 a = ubu[d * T + t];
      for (int k = 0; k < taps; ++k)
        for (int e = 0; e < D; ++e) {
          const double2 qg = cmul(Gs[(k * D + d) * D + e], Uf[e * lw + j + k]);
          const double2 qp = cmul(Ps[(k * D + d) * D + e], Bf[e * lw + j + k]);
          a.x += qp.x - qg.x; a.y += qp.y - qg.y;
        }
      const double2 o = yo[d * T + t];
      yo[d * T + t] = make_double2(o.x + a.x, o.y + a.y);
    }
  }
}

enum { kWpeGradInverse = PBB_WPE_GRAD_INVERSE, kWpeGradPlain = PBB_WPE_GRAD_PLAIN, kWpeGradInverseAll = PBB_WPE_GRAD_INVERSE_ALL };

// the backward of w = 1 / max(p, 1e-10 M), M = max p (fmax from 0, as the forward), over p[0, count): the gradient of
// p given wbar, torch.maximum's and amax's rule (ties split evenly).  Every thread of the CTA calls it; red holds
// blockDim.x doubles.  Sums run per thread in index order, then over the threads in order.
__device__ __forceinline__ void wpe_inverse_backward(const double* p, const double* wbar, double* pbar, long long count,
                                                     double* red) {
  const int tid = threadIdx.x, nt = blockDim.x;
  double mx = 0.0;
  for (long long t = tid; t < count; t += nt) mx = fmax(mx, p[t]);
  mx = wpe_block_max(mx, red);
  const double eps = 1e-10 * mx;
  double gb = 0.0, ties = 0.0;
  for (long long t = tid; t < count; t += nt) {
    const double v = p[t], z = fmax(v, eps);
    const double zb = -wbar[t] / (z * z);
    pbar[t] = v > eps ? zb : v == eps ? 0.5 * zb : 0.0;
    gb += v < eps ? zb : v == eps ? 0.5 * zb : 0.0;
    ties += v == mx;
  }
  __syncthreads();
  red[tid] = gb;
  red[nt + tid] = ties;
  __syncthreads();
  gb = 0.0;
  ties = 0.0;
  for (int i = 0; i < nt; ++i) {
    gb += red[i];
    ties += red[nt + i];
  }
  const double share = 1e-10 * gb / ties;
  for (long long t = tid; t < count; t += nt)
    if (p[t] == mx) pbar[t] += share;
  __syncthreads();
}

// get_power_inverse's max over the whole array: pbar from lamc and wbar over all `count` values (one CTA)
__global__ void __launch_bounds__(1024) wpe_power_inverse_backward_kernel(const double* __restrict__ lamc,
                                                                          const double* __restrict__ wbar,
                                                                          double* __restrict__ pbar, long long count) {
  __shared__ double red[2048];
  wpe_inverse_backward(lamc, wbar, pbar, count, red);
}

__host__ __device__ inline size_t wpe_power_backward_smem_bytes(int D, int taps, bool filter) {
  return filter ? ((size_t)taps * D * D + (size_t)D * (kWpeFilterChunk + taps - 1)) * sizeof(double2) +
                      512 * sizeof(double)
                : 512 * sizeof(double);
}

// The power chain's backward for one bin per CTA (256 threads): x = y - G^H Yt (G null: x = y), lamc (bins, T) the
// forward's lambda_c.  mode kWpeGradInverse: gin is wbar of w = 1 / max(lambda_c, 1e-10 max_t lambda_c);
// kWpeGradPlain: gin is lambda_c's gradient.  lambda_c's gradient goes through the adjoint of the psd_context mean,
// lambdabar_t = sum_{s : |s - t| <= c} lambdabar_c,s / n_s (n_s the frames in s's window), and
// xbar_dt += (2 / D) lambdabar_t x_dt (xbar (bins, D, T) contiguous, accumulated).  lamc and pbar are overwritten.
template <class TIn>
__global__ void __launch_bounds__(256) wpe_power_backward_kernel(const TIn* __restrict__ y, WpeStrides ys, WpeShape s,
                                                                 const double2* __restrict__ G, double* lamc,
                                                                 const double* __restrict__ gin, int mode,
                                                                 double* pbar, double2* __restrict__ xbar) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D = s.D, taps = s.taps, n = s.n, tid = threadIdx.x, nt = blockDim.x;
  const int lw = kWpeFilterChunk + taps - 1;
  const long long T = s.T, bin = blockIdx.x;
  double* red = reinterpret_cast<double*>(smem_raw);
  double2* Gs = reinterpret_cast<double2*>(red + 512);
  double2* Yd = Gs + n * D;
  double* lc = lamc + bin * T;
  double* pb = pbar + bin * T;
  const double* gb = gin + bin * T;
  if (mode == kWpeGradInverse) {
    wpe_inverse_backward(lc, gb, pb, T, red);
  } else {
    for (long long t = tid; t < T; t += nt) pb[t] = gb[t];
    __syncthreads();
  }
  // lambdabar into lc
  const long long c = s.psd_context;
  if (c < 0) {
    double v = 0.0;
    for (long long t = tid; t < T; t += nt) v += pb[t];
    __syncthreads();
    red[tid] = v;
    __syncthreads();
    v = 0.0;
    for (int i = 0; i < nt; ++i) v += red[i];
    const double m = v / T;
    for (long long t = tid; t < T; t += nt) lc[t] = m;
  } else if (c == 0) {
    for (long long t = tid; t < T; t += nt) lc[t] = pb[t];
  } else {
    for (long long t = tid; t < T; t += nt) {
      const long long lo = t - c < 0 ? 0 : t - c, hi = t + c >= T ? T - 1 : t + c;
      pb[t] /= (double)(hi - lo + 1);
    }
    __syncthreads();
    for (long long t = tid; t < T; t += nt) {
      const long long lo = t - c < 0 ? 0 : t - c, hi = t + c >= T ? T - 1 : t + c;
      double v = 0.0;
      for (long long u = lo; u <= hi; ++u) v += pb[u];
      lc[t] = v;
    }
  }
  const TIn* yb = y + bin * ys.b;
  double2* xo = xbar + bin * D * T;
  const double scale = 2.0 / D;
  if (G != nullptr)
    for (int i = tid; i < n * D; i += nt) Gs[i] = G[bin * n * D + i];
  for (long long t0 = 0; t0 < T; t0 += kWpeFilterChunk) {
    const long long ws = t0 - s.delay - taps + 1;
    __syncthreads();
    if (G != nullptr)
      for (int i = tid; i < D * lw; i += nt) {
        const int d = i / lw, j = i - d * lw;
        const long long f = ws + j;
        Yd[i] = f >= 0 && f < T ? wpe_load(yb, d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
      }
    __syncthreads();
    for (int i = tid; i < D * kWpeFilterChunk; i += nt) {
      const int d = i / kWpeFilterChunk, j = i - d * kWpeFilterChunk;
      const long long t = t0 + j;
      if (t >= T) continue;
      double2 x = wpe_load(yb, d * ys.d + t * ys.t);
      if (G != nullptr) {
        double2 acc = make_double2(0.0, 0.0);
        for (int k = 0; k < taps; ++k)
          for (int e = 0; e < D; ++e) {
            const double2 qv = cmulc(Yd[e * lw + j + taps - 1 - k], Gs[(k * D + e) * D + d]);
            acc.x += qv.x; acc.y += qv.y;
          }
        x.x -= acc.x;
        x.y -= acc.y;
      }
      const double f = scale * lc[t];
      const double2 o = xo[d * T + t];
      xo[d * T + t] = make_double2(o.x + f * x.x, o.y + f * x.y);
    }
  }
}

// build_y_tilde: out (bins, taps D, T) contiguous, row k D + d at frame t = Y_{d, t - delay - k} (0 before frame 0)
template <class TIn>
__global__ void wpe_y_tilde_kernel(const TIn* __restrict__ y, WpeStrides ys, long long bins, int D, long long T,
                                   int taps, int delay, TIn* __restrict__ out) {
  const long long per = (long long)taps * D * T;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < bins * per;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / per, rest = i - b * per;
    const int row = (int)(rest / T);
    const long long t = rest - row * T;
    const int k = row / D, d = row - k * D;
    const long long f = t - delay - k;
    const double2 v = f >= 0 ? wpe_load(y, b * ys.b + d * ys.d + f * ys.t) : make_double2(0.0, 0.0);
    wpe_store(out, i, v);
  }
}

}  // namespace pbb
