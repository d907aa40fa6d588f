// BSS Eval v3 (mir_eval.separation.bss_eval_sources, pb_bss/evaluation/module_mir_eval.py) -- see include/pbb.h.
//
// Per batch item: K references s_i and E estimates, T samples, L = 512-tap distortion filters, N = K L.
//   1. bss_corr_kernel: r_as[d] = sum_v s_a[v - d] x_s[v] for every reference a, signal s (references, then
//      estimates) and lag d < L, as a GEMM of the L x T shifted copies of s_a (staged in shared memory) with the
//      T x (K + E) signals, on fp64 m8n8k4 mma.sync.  T is split into at most kCorrParts parts (a function of T
//      only); bss_corr_reduce_kernel sums the parts in order.
//   2. bss_assemble_kernel: the augmented system [G | D] (N x (N + E)) and, for K > 1, the K diagonal blocks
//      [G_jj | D_j] (L x (L + E)).
//   3. Blocked LU with partial pivoting of every augmented matrix (bss_lu_panel_kernel, one CTA per matrix, swaps
//      whole rows; bss_lu_trsm_kernel; bss_lu_update_kernel, the trailing update on mma.sync), which leaves
//      L^-1 P D in the right-hand columns; bss_backsub_kernel solves U c = L^-1 P D in place.
//   4. bss_project_kernel: P_all x_e and P_j x_e over T + L - 1 samples as 512-tap convolutions on mma.sync, tiled
//      like step 1, and the per-tile sums of squares of P_j, x - P_j, P_all - P_j (per (e, j)), P_all and x - P_all
//      (per e), reduced in a fixed order and never stored as signals.
//   5. bss_ratio_kernel: the tile sums in order, SDR / SIR / SAR with mir_eval's _safe_db, and the first maximiser
//      of the mean SIR over itertools.permutations(range(E), K) with np.mean / np.argmax semantics.
// No float atomics anywhere: every result is bitwise reproducible and independent of the rest of the batch.
#pragma once
#include <math_constants.h>

#include "common.cuh"

namespace pbb {

constexpr int kBssL = PBB_BSS_EVAL_FILTER;   // 512
constexpr int kCorrChunk = 128;              // samples staged per step of bss_corr_kernel
constexpr int kCorrParts = 64;               // at most this many parts of T per (item, reference)
constexpr int kProjTile = 128;               // output samples per CTA of bss_project_kernel
constexpr int kPanel = 32;                   // LU panel width
constexpr int kRhsPad = 16;                  // row stride of an augmented matrix = n + kRhsPad (E <= 9)

// flags per item (bss_status_kernel folds them into the status word)
enum { kBssZeroSignal = 1, kBssNonFinite = 2, kBssZeroPivot = 4 };

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

struct BssShape {
  long long T;    // samples
  int K, E, S;    // references, estimates, K + E
  int N;          // K L
  int parts;      // parts of T in bss_corr_kernel
  long long span; // samples per part (a multiple of kCorrChunk)
  long long tiles;// kProjTile tiles of T + L - 1
};

// ---- 0. all-zero and non-finite signals ----------------------------------------------------------------------
// grid (S, items): one CTA per signal; x (items, S, T)
__global__ void bss_check_kernel(const double* __restrict__ x, long long T, int S, int* __restrict__ flags) {
  const long long item = blockIdx.y;
  const double* p = x + (item * S + blockIdx.x) * T;
  int nonzero = 0, bad = 0;
  for (long long t = threadIdx.x; t < T; t += blockDim.x) {
    const double v = p[t];
    nonzero |= v != 0.0;
    bad |= !isfinite(v);
  }
  nonzero = __syncthreads_or(nonzero);
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0 && (!nonzero || bad))
    atomicOr(flags + item, (nonzero ? 0 : kBssZeroSignal) | (bad ? kBssNonFinite : 0));
}

// ---- 1. lag correlations ---------------------------------------------------------------------------------------
// grid (parts, K, items), 256 threads.  Warp w owns lags [64 w, 64 w + 64) (8 m-tiles), all NS n-tiles of signals.
// part (items, K, parts, S, L).
template <int NS>
__global__ void __launch_bounds__(256) bss_corr_kernel(const double* __restrict__ x, BssShape sh,
                                                       double* __restrict__ part) {
  constexpr int LD = kCorrChunk + 4;
  __shared__ double aseg[kCorrChunk + kBssL];
  __shared__ double xs[8 * NS][LD];
  const int p = blockIdx.x, a = blockIdx.y;
  const long long item = blockIdx.z;
  const double* sig = x + item * sh.S * sh.T;
  const double* ref = sig + (long long)a * sh.T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = lane >> 2, q = lane & 3;
  double acc[8][NS][2];
#pragma unroll
  for (int m = 0; m < 8; ++m)
#pragma unroll
    for (int n = 0; n < NS; ++n) acc[m][n][0] = acc[m][n][1] = 0.0;
  const long long v_begin = p * sh.span, v_end = min(sh.T, v_begin + sh.span);
  for (long long v0 = v_begin; v0 < v_end; v0 += kCorrChunk) {
    __syncthreads();
    for (int i = threadIdx.x; i < kCorrChunk + kBssL - 1; i += blockDim.x) {
      const long long v = v0 - (kBssL - 1) + i;
      aseg[i] = v >= 0 && v < sh.T ? ref[v] : 0.0;
    }
    for (int i = threadIdx.x; i < 8 * NS * kCorrChunk; i += blockDim.x) {
      const int s = i / kCorrChunk, c = i % kCorrChunk;
      xs[s][c] = s < sh.S && v0 + c < sh.T ? sig[(long long)s * sh.T + v0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll 2
    for (int k = 0; k < kCorrChunk; k += 4) {
      double b[NS];
#pragma unroll
      for (int n = 0; n < NS; ++n) b[n] = xs[8 * n + r][k + q];
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        // A[d, v] = s_a[v - d], d = 64 warp + 8 m + r, v = v0 + k + q
        const double av = aseg[k + q - (64 * warp + 8 * m + r) + kBssL - 1];
#pragma unroll
        for (int n = 0; n < NS; ++n) dmma(acc[m][n], av, b[n]);
      }
    }
  }
  double* out = part + ((item * sh.K + a) * sh.parts + p) * sh.S * kBssL;
#pragma unroll
  for (int m = 0; m < 8; ++m)
#pragma unroll
    for (int n = 0; n < NS; ++n)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int s = 8 * n + 2 * q + c, d = 64 * warp + 8 * m + r;
        if (s < sh.S) out[s * kBssL + d] = acc[m][n][c];
      }
}

// R (items, K, S, L) = sum over the parts, in order
__global__ void bss_corr_reduce_kernel(const double* __restrict__ part, BssShape sh, long long items,
                                       double* __restrict__ R) {
  const long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long per = (long long)sh.S * kBssL;
  if (id >= items * sh.K * per) return;
  const long long ia = id / per, rest = id % per;
  const double* p = part + ia * sh.parts * per + rest;
  double s = 0.0;
  for (int i = 0; i < sh.parts; ++i) s += p[i * per];
  R[id] = s;
}

// ---- 2. the augmented systems ----------------------------------------------------------------------------------
// G (items, N, N + kRhsPad): G[(i,t1), (j,t2)] = r_ij[t1 - t2] (r_ji[t2 - t1] for t1 < t2), columns N + e: r_(i, K+e)[t1].
// Gb (items, K, L, L + kRhsPad): the diagonal blocks, when K > 1.
__global__ void bss_assemble_kernel(const double* __restrict__ R, BssShape sh, long long items, double* __restrict__ G,
                                    double* __restrict__ Gb) {
  const long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int N = sh.N, ld = N + kRhsPad;
  const long long per = (long long)N * ld;
  if (id >= items * per) return;
  const long long item = id / per;
  const int row = (int)((id % per) / ld), col = (int)(id % ld);
  const double* Ri = R + item * sh.K * sh.S * kBssL;
  const int i = row / kBssL, t1 = row % kBssL;
  double v = 0.0;
  if (col < N) {
    const int j = col / kBssL, t2 = col % kBssL;
    v = t1 >= t2 ? Ri[((long long)i * sh.S + j) * kBssL + t1 - t2] : Ri[((long long)j * sh.S + i) * kBssL + t2 - t1];
  } else if (col < N + sh.E) {
    v = Ri[((long long)i * sh.S + sh.K + col - N) * kBssL + t1];
  }
  G[id] = v;
  if (Gb != nullptr && (col < N ? col / kBssL == i : true)) {
    const int c = col < N ? col % kBssL : kBssL + col - N;
    Gb[((item * sh.K + i) * kBssL + t1) * (kBssL + kRhsPad) + c] = v;
  }
}

// ---- 3. LU with partial pivoting of [A | B], n x (n + E), row stride ld ----------------------------------------
struct LuBatch {
  double* A;
  int n, ld, ncols;       // ncols = n + E
  int per_item;           // matrices per item (flags index = matrix / per_item)
  int* flags;
};

// One CTA (512 threads) per matrix: columns k0 .. k0 + kPanel - 1 of rows k0 .. n - 1.  The pivot is the first row
// of largest |a| (LAPACK's idamax); whole rows are swapped, so the right-hand columns see every interchange.
__global__ void __launch_bounds__(512) bss_lu_panel_kernel(LuBatch b, int k0) {
  __shared__ double red_v[32];
  __shared__ int red_i[32];
  __shared__ double prow[kPanel];
  __shared__ int piv_s;
  double* A = b.A + (long long)blockIdx.x * b.n * b.ld;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kend = min(k0 + kPanel, b.n);
  for (int j = k0; j < kend; ++j) {
    double best = -1.0;
    int bi = b.n;
    for (int i = j + tid; i < b.n; i += blockDim.x) {
      const double v = fabs(A[(long long)i * b.ld + j]);
      if (v > best) { best = v; bi = i; }   // NaN never wins (idamax)
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = best; red_i[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      best = lane < (int)(blockDim.x >> 5) ? red_v[lane] : -1.0;
      bi = lane < (int)(blockDim.x >> 5) ? red_i[lane] : b.n;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (lane == 0) {
        const int p = bi < b.n ? bi : j;    // an all-NaN column keeps its row
        piv_s = p;
        if (A[(long long)p * b.ld + j] == 0.0) atomicOr(b.flags + blockIdx.x / b.per_item, kBssZeroPivot);
      }
    }
    __syncthreads();
    const int p = piv_s;
    if (p != j) {
      double* rj = A + (long long)j * b.ld;
      double* rp = A + (long long)p * b.ld;
      for (int c = tid; c < b.ncols; c += blockDim.x) {
        const double t = rj[c];
        rj[c] = rp[c];
        rp[c] = t;
      }
      __syncthreads();
    }
    if (tid < kend - j) prow[tid] = A[(long long)j * b.ld + j + tid];
    __syncthreads();
    const double pv = prow[0];
    const int jj = j - k0, cend = kend - k0;
    for (int i = j + 1 + tid; i < b.n; i += blockDim.x) {
      // the row's panel entries are loaded together (one memory latency per row, not one per column)
      double* ri = A + (long long)i * b.ld + k0;
      double v[kPanel];
#pragma unroll
      for (int c = 0; c < kPanel; ++c)
        if (c >= jj && c < cend) v[c] = ri[c];
      double l = 0.0;
#pragma unroll
      for (int c = 0; c < kPanel; ++c)
        if (c == jj) l = v[c] / pv;
#pragma unroll
      for (int c = 0; c < kPanel; ++c) {
        if (c == jj) ri[c] = l;
        else if (c > jj && c < cend) ri[c] = fma(-l, prow[c - jj], v[c]);
      }
    }
    __syncthreads();
  }
}

// U12 = L11^-1 A12 for the columns right of the panel; grid (column tiles of 128, matrices)
__global__ void __launch_bounds__(128) bss_lu_trsm_kernel(LuBatch b, int k0) {
  __shared__ double L[kPanel][kPanel + 1];
  double* A = b.A + (long long)blockIdx.y * b.n * b.ld;
  const int nb = min(kPanel, b.n - k0);
  for (int i = threadIdx.x; i < kPanel * kPanel; i += blockDim.x) {
    const int r = i / kPanel, c = i % kPanel;
    L[r][c] = r < nb && c < nb ? A[(long long)(k0 + r) * b.ld + k0 + c] : 0.0;
  }
  __syncthreads();
  const int col = k0 + nb + blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= b.ncols) return;
  double x[kPanel];
#pragma unroll
  for (int r = 0; r < kPanel; ++r) x[r] = r < nb ? A[(long long)(k0 + r) * b.ld + col] : 0.0;
#pragma unroll
  for (int r = 1; r < kPanel; ++r)
#pragma unroll
    for (int c = 0; c < r; ++c) x[r] = fma(-L[r][c], x[c], x[r]);
#pragma unroll
  for (int r = 0; r < kPanel; ++r)
    if (r < nb) A[(long long)(k0 + r) * b.ld + col] = x[r];
}

// A22 -= L21 U12 on mma.sync: 64 x 64 tiles, 4 warps of 32 x 32; grid (column tiles, row tiles, matrices)
__global__ void __launch_bounds__(128) bss_lu_update_kernel(LuBatch b, int k0) {
  constexpr int LD = kPanel + 4;
  __shared__ double As[64][LD];   // L21 tile [row][k]
  __shared__ double Bs[64][LD];   // U12 tile transposed [col][k]
  double* A = b.A + (long long)blockIdx.z * b.n * b.ld;
  const int r0 = k0 + kPanel + blockIdx.y * 64, c0 = k0 + kPanel + blockIdx.x * 64;
  for (int i = threadIdx.x; i < 64 * kPanel; i += blockDim.x) {
    const int rr = i / kPanel, k = i % kPanel;
    As[rr][k] = r0 + rr < b.n ? A[(long long)(r0 + rr) * b.ld + k0 + k] : 0.0;
    const int k2 = i / 64, cc = i % 64;
    Bs[cc][k2] = c0 + cc < b.ncols ? A[(long long)(k0 + k2) * b.ld + c0 + cc] : 0.0;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, q = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  double acc[4][4][2];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n) acc[m][n][0] = acc[m][n][1] = 0.0;
#pragma unroll
  for (int k = 0; k < kPanel; k += 4) {
    double a[4], bb[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) a[m] = As[wm + 8 * m + r][k + q];
#pragma unroll
    for (int n = 0; n < 4; ++n) bb[n] = Bs[wn + 8 * n + r][k + q];
#pragma unroll
    for (int m = 0; m < 4; ++m)
#pragma unroll
      for (int n = 0; n < 4; ++n) dmma(acc[m][n], a[m], bb[n]);
  }
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int row = r0 + wm + 8 * m + r, col = c0 + wn + 8 * n + 2 * q + c;
        if (row < b.n && col < b.ncols) {
          double* e = A + (long long)row * b.ld + col;
          *e -= acc[m][n][c];
        }
      }
}

// U c = y for the E right-hand columns, in place, 32-row blocks from the bottom; one CTA (256 threads) per matrix.
// The diagonal block is staged in shared memory and solved by one warp; the rows above are updated by all threads.
__global__ void __launch_bounds__(256) bss_backsub_kernel(LuBatch b) {
  __shared__ double xb[kPanel][kRhsPad];
  __shared__ double U[kPanel][kPanel + 1];
  double* A = b.A + (long long)blockIdx.x * b.n * b.ld;
  const int E = b.ncols - b.n, tid = threadIdx.x;
  for (int r0 = ((b.n - 1) / kPanel) * kPanel; r0 >= 0; r0 -= kPanel) {
    const int nb = min(kPanel, b.n - r0);
    for (int i = tid; i < kPanel * kPanel; i += blockDim.x) {
      const int rr = i / kPanel, c = i % kPanel;
      U[rr][c] = rr < nb && c < nb ? A[(long long)(r0 + rr) * b.ld + r0 + c] : 0.0;
    }
    __syncthreads();
    if (tid < 32) {
      const int row = r0 + tid;
      double y[kRhsPad];
#pragma unroll
      for (int e = 0; e < kRhsPad; ++e) y[e] = tid < nb && e < E ? A[(long long)row * b.ld + b.n + e] : 0.0;
      for (int rr = nb - 1; rr >= 0; --rr) {
        const double u = U[tid][rr], d = U[rr][rr];
#pragma unroll
        for (int e = 0; e < kRhsPad; ++e) {
          if (e < E) {
            const double xe = __shfl_sync(0xffffffffu, tid == rr ? y[e] / d : 0.0, rr);
            if (tid == rr) y[e] = xe;
            else if (tid < rr) y[e] = fma(-u, xe, y[e]);
          }
        }
      }
#pragma unroll
      for (int e = 0; e < kRhsPad; ++e) {
        xb[tid][e] = y[e];
        if (tid < nb && e < E) A[(long long)row * b.ld + b.n + e] = y[e];
      }
    }
    __syncthreads();
    for (int i = tid; i < r0; i += blockDim.x) {
      const double* ui = A + (long long)i * b.ld + r0;
      double u[kPanel];
#pragma unroll
      for (int c = 0; c < kPanel; ++c) u[c] = c < nb ? ui[c] : 0.0;
      double* yi = A + (long long)i * b.ld + b.n;
#pragma unroll 1
      for (int e = 0; e < E; ++e) {
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < kPanel; ++c) s = fma(u[c], xb[c][e], s);
        yi[e] -= s;
      }
    }
    __syncthreads();
  }
}

// ---- 4. projection energies ------------------------------------------------------------------------------------
// grid (tiles, items), 256 threads; warp w owns output samples [16 w, 16 w + 16) of the tile (2 m-tiles), all
// NS n-tiles of estimates.  G and Gb hold the filters in their right-hand columns.  sums (items, tiles, K + 1, 3,
// 8 NS): slot j < K: sum P_j^2, sum (x - P_j)^2, sum (P_all - P_j)^2; slot K: sum P_all^2, sum (x - P_all)^2, 0.
template <int NS>
struct ProjSmem {
  double coef[8 * NS][kBssL + 4];
  double seg[kProjTile + kBssL];
  double red[8][3][8 * NS];
};

template <int NS>
__device__ __forceinline__ void bss_project_pass(ProjSmem<NS>& sm, const double* __restrict__ src, long long T,
                                                 long long t0, const double* __restrict__ filt, int ldf, int E,
                                                 double (&acc)[2][NS][2]) {
  // the filter of estimate e is column e of filt: filt[tau * ldf + e]
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * NS * kBssL; i += blockDim.x) {
    const int e = i / kBssL, tau = i % kBssL;
    sm.coef[e][tau] = e < E ? filt[(long long)tau * ldf + e] : 0.0;
  }
  for (int i = threadIdx.x; i < kProjTile + kBssL - 1; i += blockDim.x) {
    const long long t = t0 - (kBssL - 1) + i;
    sm.seg[i] = t >= 0 && t < T ? src[t] : 0.0;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, q = lane & 3;
#pragma unroll 4
  for (int k = 0; k < kBssL; k += 4) {
    double b[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) b[n] = sm.coef[8 * n + r][k + q];
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      // A[t, tau] = s[t - tau], t = t0 + 16 warp + 8 m + r, tau = k + q
      const double av = sm.seg[16 * warp + 8 * m + r - (k + q) + kBssL - 1];
#pragma unroll
      for (int n = 0; n < NS; ++n) dmma(acc[m][n], av, b[n]);
    }
  }
}

template <int NS>
__global__ void __launch_bounds__(256) bss_project_kernel(const double* __restrict__ x, BssShape sh,
                                                          const double* __restrict__ G, const double* __restrict__ Gb,
                                                          double* __restrict__ sums) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ProjSmem<NS>& sm = *reinterpret_cast<ProjSmem<NS>*>(smem_raw);
  const long long tile = blockIdx.x, item = blockIdx.y, t0 = tile * kProjTile;
  const int K = sh.K, E = sh.E, N = sh.N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, q = lane & 3;
  const double* sig = x + item * sh.S * sh.T;
  const double* Gi = G + item * (long long)N * (N + kRhsPad);
  const long long Tp = sh.T + kBssL - 1;
  double pall[2][NS][2], xv[2][NS][2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < NS; ++n)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        pall[m][n][c] = 0.0;
        const long long t = t0 + 16 * warp + 8 * m + r;
        const int e = 8 * n + 2 * q + c;
        xv[m][n][c] = e < E && t < sh.T ? sig[(long long)(K + e) * sh.T + t] : 0.0;
      }
  for (int i = 0; i < K; ++i)
    bss_project_pass<NS>(sm, sig + (long long)i * sh.T, sh.T, t0, Gi + (long long)i * kBssL * (N + kRhsPad) + N,
                         N + kRhsPad, E, pall);
  double* out = sums + (item * sh.tiles + tile) * (K + 1) * 3 * 8 * NS;
  // per-thread sums over its rows, warp sums over the 8 row groups (lanes of equal q), warp partials in shared
  // memory, and the 8 warps in order
  auto flush = [&](double (&v)[3][NS][2], int slot) {
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int n = 0; n < NS; ++n)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          double w = v[s][n][c];
          w += __shfl_xor_sync(0xffffffffu, w, 4);
          w += __shfl_xor_sync(0xffffffffu, w, 8);
          w += __shfl_xor_sync(0xffffffffu, w, 16);
          if (r == 0) sm.red[warp][s][8 * n + 2 * q + c] = w;
        }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * 8 * NS; i += blockDim.x) {
      const int s = i / (8 * NS), e = i % (8 * NS);
      double w = 0.0;
      for (int wi = 0; wi < 8; ++wi) w += sm.red[wi][s][e];
      out[(long long)slot * 3 * 8 * NS + i] = w;
    }
    __syncthreads();
  };
  double v[3][NS][2];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < NS; ++n)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const long long t = t0 + 16 * warp + 8 * m + r;
        const bool ok = t < Tp;
        const double p = ok ? pall[m][n][c] : 0.0, d = ok ? xv[m][n][c] - pall[m][n][c] : 0.0;
        if (m == 0) { v[0][n][c] = p * p; v[1][n][c] = d * d; v[2][n][c] = 0.0; }
        else { v[0][n][c] = fma(p, p, v[0][n][c]); v[1][n][c] = fma(d, d, v[1][n][c]); }
      }
  flush(v, K);
  for (int j = 0; j < K; ++j) {
    double pj[2][NS][2];
    if (K == 1) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < NS; ++n) { pj[m][n][0] = pall[m][n][0]; pj[m][n][1] = pall[m][n][1]; }
    } else {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < NS; ++n) pj[m][n][0] = pj[m][n][1] = 0.0;
      bss_project_pass<NS>(sm, sig + (long long)j * sh.T, sh.T, t0,
                           Gb + (item * K + j) * (long long)kBssL * (kBssL + kRhsPad) + kBssL, kBssL + kRhsPad, E, pj);
    }
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int n = 0; n < NS; ++n)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const long long t = t0 + 16 * warp + 8 * m + r;
          const bool ok = t < Tp;
          const double p = ok ? pj[m][n][c] : 0.0, d = ok ? xv[m][n][c] - pj[m][n][c] : 0.0,
                       f = ok ? pall[m][n][c] - pj[m][n][c] : 0.0;
          if (m == 0) { v[0][n][c] = p * p; v[1][n][c] = d * d; v[2][n][c] = f * f; }
          else {
            v[0][n][c] = fma(p, p, v[0][n][c]);
            v[1][n][c] = fma(d, d, v[1][n][c]);
            v[2][n][c] = fma(f, f, v[2][n][c]);
          }
        }
    flush(v, j);
  }
}

// ---- 5. ratios and the permutation ----------------------------------------------------------------------------
__device__ __forceinline__ double safe_db(double num, double den) {
  return den == 0.0 ? CUDART_INF : 10.0 * log10(num / den);
}

// np.mean of K values: numpy's pairwise sum (sequential from 0 below 8 values, eight partial sums at 8) over K
__device__ __forceinline__ double np_mean(const double* v, int K) {
  double s;
  if (K < 8) {
    s = 0.0;
    for (int k = 0; k < K; ++k) s += v[k];
  } else {
    s = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
  }
  return s / K;
}

// one CTA (256 threads) per item; pairs (items, 3, E, K) may be null
__global__ void __launch_bounds__(256) bss_ratio_kernel(const double* __restrict__ sums, BssShape sh, int permute,
                                                        const int* __restrict__ flags, long long item0,
                                                        double* __restrict__ sdr, double* __restrict__ sir,
                                                        double* __restrict__ sar, long long* __restrict__ selection,
                                                        double* __restrict__ pairs) {
  constexpr int kMaxE = PBB_BSS_EVAL_MAX_SOURCES + 1;
  __shared__ double tot[PBB_BSS_EVAL_MAX_SOURCES + 1][3][kRhsPad];
  __shared__ double rat[3][kMaxE][PBB_BSS_EVAL_MAX_SOURCES];
  __shared__ double best_v[256];
  __shared__ long long best_i[256];
  __shared__ int best_nan[256];
  const long long item = blockIdx.x, g = item0 + item;
  const int K = sh.K, E = sh.E, tid = threadIdx.x;
  const int W = sh.E > 8 ? 16 : 8;   // 8 NS
  const long long per = (long long)(K + 1) * 3 * W;
  for (int i = tid; i < per; i += blockDim.x) {
    const double* p = sums + item * sh.tiles * per + i;
    double s = 0.0;
    for (long long t = 0; t < sh.tiles; ++t) s += p[t * per];
    const int slot = i / (3 * W), qq = (i / W) % 3, e = i % W;
    if (e < kRhsPad) tot[slot][qq][e] = s;
  }
  __syncthreads();
  const bool bad = flags[item] != 0;
  for (int i = tid; i < E * K; i += blockDim.x) {
    const int e = i / K, j = i % K;
    const double nan = CUDART_NAN;
    const double vd = bad ? nan : safe_db(tot[j][0][e], tot[j][1][e]);
    const double vi = bad ? nan : safe_db(tot[j][0][e], tot[j][2][e]);
    const double va = bad ? nan : safe_db(tot[K][0][e], tot[K][1][e]);
    rat[0][e][j] = vd;
    rat[1][e][j] = vi;
    rat[2][e][j] = va;
    if (pairs != nullptr) {
      double* pp = pairs + g * 3 * E * K;
      pp[i] = vd;
      pp[E * K + i] = vi;
      pp[2 * E * K + i] = va;
    }
  }
  __syncthreads();
  if (!permute) {
    if (tid < K) {
      sdr[g * K + tid] = rat[0][tid][tid];
      sir[g * K + tid] = rat[1][tid][tid];
      sar[g * K + tid] = rat[2][tid][tid];
    }
    return;
  }
  // itertools.permutations(range(E), K) in lexicographic order; thread tid takes ranks tid, tid + 256, ...
  long long nperm = 1;
  for (int k = 0; k < K; ++k) nperm *= E - k;
  double bv = -CUDART_INF;
  long long bidx = -1;
  int has_nan = 0;
  for (long long idx = tid; idx < nperm; idx += blockDim.x) {
    long long rest = idx, block = nperm;
    unsigned used = 0;
    double v[PBB_BSS_EVAL_MAX_SOURCES];
    for (int k = 0; k < K; ++k) {
      block /= E - k;
      int d = (int)(rest / block);
      rest %= block;
      int e = 0;
      for (;; ++e)
        if (!(used >> e & 1u) && d-- == 0) break;
      used |= 1u << e;
      v[k] = rat[1][e][k];
    }
    const double m = np_mean(v, K);
    if (has_nan) continue;
    if (m != m) { has_nan = 1; bidx = idx; }
    else if (bidx < 0 || m > bv) { bv = m; bidx = idx; }
  }
  best_v[tid] = bv;
  best_i[tid] = bidx;
  best_nan[tid] = has_nan;
  __syncthreads();
  if (tid == 0) {
    // np.argmax: the first NaN if there is one, else the first maximum
    long long pick = -1;
    double pv = -CUDART_INF;
    bool nan_seen = false;
    for (int t = 0; t < (int)blockDim.x; ++t) {
      if (best_i[t] < 0) continue;
      if (best_nan[t]) {
        if (!nan_seen || best_i[t] < pick) pick = best_i[t];
        nan_seen = true;
      } else if (!nan_seen && (pick < 0 || best_v[t] > pv || (best_v[t] == pv && best_i[t] < pick))) {
        pv = best_v[t];
        pick = best_i[t];
      }
    }
    long long rest = pick, block = nperm;
    unsigned used = 0;
    for (int k = 0; k < K; ++k) {
      block /= E - k;
      int d = (int)(rest / block);
      rest %= block;
      int e = 0;
      for (;; ++e)
        if (!(used >> e & 1u) && d-- == 0) break;
      used |= 1u << e;
      sdr[g * K + k] = rat[0][e][k];
      sir[g * K + k] = rat[1][e][k];
      sar[g * K + k] = rat[2][e][k];
      selection[g * K + k] = e;
    }
  }
}

// status = ((item + 1) << 3) | flags of the first flagged item, unless an earlier group set it already
__global__ void bss_status_kernel(const int* __restrict__ flags, long long items, long long item0,
                                  long long* __restrict__ status) {
  if (threadIdx.x != 0 || *status != 0) return;
  for (long long i = 0; i < items; ++i)
    if (flags[i]) {
      *status = ((item0 + i + 1) << 3) | flags[i];
      return;
    }
}

}  // namespace pbb
