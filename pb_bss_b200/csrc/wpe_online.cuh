// Frame-online WPE (nara_wpe.wpe.online_wpe_step, and online_wpe: the step over a whole stream) -- see
// include/pbb.h.
//
// One CTA per bin runs the recursive least-squares recursion over all T frames of a launch.  n = taps D <= 96.
// The inverse correlation Q (n x n complex) lives in registers for the whole launch: the 256 threads form a 16 x 16
// grid, thread (r, c) owns the R x R entries Q[r + 16 i][c + 16 j] (R = ceil(n / 16) <= 6, a template argument; the
// rows and columns past n stay zero).  The filter G is kept in shared memory channel-major, G_s[d][i] = G[i][d], and
// the last taps + delay + 1 frames in a ring.  Per frame t:
//   A. warp 7 stores the (prefetched) frame y_t in the ring, forms its power mean_d |y_dt|^2 and lambda_t, the mean
//      of the ring's taps + delay + 1 frame powers summed from the oldest frame (or takes lambda from the caller),
//      then prefetches y_{t+1}.  Every thread makes one pass over its Q entries that forms its partial sums of both
//      u = Q w (over its columns) and v = w^H Q (over its rows); u is summed over the 16 column threads by
//      shuffles, v over the row pair of a warp by a shuffle and over the eight warps in shared memory.
//   -- barrier
//   B. every warp forms den = alpha lambda + w^H u by the same fixed-order sum, so den needs no barrier; every
//      thread sums the eight v partials of its columns in warp order, forms k = u / den for its rows and updates its
//      entries Q <- (Q - k v) / alpha.  Warp d mod 8 forms pred_d = y_d - G[:, d]^H w, stores it to z and updates
//      G[:, d] += k conj(pred_d).  Threads < n build the next frame's window in the other window buffer.
//   -- barrier
// Two barriers per frame; the reductions on the critical path are the 4-level u shuffle, the 8-way v sum, the
// 5-level den shuffle and, for pred, n / 32 multiply-adds and a 5-level shuffle per channel of a warp.
// Every sum has a fixed order and the power of a frame is recomputed from the ring in frame-age order, never kept as
// a running sum: a stream split into several launches (the history and Q, G passed on) is bitwise equal to one.
#pragma once
#include "wpe.cuh"

namespace pbb {

constexpr int kWpeOnlineThreads = 256;
constexpr int kWpeOnlineSmemMax = 232448;  // opt-in shared memory of one CTA on sm_90 (227 KB)

struct WpeOnlineShape {
  long long T;
  int D, taps, delay, n, L;  // L = taps + delay + 1 frames in the buffer
  double alpha, inv_alpha;
};

// window buffers (2 x 96), u (96), v partials (8 x 96), G (D x n), ring (L x D) complex; frame powers (L), lambda
__host__ __device__ inline size_t wpe_online_smem_bytes(int D, int taps, int delay) {
  const size_t n = (size_t)taps * D, L = (size_t)taps + delay + 1;
  return sizeof(double2) * (11 * (size_t)kWpeMaxN + D * n + L * D) + sizeof(double) * (L + 1);
}

__device__ __forceinline__ double2 wpe_cfma(double2 a, double2 b, double2 c) {  // c + a b
  return make_double2(__fma_rn(a.x, b.x, __fma_rn(-a.y, b.y, c.x)), __fma_rn(a.x, b.y, __fma_rn(a.y, b.x, c.y)));
}
__device__ __forceinline__ double2 wpe_cfmac(double2 a, double2 b, double2 c) {  // c + conj(a) b
  return make_double2(__fma_rn(a.x, b.x, __fma_rn(a.y, b.y, c.x)), __fma_rn(a.x, b.y, __fma_rn(-a.y, b.x, c.y)));
}
__device__ __forceinline__ double2 wpe_cadd(double2 a, double2 b) {
  return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y));
}
__device__ __forceinline__ double2 wpe_shfl_xor(double2 v, int o) {
  return make_double2(__shfl_xor_sync(0xffffffffu, v.x, o), __shfl_xor_sync(0xffffffffu, v.y, o));
}
// butterfly sum over the 32 lanes: every lane ends with the same bits
__device__ __forceinline__ double2 wpe_warp_csum(double2 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = wpe_cadd(v, wpe_shfl_xor(v, o));
  return v;
}
__device__ __forceinline__ double wpe_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// mean_d |x_d|^2 of one frame, x = this lane's channel (zero for lanes >= D); the whole warp calls it
__device__ __forceinline__ double wpe_frame_power(double2 x, int D) {
  return __ddiv_rn(wpe_warp_sum(__fma_rn(x.x, x.x, __dmul_rn(x.y, x.y))), (double)D);
}

// grid (bins), 256 threads.  y (b, d, t) T frames; hist (b, d, t) the L - 1 frames before them (null: zeros);
// power (bins) lambda of the only frame when not null (T = 1); Qin (bins, n, n), Gin (bins, n, D) complex128
// row-major (null: identity, zeros); z (b, d, t) the predictions; Qout, Gout like Qin, Gin (may be Qin, Gin).
template <int R, class TIn>
__global__ void __launch_bounds__(kWpeOnlineThreads, 1)
    wpe_online_kernel(const TIn* __restrict__ y, WpeStrides ys, const TIn* __restrict__ hist, WpeStrides hs,
                      const double* __restrict__ power, const double2* Qin, const double2* Gin, TIn* __restrict__ z,
                      WpeStrides zs, double2* Qout, double2* Gout, WpeOnlineShape s) {
  extern __shared__ __align__(16) double2 osm[];
  const int D = s.D, n = s.n, L = s.L;
  double2* wsm = osm;                       // [2][96] windows of even and odd frames, zero past n
  double2* usm = wsm + 2 * kWpeMaxN;        // [96] u
  double2* vsm = usm + kWpeMaxN;            // [8][96] per-warp partials of v
  double2* gsm = vsm + 8 * kWpeMaxN;        // [D][n] G, channel-major
  double2* ring = gsm + D * n;              // [L][D] frame g in slot g mod L
  double* psm = reinterpret_cast<double*>(ring + L * D);  // [L] frame powers, same slots
  double* lsm = psm + L;                    // lambda of the current frame
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, tr = tid >> 4, tc = tid & 15;
  const long long bin = blockIdx.x;
  y += bin * ys.b;
  z += bin * zs.b;
  if (hist) hist += bin * hs.b;
  const double2 zero = make_double2(0.0, 0.0);

  double2 q[R][R];
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const int r = tr + 16 * i, c = tc + 16 * j;
      q[i][j] = zero;
      if (r < n && c < n)
        q[i][j] = Qin ? Qin[(bin * n + r) * n + c] : make_double2(r == c ? 1.0 : 0.0, 0.0);
    }
  for (int e = tid; e < n * D; e += kWpeOnlineThreads) {
    const int i = e / D, d = e - i * D;
    gsm[d * n + i] = Gin ? Gin[bin * n * D + e] : zero;
  }
  for (int e = tid; e < 2 * kWpeMaxN; e += kWpeOnlineThreads) wsm[e] = zero;
  for (int e = tid; e < (L - 1) * D; e += kWpeOnlineThreads) {
    const int g = e / D, d = e - g * D;
    ring[e] = hist ? wpe_load(hist, g * hs.t + d * hs.d) : zero;
  }
  __syncthreads();
  for (int g = warp; g < L - 1; g += kWpeOnlineThreads / 32) {
    const double p = wpe_frame_power(lane < D ? ring[g * D + lane] : zero, D);
    if (lane == 0) psm[g] = p;
  }
  // window of frame 0 (global frame L - 1): w[d taps + k] = frame L - 2 - delay - k = taps - 1 - k
  if (tid < n) {
    const int d = tid / s.taps, k = tid - d * s.taps;
    wsm[tid] = ring[(s.taps - 1 - k) * D + d];
  }
  double2 ynext = zero;
  if (warp == 7 && lane < D && s.T > 0) ynext = wpe_load(y, lane * ys.d);
  __syncthreads();

  for (long long t = 0; t < s.T; ++t) {
    const int par = (int)(t & 1);
    const double2* wv = wsm + par * kWpeMaxN;
    const long long gt = t + L - 1;  // global frame index: the history holds frames 0 .. L - 2
    const int slot = (int)(gt % L);
    // ---- A. ingest y_t and lambda_t (warp 7); u and v partials (all)
    if (warp == 7) {
      if (lane < D) ring[slot * D + lane] = ynext;
      const double p = wpe_frame_power(ynext, D);
      if (lane == 0) psm[slot] = p;
      __syncwarp();
      double lam;
      if (power) {
        lam = power[bin];
      } else {
        double acc = 0.0;  // frame powers from the oldest frame of the buffer (global frame gt - L + 1)
        for (int j = lane; j < L; j += 32) acc = __dadd_rn(acc, psm[(int)((gt + 1 + j) % L)]);
        lam = __ddiv_rn(wpe_warp_sum(acc), (double)L);
      }
      if (lane == 0) *lsm = lam;
      if (t + 1 < s.T && lane < D) ynext = wpe_load(y, (t + 1) * ys.t + lane * ys.d);
    }
    // row i: u over the columns j in order, then its 16-lane sum; v of column j sums the rows i in order
    double2 wc[R], vp[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      wc[j] = wv[tc + 16 * j];
      vp[j] = zero;
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const double2 wr = wv[tr + 16 * i];
      double2 up = zero;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        up = wpe_cfma(q[i][j], wc[j], up);
        vp[j] = wpe_cfmac(wr, q[i][j], vp[j]);
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) up = wpe_cadd(up, wpe_shfl_xor(up, o));
      if (tc == 0) usm[tr + 16 * i] = up;
    }
#pragma unroll
    for (int j = 0; j < R; ++j) {
      vp[j] = wpe_cadd(vp[j], wpe_shfl_xor(vp[j], 16));
      if (lane < 16) vsm[warp * kWpeMaxN + tc + 16 * j] = vp[j];
    }
    __syncthreads();
    // ---- B. den (every warp, same sum), the rank-1 update of Q, pred and G, the next window
    const double lam = *lsm;
    double2 acc = zero;
    for (int e = lane; e < n; e += 32) acc = wpe_cfmac(wv[e], usm[e], acc);
    acc = wpe_warp_csum(acc);
    const double2 den = make_double2(__dadd_rn(s.alpha * lam, acc.x), acc.y);
    double2 vj[R], ki[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      double2 v = vsm[tc + 16 * j];
#pragma unroll
      for (int w = 1; w < 8; ++w) v = wpe_cadd(v, vsm[w * kWpeMaxN + tc + 16 * j]);
      vj[j] = v;
      ki[j] = cdiv(usm[tr + 16 * j], den);
    }
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const double2 kv = cmul(ki[i], vj[j]);
        q[i][j] = make_double2(__dmul_rn(__dadd_rn(q[i][j].x, -kv.x), s.inv_alpha),
                               __dmul_rn(__dadd_rn(q[i][j].y, -kv.y), s.inv_alpha));
      }
    for (int d = warp; d < D; d += kWpeOnlineThreads / 32) {
      double2 g = zero;
      for (int e = lane; e < n; e += 32) g = wpe_cfmac(gsm[d * n + e], wv[e], g);
      g = wpe_warp_csum(g);
      const double2 yv = ring[slot * D + d];
      const double2 pred = make_double2(__dadd_rn(yv.x, -g.x), __dadd_rn(yv.y, -g.y));
      if (lane == 0) wpe_store(z, t * zs.t + d * zs.d, pred);
      const double2 pc = make_double2(pred.x, -pred.y);
      for (int e = lane; e < n; e += 32) gsm[d * n + e] = wpe_cadd(gsm[d * n + e], cmul(cdiv(usm[e], den), pc));
    }
    if (tid < n) {  // window of frame t + 1: w[d taps + k] = global frame gt - delay - k
      const int d = tid / s.taps, k = tid - d * s.taps;
      wsm[(par ^ 1) * kWpeMaxN + tid] = ring[(int)((gt - s.delay - k) % L) * D + d];
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const int r = tr + 16 * i, c = tc + 16 * j;
      if (r < n && c < n) Qout[(bin * n + r) * n + c] = q[i][j];
    }
  for (int e = tid; e < n * D; e += kWpeOnlineThreads) {
    const int i = e / D, d = e - i * D;
    Gout[bin * n * D + e] = gsm[d * n + i];
  }
}

}  // namespace pbb
