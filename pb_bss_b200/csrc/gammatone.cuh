// The gammatone filterbank (pbb_gammatone in include/pbb.h): four direct-form-II-transposed second-order sections
// per filter, one 8-state linear recurrence, made parallel over time by a scan over chunks of L samples.
//
//   gammatone_chunk_kernel<T, false>  zero-start end state of every (row, filter, chunk) -> state workspace
//   gammatone_carry_kernel            s_{c+1} = M s_c + z_c over the chunks of every (row, filter), in place: the
//                                     workspace then holds every chunk's start state.  Two levels: the end states of
//                                     groups of kGtGroup chunks, a carry over the groups with M^kGtGroup, then the
//                                     chunks of every group from its start; the sequential depth is 2 kGtGroup + C /
//                                     kGtGroup steps instead of C.
//   gammatone_chunk_kernel<T, true>   every chunk again from its start state, writing the output
//
// The chunk passes: a CTA owns 32 consecutive chunks of the flattened (row, chunk) index (chunks of several rows when
// the rows are short) and kGtFilters filters, one warp per filter and one lane per chunk.  The CTA stages the input of
// its 32 chunks in steps of kGtStep samples in shared memory, read once for its filters, and each warp stages its
// outputs the same way, so both the loads and the stores move whole 128-byte runs of one chunk.
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kGtFilters = 8;                    // filters (warps) per CTA of the chunk passes
constexpr int kGtThreads = 32 * kGtFilters;
constexpr int kGtStep = 16;                      // samples per staged step
constexpr int kGtGroup = PBB_GAMMATONE_CARRY_GROUP;
constexpr int kGtCoef = 10;                      // b0, b1 of the four sections, a1, a2

struct GtParams {
  const void* x;          // (rows, N)
  long long rows, N;
  long long chunks;       // C = ceil(N / L)
  long long total;        // rows * C
  long long groups;       // ceil(C / kGtGroup)
  int n, L;
  const double* coef;     // (n, kGtCoef)
  const double* trans;    // (n, 2, 8, 8): M, M^kGtGroup
  double* state;          // (rows * n, C, 8): end states, then start states
  double* group;          // (rows * n, groups, 8)
  double* out;            // (n, rows, N)
};

// One sample through the cascade.  u <- b1 w + v - a1 y keeps y -> u -> y at two dependent FMAs per sample.
struct GtCascade {
  double b0[4], b1[4], na1, na2;
  double u[4], v[4];
  __device__ __forceinline__ double step(double w) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double y = fma(b0[k], w, u[k]);
      u[k] = fma(na1, y, fma(b1[k], w, v[k]));
      v[k] = na2 * y;
      w = y;
    }
    return w;
  }
};

template <class T, bool kOutput>
__global__ void __launch_bounds__(kGtThreads, 3) gammatone_chunk_kernel(const GtParams p) {
  __shared__ double xs[2][32][kGtStep + 1];
  __shared__ double ys[kOutput ? kGtFilters : 1][32][kGtStep + 1];
  __shared__ long long cbase[32];                // row * N + c * L of each chunk of the CTA
  __shared__ int clen[32];                       // its samples (0 past the last chunk)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long nft = (p.n + kGtFilters - 1) / kGtFilters;
  const long long cg = blockIdx.x / nft;
  const int f = (int)(blockIdx.x % nft) * kGtFilters + warp;
  const long long g = cg * 32 + lane;            // this lane's chunk
  const long long row = g / p.chunks, c = g - row * p.chunks;
  if (threadIdx.x < 32) {
    const bool ok = g < p.total;
    cbase[lane] = ok ? row * p.N + c * p.L : 0;
    clen[lane] = ok ? (int)min((long long)p.L, p.N - c * p.L) : 0;
  }
  const bool active = f < p.n;                   // warp-uniform
  const bool mine = active && g < p.total;
  GtCascade cs;
  double* st = p.state + (((row * p.n + f) * p.chunks + c) << 3);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    cs.b0[k] = active ? p.coef[f * kGtCoef + 2 * k] : 0.0;
    cs.b1[k] = active ? p.coef[f * kGtCoef + 2 * k + 1] : 0.0;
    const bool carried = kOutput && mine && p.chunks > 1;
    cs.u[k] = carried ? st[2 * k] : 0.0;
    cs.v[k] = carried ? st[2 * k + 1] : 0.0;
  }
  cs.na1 = active ? -p.coef[f * kGtCoef + 8] : 0.0;
  cs.na2 = active ? -p.coef[f * kGtCoef + 9] : 0.0;
  __syncthreads();
  const T* __restrict__ x = static_cast<const T*>(p.x);
  double* __restrict__ out = p.out + (long long)f * p.rows * p.N;
  const int run = p.chunks == 1 ? (int)p.N : p.L;
  for (int j0 = 0; j0 < run; j0 += kGtStep) {
    double(*xb)[kGtStep + 1] = xs[(j0 / kGtStep) & 1];  // double buffer: one barrier per step
#pragma unroll
    for (int e = threadIdx.x; e < 32 * kGtStep; e += kGtThreads) {
      const int cc = e / kGtStep, s = e % kGtStep, t = j0 + s;
      xb[cc][s] = t < clen[cc] ? (double)x[cbase[cc] + t] : 0.0;
    }
    __syncthreads();
    if (active) {
#pragma unroll
      for (int s = 0; s < kGtStep; ++s) {
        const double y = cs.step(xb[lane][s]);
        if (kOutput) ys[warp][lane][s] = y;
      }
      if (kOutput) {
        __syncwarp();
        const int s = lane % kGtStep, t = j0 + s;
#pragma unroll 4
        for (int cc = lane / kGtStep; cc < 32; cc += 32 / kGtStep)
          if (t < clen[cc]) out[cbase[cc] + t] = ys[warp][cc][s];
        __syncwarp();
      }
    }
  }
  if (!kOutput && mine) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      st[2 * k] = cs.u[k];
      st[2 * k + 1] = cs.v[k];
    }
  }
}

// r = add + m s over the 8 lanes of a unit (lane i holds s_i and row i of the matrix); two accumulators halve the
// dependent chain.
__device__ __forceinline__ double gt_matvec(const double (&m)[8], double s, double add, unsigned mask) {
  double r0 = add, r1 = 0.0;
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    r0 = fma(m[j], __shfl_sync(mask, s, j, 8), r0);
    r1 = fma(m[j + 1], __shfl_sync(mask, s, j + 1, 8), r1);
  }
  return r0 + r1;
}

// One CTA per (row, filter) sequence; units of 8 lanes, one state component per lane.
__global__ void __launch_bounds__(256) gammatone_carry_kernel(const GtParams p) {
  const long long q = blockIdx.x;                // row * n + f
  const int f = (int)(q % p.n);
  const int unit = threadIdx.x >> 3, i = threadIdx.x & 7, units = blockDim.x >> 3;
  const unsigned mask = 0xffu << (threadIdx.x & 24);
  const long long C = p.chunks, NG = p.groups;
  double* z = p.state + q * C * 8;
  double* gs = p.group + q * NG * 8;
  const double* tr = p.trans + (size_t)f * 128;
  double m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = tr[i * 8 + j];
  // The group's end states are loaded into registers up front, so the sequential steps wait on no memory.
  double zc[kGtGroup];
  // end state of every group but the last, from zero
  for (long long gi = unit; gi < NG - 1; gi += units) {
#pragma unroll
    for (int k = 0; k < kGtGroup; ++k) zc[k] = z[(gi * kGtGroup + k) * 8 + i];
    double e = 0.0;
#pragma unroll
    for (int k = 0; k < kGtGroup; ++k) e = gt_matvec(m, e, zc[k], mask);
    gs[gi * 8 + i] = e;
  }
  __syncthreads();
  // start state of every group: S_0 = 0, S_{g+1} = M^kGtGroup S_g + E_g (in place; E_{g+1} is loaded one step ahead)
  if (unit == 0) {
    double mg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) mg[j] = tr[64 + i * 8 + j];
    double s = 0.0, next = NG > 1 ? gs[i] : 0.0;
    for (long long gi = 0; gi < NG - 1; ++gi) {
      const double e = next;
      if (gi + 2 < NG) next = gs[(gi + 1) * 8 + i];
      gs[gi * 8 + i] = s;
      s = gt_matvec(mg, s, e, mask);
    }
    gs[(NG - 1) * 8 + i] = s;
  }
  __syncthreads();
  // start state of every chunk (in place over its end state)
  for (long long gi = unit; gi < NG; gi += units) {
#pragma unroll
    for (int k = 0; k < kGtGroup; ++k) {
      const long long c = gi * kGtGroup + k;
      zc[k] = c < C ? z[c * 8 + i] : 0.0;
    }
    double s = gs[gi * 8 + i];
#pragma unroll
    for (int k = 0; k < kGtGroup; ++k) {
      const long long c = gi * kGtGroup + k;
      if (c < C) z[c * 8 + i] = s;
      s = gt_matvec(m, s, zc[k], mask);
    }
  }
}

}  // namespace pbb
