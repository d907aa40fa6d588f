// k-means of sklearn.cluster.KMeans(n_clusters=K) as pb_bss/distribution/gmm.py:201-230 (BinaryGMMTrainer) calls it:
// centring (KMeans.fit), _tolerance, _kmeans_plusplus, _kmeans_single_lloyd with lloyd_iter_chunked_dense,
// _relocate_empty_clusters_dense, _average_centers, _center_shift and _inertia_dense, and KMeans.predict.  fp64.
//
// Every reduction runs in an order fixed by N alone: the points are split into at most kKmMaxChunks contiguous
// chunks (km_chunking), a chunk is always worked by one CTA of kKmThreads threads in a fixed pattern, and chunk
// partials are combined in chunk order.  No float atomics, so results are bitwise repeatable and do not depend on
// the grid size.  The fit runs as two cooperative launches with grid-wide barriers (grid_barrier, common.cuh).
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kKmThreads = 128;    // block size of every k-means kernel: the fixed reduction trees assume it
constexpr int kKmTile = 128;       // points per staged tile of the Lloyd E-step (one per thread)
constexpr int kKmMaxChunks = 256;
constexpr int kKmMaxK = PBB_KMEANS_MAX_K, kKmMaxE = PBB_KMEANS_MAX_E, kKmMaxTrials = 4;  // 2 + int(log 16)
constexpr int kKmPairsPerThread = (kKmMaxK * kKmMaxE + kKmThreads - 1) / kKmThreads;

struct KmChunks {
  long long cs;  // points per chunk (the last one may be shorter)
  int nch;
};
__host__ __device__ inline KmChunks km_chunking(long long N) {
  long long n0 = (N + 127) / 128;
  if (n0 > kKmMaxChunks) n0 = kKmMaxChunks;
  if (n0 < 1) n0 = 1;
  const long long cs = (N + n0 - 1) / n0;
  return {cs, (int)((N + cs - 1) / cs)};
}
__host__ __device__ inline int km_trials(int K) {  // n_local_trials = 2 + int(np.log(K))
  return K >= 8 ? 4 : (K >= 3 ? 3 : 2);             // log 3 = 1.10, log 8 = 2.08, log 16 = 2.77
}

// Workspace layout (pbb_kmeans_workspace_bytes): doubles first, then 64-bit integers.
struct KmWork {
  double *xc, *xn, *closest, *dtc, *cum;         // N*E, N, N, L*N, N
  double *part_col, *part_var, *part_pot, *part_tot, *part_sum, *part_val;  // per chunk
  double *mean, *tol, *cinit, *sums;             // E, 1, K*E, K*E + K
  long long *part_cnt, *part_idx;                // nch*L, nch
  unsigned *bar;                                 // two barrier counters
};
__host__ __device__ inline size_t km_layout(long long N, int E, int K, char* base, KmWork* w) {
  const KmChunks ch = km_chunking(N);
  const int L = km_trials(K);
  const size_t nch = (size_t)ch.nch, KE = (size_t)K * E;
  size_t o = 0;
  double* d = reinterpret_cast<double*>(base);
  auto take = [&](size_t n) { double* p = d ? d + o : nullptr; o += n; return p; };
  double* xc = take((size_t)N * E);
  double* xn = take(N);
  double* closest = take(N);
  double* dtc = take((size_t)L * N);
  double* cum = take(N);
  double* part_col = take(nch * E);
  double* part_var = take(nch * E);
  double* part_pot = take(nch * L);
  double* part_tot = take(nch);
  double* part_sum = take(nch * (KE + K));
  double* part_val = take(nch);
  double* mean = take(E);
  double* tol = take(1);
  double* cinit = take(KE);
  double* sums = take(KE + K);
  size_t bytes = o * sizeof(double);
  long long* ip = base ? reinterpret_cast<long long*>(base + bytes) : nullptr;
  bytes += (nch * L + nch) * sizeof(long long);
  unsigned* bar = base ? reinterpret_cast<unsigned*>(base + bytes) : nullptr;
  bytes += 4 * sizeof(unsigned);
  if (w) *w = {xc, xn, closest, dtc, cum, part_col, part_var, part_pot, part_tot, part_sum, part_val,
               mean, tol, cinit, sums, ip, ip ? ip + nch * L : nullptr, bar};
  return bytes;
}

// Sum over the kKmThreads threads in a fixed tree (all threads receive it).
__device__ inline double km_block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const double s = (red[0] + red[1]) + (red[2] + red[3]);
  __syncthreads();
  return s;
}

// Largest value, first index on ties, over the kKmThreads threads (all threads receive it).  idx < 0 = none.
__device__ inline void km_block_argmax(double& v, long long& idx, double* red, long long* redi) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (oi >= 0 && (idx < 0 || ov > v || (ov == v && oi < idx))) { v = ov; idx = oi; }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) { red[warp] = v; redi[warp] = idx; }
  __syncthreads();
  v = red[0]; idx = redi[0];
  for (int w = 1; w < kKmThreads / 32; ++w)
    if (redi[w] >= 0 && (idx < 0 || red[w] > v || (red[w] == v && redi[w] < idx))) { v = red[w]; idx = redi[w]; }
  __syncthreads();
}

// _euclidean_distances(a, X, Y_norm_squared=x_squared_norms, squared=True) of sklearn.metrics.pairwise for one
// point: max((-2 a.x + |a|^2) + |x|^2, 0)
__device__ __forceinline__ double km_sq_dist(const double* __restrict__ a, double an, const double* __restrict__ x,
                                             double xn, int E) {
  double dot = 0.0;
  for (int e = 0; e < E; ++e) dot = fma(a[e], x[e], dot);
  return fmax(__dadd_rn(__dadd_rn(-2.0 * dot, an), xn), 0.0);
}

// KMeans.fit up to the initial centres.  Phases, separated by grid barriers:
//   1. column sums per chunk, non-finite check;  2. X_mean, the centred copy xc = x - X_mean, the row norms
//   (row_norms(X, squared=True)) and the column sums of squares of xc (np.var);  3. _tolerance; with init the
//   initial centres init - X_mean, else _kmeans_plusplus: the first centre xc[first] and its closest distances,
//   then K - 1 rounds of (a) the inclusive scan of closest_dist_sq, (b) np.searchsorted of uniforms * current_pot
//   (as the count of scan values below each target, clipped to N - 1), (c) the candidates' distances and potentials,
//   and the first argmin of the potentials.  cum[i] = chunk prefix + (thread-run prefix + sequential run sum).
__global__ void __launch_bounds__(kKmThreads, 1) kmeans_init_kernel(const double* __restrict__ x, long long N, int E,
                                                                  int K, long long first,
                                                                  const double* __restrict__ uniforms,
                                                                  const double* __restrict__ init, KmWork w,
                                                                  int* status) {
  __shared__ double red[32];
  __shared__ long long redi[32];
  __shared__ double colpart[kKmThreads];
  __shared__ double smean[kKmMaxE];
  __shared__ double runpre[kKmThreads];
  __shared__ int sbest;
  unsigned gen = 0;
  const KmChunks ch = km_chunking(N);
  const int L = km_trials(K);
  const int t = threadIdx.x;
  const int G = kKmThreads / E;  // row groups of the column sums (E <= 64, so G >= 2)
  const int ce = t % E, cg = t / E;

  // 1. column sums
  int bad = 0;
  for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
    const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
    double s = 0.0;
    if (cg < G)
      for (long long i = i0 + cg; i < i1; i += G) {
        const double v = x[(size_t)i * E + ce];
        bad |= !isfinite(v);
        s += v;
      }
    colpart[t] = s;
    __syncthreads();
    if (t < E) {
      double a = colpart[t];
      for (int g = 1; g < G; ++g) a += colpart[g * E + t];
      w.part_col[(size_t)c * E + t] = a;
    }
    __syncthreads();
  }
  if (bad) atomicOr(status, 1);
  grid_barrier(w.bar, gen);

  // 2. mean, centred copy, row norms, sums of squares
  if (t < E) {
    double a = 0.0;
    for (int c = 0; c < ch.nch; ++c) a += w.part_col[(size_t)c * E + t];
    smean[t] = a / (double)N;
  }
  __syncthreads();
  for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
    const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
    double s = 0.0;
    if (cg < G)
      for (long long i = i0 + cg; i < i1; i += G) {
        const double v = x[(size_t)i * E + ce] - smean[ce];
        w.xc[(size_t)i * E + ce] = v;
        s = fma(v, v, s);
      }
    colpart[t] = s;
    __syncthreads();
    if (t < E) {
      double a = colpart[t];
      for (int g = 1; g < G; ++g) a += colpart[g * E + t];
      w.part_var[(size_t)c * E + t] = a;
    }
    for (long long i = i0 + t; i < i1; i += kKmThreads) {
      const double* r = w.xc + (size_t)i * E;
      double n = 0.0;
      for (int e = 0; e < E; ++e) n = fma(r[e], r[e], n);
      w.xn[i] = n;
    }
    __syncthreads();
  }
  grid_barrier(w.bar, gen);

  // 3. tolerance and the initial centres
  if (blockIdx.x == 0) {
    if (t < E) w.mean[t] = smean[t];
    if (t == 0) {
      double v = 0.0;
      for (int e = 0; e < E; ++e) {
        double a = 0.0;
        for (int c = 0; c < ch.nch; ++c) a += w.part_var[(size_t)c * E + e];
        v += a / (double)N;
      }
      *w.tol = v / (double)E * 1e-4;
    }
  }
  if (init != nullptr) {
    if (blockIdx.x == 0)
      for (int j = t; j < K * E; j += kKmThreads) w.cinit[j] = init[j] - smean[j % E];
    return;
  }
  const double* a0 = w.xc + (size_t)first * E;
  if (blockIdx.x == 0)
    for (int e = t; e < E; e += kKmThreads) w.cinit[e] = a0[e];
  for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
    const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
    double s = 0.0;
    for (long long i = i0 + t; i < i1; i += kKmThreads) {
      const double d = km_sq_dist(a0, w.xn[first], w.xc + (size_t)i * E, w.xn[i], E);
      w.closest[i] = d;
      s += d;
    }
    s = km_block_sum(s, red);
    if (t == 0) w.part_pot[(size_t)c * L] = s;
  }
  int best = 0;
  for (int r = 1; r < K; ++r) {
    grid_barrier(w.bar, gen);
    // (a) current_pot, closest_dist_sq = the chosen candidate's distances, chunk scans
    double pot = 0.0;
    for (int c = 0; c < ch.nch; ++c) pot += w.part_pot[(size_t)c * L + best];
    const long long run = (ch.cs + kKmThreads - 1) / kKmThreads;
    for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
      const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
      const long long j0 = min(i1, i0 + t * run), j1 = min(i1, j0 + run);
      double s = 0.0;
      for (long long i = j0; i < j1; ++i) {
        const double d = r > 1 ? w.dtc[(size_t)best * N + i] : w.closest[i];
        w.closest[i] = d;
        s += d;
      }
      runpre[t] = s;
      __syncthreads();
      if (t == 0) {
        double p = 0.0;
        for (int q = 0; q < kKmThreads; ++q) { const double v = runpre[q]; runpre[q] = p; p += v; }
        w.part_tot[c] = p;
      }
      __syncthreads();
      double p = runpre[t];
      for (long long i = j0; i < j1; ++i) { p += w.closest[i]; w.cum[i] = p; }
      __syncthreads();
    }
    grid_barrier(w.bar, gen);
    // (b) searchsorted
    double target[kKmMaxTrials];
#pragma unroll
    for (int l = 0; l < kKmMaxTrials; ++l) target[l] = l < L ? uniforms[(size_t)(r - 1) * L + l] * pot : 0.0;
    __shared__ double chpre;
    for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
      if (t == 0) {
        double p = 0.0;
        for (int q = 0; q < c; ++q) p += w.part_tot[q];
        chpre = p;
      }
      __syncthreads();
      const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
#pragma unroll
      for (int l = 0; l < kKmMaxTrials; ++l) {
        if (l >= L) break;
        int n = 0;
        for (long long i = i0 + t; i < i1; i += kKmThreads) n += (chpre + w.cum[i]) < target[l];
        n = __reduce_add_sync(0xffffffffu, n);
        if ((t & 31) == 0) redi[(t >> 5) * kKmMaxTrials + l] = n;
      }
      __syncthreads();
      if (t < L) {
        long long n = 0;
        for (int q = 0; q < kKmThreads / 32; ++q) n += redi[q * kKmMaxTrials + t];
        w.part_cnt[(size_t)c * L + t] = n;
      }
      __syncthreads();
    }
    grid_barrier(w.bar, gen);
    // (c) candidate distances and potentials
    long long cand[kKmMaxTrials];
#pragma unroll
    for (int l = 0; l < kKmMaxTrials; ++l) {
      if (l >= L) break;
      long long n = 0;
      for (int c = 0; c < ch.nch; ++c) n += w.part_cnt[(size_t)c * L + l];
      cand[l] = min(n, N - 1);
    }
    for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
      const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
#pragma unroll
      for (int l = 0; l < kKmMaxTrials; ++l) {
        if (l >= L) break;
        const double* a = w.xc + (size_t)cand[l] * E;
        const double an = w.xn[cand[l]];
        double s = 0.0;
        for (long long i = i0 + t; i < i1; i += kKmThreads) {
          const double d = fmin(w.closest[i], km_sq_dist(a, an, w.xc + (size_t)i * E, w.xn[i], E));
          w.dtc[(size_t)l * N + i] = d;
          s += d;
        }
        s = km_block_sum(s, red);
        if (t == 0) w.part_pot[(size_t)c * L + l] = s;
      }
    }
    grid_barrier(w.bar, gen);
    if (t == 0) {
      double bp = 0.0;
      int b = 0;
      for (int l = 0; l < L; ++l) {
        double p = 0.0;
        for (int c = 0; c < ch.nch; ++c) p += w.part_pot[(size_t)c * L + l];
        if (l == 0 || p < bp) { bp = p; b = l; }
      }
      sbest = b;
    }
    __syncthreads();
    best = sbest;
    if (blockIdx.x == 0)
      for (int e = t; e < E; e += kKmThreads) {
        long long cb = cand[0];
#pragma unroll
        for (int l = 1; l < kKmMaxTrials; ++l)
          if (l == best) cb = cand[l];
        w.cinit[(size_t)r * E + e] = w.xc[(size_t)cb * E + e];
      }
  }
}

// Shared memory of kmeans_lloyd_kernel (dynamic): centres, old centres, their squared norms, weights, a staged tile.
__host__ __device__ inline size_t km_lloyd_smem(int E, int K) {
  return ((size_t)2 * K * E + 2 * K + (size_t)kKmTile * (E + 1)) * sizeof(double) + kKmTile * sizeof(int);
}

// _kmeans_single_lloyd (max_iter iterations of lloyd_iter_chunked_dense) from the centred initial centres cinit.
// Per iteration: (A) per chunk, the labels (first argmin of |c|^2 - 2 x.c, as _update_chunk_dense), the count of
// changed labels and the per-cluster sums and weights;  (B) the chunk partials summed in chunk order into w.sums,
// spread over the grid;  (C) in every CTA alike: _relocate_empty_clusters_dense (the farthest points from their old
// centres, largest first, ties to the lower index, one grid pass each), _average_centers, _center_shift and the
// convergence decision;  a third grid barrier ends the pass, so no CTA rewrites the change counts, the relocation
// partials or the labels (A) before every CTA has read them in (C).  Then the final E-step when the convergence was
// not strict, the inertia (_inertia_dense), the centres plus X_mean, n_iter and the count of distinct labels.
// (_relocate_empty_clusters_dense returns without moving a point when the largest distance is 0, as here.)
__global__ void __launch_bounds__(kKmThreads, 1) kmeans_lloyd_kernel(long long N, int E, int K, int max_iter, KmWork w,
                                                                   double* __restrict__ centres_out,
                                                                   int* __restrict__ labels, double* inertia,
                                                                   int* n_iter, int* status) {
  extern __shared__ double sm[];
  double* cen = sm;                  // K*E
  double* cold = cen + K * E;        // K*E
  double* cn = cold + K * E;         // K
  double* wk = cn + K;               // K
  double* xs = wk + K;               // kKmTile * (E + 1)
  int* lab = reinterpret_cast<int*>(xs + kKmTile * (E + 1));
  __shared__ double red[32];
  __shared__ long long redi[32];
  __shared__ long long far[kKmMaxK];
  __shared__ int empty[kKmMaxK];
  unsigned gen = 0;
  const KmChunks ch = km_chunking(N);
  const int t = threadIdx.x, KE = K * E, ES = E + 1;
  if (*status & 1) {  // non-finite input: nothing to fit
    if (blockIdx.x == 0 && t == 0) { *n_iter = 0; *inertia = NAN; }
    return;
  }
  for (int j = t; j < KE; j += kKmThreads) cen[j] = w.cinit[j];
  __syncthreads();
  auto centre_norms = [&]() {
    for (int k = t; k < K; k += kKmThreads) {
      double n = 0.0;
      for (int e = 0; e < E; ++e) n = fma(cen[k * E + e], cen[k * E + e], n);
      cn[k] = n;
    }
    __syncthreads();
  };
  auto stage = [&](long long i0, int np) {
    for (int j = t; j < np * E; j += kKmThreads) xs[(j / E) * ES + j % E] = w.xc[(size_t)i0 * E + j];
    __syncthreads();
  };
  auto nearest = [&](const double* xr) {
    int best = 0;
    double bd = 0.0;
    for (int k = 0; k < K; ++k) {
      double dot = 0.0;
      for (int e = 0; e < E; ++e) dot = fma(xr[e], cen[k * E + e], dot);
      const double d = fma(-2.0, dot, cn[k]);
      if (k == 0 || d < bd) { bd = d; best = k; }
    }
    return best;
  };
  bool strict = false;
  int it = 0;
  for (; it < max_iter; ++it) {
    centre_norms();
    // (A)
    for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
      const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
      double acc[kKmPairsPerThread];
#pragma unroll
      for (int q = 0; q < kKmPairsPerThread; ++q) acc[q] = 0.0;
      double cnt = 0.0;
      int changed = 0;
      for (long long b = i0; b < i1; b += kKmTile) {
        const int np = (int)min((long long)kKmTile, i1 - b);
        stage(b, np);
        if (t < np) {
          const int l = nearest(xs + t * ES);
          changed += labels[b + t] != l;
          labels[b + t] = l;
          lab[t] = l;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < kKmPairsPerThread; ++q) {
          const int j = t + q * kKmThreads;
          if (j < KE) {
            const int k = j / E, e = j % E;
            double s = acc[q];
            for (int p = 0; p < np; ++p)
              if (lab[p] == k) s += xs[p * ES + e];
            acc[q] = s;
          }
        }
        if (t < K)
          for (int p = 0; p < np; ++p) cnt += lab[p] == t;
        __syncthreads();
      }
      double* ps = w.part_sum + (size_t)c * (KE + K);
#pragma unroll
      for (int q = 0; q < kKmPairsPerThread; ++q) {
        const int j = t + q * kKmThreads;
        if (j < KE) ps[j] = acc[q];
      }
      if (t < K) ps[KE + t] = cnt;
      changed = __reduce_add_sync(0xffffffffu, changed);
      if ((t & 31) == 0) redi[t >> 5] = changed;
      __syncthreads();
      if (t == 0) w.part_idx[c] = redi[0] + redi[1] + redi[2] + redi[3];
      __syncthreads();
    }
    grid_barrier(w.bar, gen);
    // (B)
    for (long long j = (long long)blockIdx.x * kKmThreads + t; j < KE + K; j += (long long)gridDim.x * kKmThreads) {
      double s = 0.0;
      for (int c = 0; c < ch.nch; ++c) s += w.part_sum[(size_t)c * (KE + K) + j];
      w.sums[j] = s;
    }
    grid_barrier(w.bar, gen);
    // (C)
    for (int j = t; j < KE; j += kKmThreads) { cold[j] = cen[j]; cen[j] = w.sums[j]; }
    for (int k = t; k < K; k += kKmThreads) wk[k] = w.sums[KE + k];
    long long nchanged = 0;
    for (int c = 0; c < ch.nch; ++c) nchanged += w.part_idx[c];
    __syncthreads();
    int n_empty = 0;
    for (int k = 0; k < K; ++k)
      if (wk[k] == 0.0) empty[n_empty++] = k;
    __syncthreads();
    if (n_empty > 0) {
      // distances = ((X - centers_old[labels])**2).sum(axis=1); the n_empty farthest points, largest first
      bool skip = false;
      for (int r = 0; r < n_empty && !skip; ++r) {
        for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
          const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
          double bv = 0.0;
          long long bi = -1;
          for (long long i = i0 + t; i < i1; i += kKmThreads) {
            bool taken = false;
            for (int q = 0; q < r; ++q) taken |= far[q] == i;
            if (taken) continue;
            const double* xr = w.xc + (size_t)i * E;
            const double* cr = cold + labels[i] * E;
            double d = 0.0;
            for (int e = 0; e < E; ++e) { const double v = xr[e] - cr[e]; d = fma(v, v, d); }
            if (bi < 0 || d > bv) { bv = d; bi = i; }
          }
          km_block_argmax(bv, bi, red, redi);
          if (t == 0) { w.part_val[c] = bv; w.part_cnt[c] = bi; }
        }
        grid_barrier(w.bar, gen);
        double bv = 0.0;
        long long bi = -1;
        for (int c = 0; c < ch.nch; ++c) {
          const long long ci = w.part_cnt[c];
          if (ci >= 0 && (bi < 0 || w.part_val[c] > bv)) { bv = w.part_val[c]; bi = ci; }
        }
        if (r == 0 && bv == 0.0) skip = true;  // more clusters than distinct points: relocating is pointless
        if (t == 0) far[r] = bi;
        __syncthreads();
        grid_barrier(w.bar, gen);  // part_val / part_cnt are rewritten by the next pass
      }
      if (!skip && t == 0)
        for (int r = 0; r < n_empty; ++r) {
          const int nk = empty[r];
          const long long fi = far[r];
          const int ok = labels[fi];
          for (int e = 0; e < E; ++e) {
            const double v = w.xc[(size_t)fi * E + e];
            cen[ok * E + e] -= v;
            cen[nk * E + e] = v;
          }
          wk[nk] = 1.0;
          wk[ok] -= 1.0;
        }
      __syncthreads();
    }
    if (t == 0) {  // _average_centers, in place and in cluster order
      int am = 0;
      for (int k = 1; k < K; ++k)
        if (wk[k] > wk[am]) am = k;
      for (int k = 0; k < K; ++k) {
        if (wk[k] > 0.0) {
          const double alpha = 1.0 / wk[k];
          for (int e = 0; e < E; ++e) cen[k * E + e] *= alpha;
        } else {
          for (int e = 0; e < E; ++e) cen[k * E + e] = cen[am * E + e];
        }
      }
      double tot = 0.0;  // (center_shift**2).sum()
      for (int k = 0; k < K; ++k) {
        double s = 0.0;
        for (int e = 0; e < E; ++e) { const double v = cen[k * E + e] - cold[k * E + e]; s = fma(v, v, s); }
        const double sh = sqrt(s);
        tot += sh * sh;
      }
      red[0] = tot;
    }
    __syncthreads();
    const double shift = red[0];
    // every CTA has read this pass's part_idx, part_val / part_cnt and the relocated points' labels before any CTA
    // rewrites them in the next pass's (A) or in the final pass
    grid_barrier(w.bar, gen);
    if (nchanged == 0) { strict = true; break; }
    if (shift <= *w.tol) break;
  }
  const int done = it < max_iter ? it + 1 : max_iter;
  // final E-step (unless strict) and the inertia
  centre_norms();
  for (int c = blockIdx.x; c < ch.nch; c += gridDim.x) {
    const long long i0 = (long long)c * ch.cs, i1 = min(N, i0 + ch.cs);
    double s = 0.0;
    unsigned seen = 0;
    for (long long b = i0; b < i1; b += kKmTile) {
      const int np = (int)min((long long)kKmTile, i1 - b);
      stage(b, np);
      if (t < np) {
        const double* xr = xs + t * ES;
        int l = labels[b + t];
        if (!strict) { l = nearest(xr); labels[b + t] = l; }
        double d = 0.0;
        for (int e = 0; e < E; ++e) { const double v = xr[e] - cen[l * E + e]; d = fma(v, v, d); }
        s += d;
        seen |= 1u << l;
      }
      __syncthreads();
    }
    s = km_block_sum(s, red);
    seen = __reduce_or_sync(0xffffffffu, seen);
    if ((t & 31) == 0) redi[t >> 5] = seen;
    __syncthreads();
    if (t == 0) {
      w.part_val[c] = s;
      w.part_cnt[c] = redi[0] | redi[1] | redi[2] | redi[3];
    }
    __syncthreads();
  }
  grid_barrier(w.bar, gen);
  if (blockIdx.x == 0) {
    for (int j = t; j < KE; j += kKmThreads) centres_out[j] = cen[j] + w.mean[j % E];
    if (t == 0) {
      double s = 0.0;
      long long seen = 0;
      for (int c = 0; c < ch.nch; ++c) { s += w.part_val[c]; seen |= w.part_cnt[c]; }
      *inertia = s;
      *n_iter = done;
      const int distinct = __popcll(seen);
      if (distinct < K) atomicOr(status, 2 | (distinct << 8));
    }
  }
}

// KMeans.predict: the first argmin of |c|^2 - 2 x.c on the raw x and the stored centres; optionally the one-hot
// (K, N) of labels_to_one_hot(labels, K, axis=-2).
__global__ void __launch_bounds__(kKmThreads) kmeans_predict_kernel(const double* __restrict__ x, long long N, int E,
                                                                     int K, const double* __restrict__ centres,
                                                                     int* __restrict__ labels,
                                                                     double* __restrict__ one_hot) {
  __shared__ double cen[kKmMaxK * kKmMaxE];
  __shared__ double cn[kKmMaxK];
  const int t = threadIdx.x;
  for (int j = t; j < K * E; j += kKmThreads) cen[j] = centres[j];
  __syncthreads();
  for (int k = t; k < K; k += kKmThreads) {
    double n = 0.0;
    for (int e = 0; e < E; ++e) n = fma(cen[k * E + e], cen[k * E + e], n);
    cn[k] = n;
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * kKmThreads + t;
  if (i >= N) return;
  const double* xr = x + (size_t)i * E;
  int best = 0;
  double bd = 0.0;
  for (int k = 0; k < K; ++k) {
    double dot = 0.0;
    for (int e = 0; e < E; ++e) dot = fma(xr[e], cen[k * E + e], dot);
    const double d = fma(-2.0, dot, cn[k]);
    if (k == 0 || d < bd) { bd = d; best = k; }
  }
  if (labels) labels[i] = best;
  if (one_hot)
    for (int k = 0; k < K; ++k) one_hot[(size_t)k * N + i] = k == best ? 1.0 : 0.0;
}

}  // namespace pbb
