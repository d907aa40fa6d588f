// Frequency permutation alignment on the device (pb_bss/permutation_alignment.py):
// DHTVPermutationAlignment.calculate_mapping (:295-355) with every similarity metric (:380-420) and
// assignment (:458-590), the score matrices and assignments of Greedy / OraclePermutationAlignment
// (:592-786), and apply_mapping (:54-104).  A DHTV plan runs in one launch: dhtv_cluster_kernel when
// its widest segment fits one thread-block cluster, else dhtv_coop_kernel.  See include/pbb.h.
#include <cooperative_groups.h>
#include <cstdlib>

#include "common.cuh"
#include "prof.cuh"

namespace pbb {

constexpr int kDhtvMaxK = 9;       // the reference asserts K < 10 (permutation_alignment.py:200)

__device__ inline double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  return s;
}

// features = mask / max(||mask||_T, tiny) per (k, f)   (:309-310, _parameterized_vector_norm :358-377)
__global__ void dhtv_normalize_kernel(const double* __restrict__ mask, double* __restrict__ feat, int KF, int T) {
  const int row = blockIdx.x;
  if (row >= KF) return;
  __shared__ double red[32];
  const double* __restrict__ m = mask + (size_t)row * T;
  double s = 0.0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) s += m[t] * m[t];
  const double n = sqrt(block_sum(s, red));
  const double d = fmax(n, kTiny);
  for (int t = threadIdx.x; t < T; t += blockDim.x) feat[(size_t)row * T + t] = m[t] / d;
}

constexpr int kDhtvSlices = 8;   // bin slices of dhtv_coop_kernel's centroid sum (summed in fixed order)

__global__ void dhtv_init_mapping_kernel(long long* __restrict__ mapping, int K, int F) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < K * F) mapping[i] = i / F;
}

// Reverse permutation of one bin from its score matrix (_mapping_from_score_matrix, :458-590), by one thread; score
// is overwritten.  greedy: K times the first maximum of the row-major flattened matrix, then blank its row and
// column; optimal: the first best of itertools.permutations(range(K)) (lexicographic order, strict >), scores summed
// left to right like Python's sum().
__device__ __forceinline__ void dhtv_assign(double* __restrict__ score, int K, int optimal, int* __restrict__ perm) {
  if (!optimal) {
    for (int r = 0; r < K; ++r) {
      int bi = 0, bj = 0;
      double best = -INFINITY;
      bool found = false;
      for (int i = 0; i < K; ++i)
        for (int j = 0; j < K; ++j) {
          const double v = score[i * K + j];
          if (!found || v > best) { best = v; bi = i; bj = j; found = true; }
        }
      for (int j = 0; j < K; ++j) score[bi * K + j] = -INFINITY;
      for (int i = 0; i < K; ++i) score[i * K + bj] = -INFINITY;
      perm[bi] = bj;
    }
    return;
  }
  int cand[kDhtvMaxK];
  for (int k = 0; k < K; ++k) { cand[k] = k; perm[k] = k; }
  double best = -INFINITY;
  while (true) {
    double sum = 0.0;
    for (int k = 0; k < K; ++k) sum += score[k * K + cand[k]];
    if (sum > best) {
      best = sum;
      for (int k = 0; k < K; ++k) perm[k] = cand[k];
    }
    int i = K - 2;  // next lexicographic permutation
    while (i >= 0 && cand[i] > cand[i + 1]) --i;
    if (i < 0) break;
    int j = K - 1;
    while (cand[j] < cand[i]) --j;
    { const int t = cand[i]; cand[i] = cand[j]; cand[j] = t; }
    for (int a = i + 1, b = K - 1; a < b; ++a, --b) { const int t = cand[a]; cand[a] = cand[b]; cand[b] = t; }
  }
}

#ifdef PBB_PHASE_TIMING
__device__ unsigned long long g_dhtv_phase[8];
__device__ unsigned long long g_dhtv_iters;
#define DH_PH(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) { long long _t = clock64(); g_dhtv_phase[i] += (unsigned long long)(_t - _tp); _tp = _t; } } while (0)
#else
#define DH_PH(i) do { } while (0)
#endif

// block_sum over the FIRST 128 threads only, in a fixed order: dhtv_coop_kernel's block size varies with K, its
// centroid norms -- and with them every score and the integer mapping -- do not
__device__ inline double block_sum_first128(double v, double* red) {
  v = warp_sum(threadIdx.x < 128 ? v : 0.0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0 && warp < 4) red[warp] = v;
  __syncthreads();
  return ((red[0] + red[1]) + red[2]) + red[3];
}

constexpr int kDhtvCoopMaxWarps = 16;

// The whole alignment plan in ONE cooperative launch, for segments too wide for dhtv_cluster_kernel.  Each iteration
// has two phases separated by grid-wide barriers: (A) centroid partial sums over kDhtvSlices bin slices, (B) per bin
// the scores, the assignment and the permutation.  The reference's early exit (:352-353) skips the remaining
// iterations of a segment.  plan: DEVICE copy of (iterations, start, end) triples.
// One CTA per bin of the segment, one WARP per (reference class, mask class) score: a single warp per bin spends
// ~25k cycles per iteration on its K^2 dot products and the assignment (latency of one dependent instruction stream);
// spread over K^2 warps the bin takes ~2k.
__global__ void __launch_bounds__(32 * kDhtvCoopMaxWarps) dhtv_coop_kernel(
    double* __restrict__ feat, double* __restrict__ partial, int* __restrict__ changed, const int* __restrict__ plan,
    int nplan, int K, int F, int T, long long* __restrict__ mapping, unsigned* __restrict__ bar, int metric,
    int optimal) {
  // metric: 1 = cos (features and centroid L2-normalised over time, score = inner product), 0 = multiply (inner
  // product of the raw masks), 2 = euclidean (score = -distance), permutation_alignment.py:309-340,380-420
  unsigned generation = 0;
#ifdef PBB_PHASE_TIMING
  long long _tp = clock64();
#endif
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* cent = reinterpret_cast<double*>(smem_raw);  // [K][T]
  __shared__ double red[4];
  __shared__ double cnorm[kDhtvMaxK];
  __shared__ double score_s[kDhtvMaxK * kDhtvMaxK];
  __shared__ int perm_s[kDhtvMaxK];
  __shared__ int ident_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int gthreads = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + tid;
  int idx = 0;
  for (int p = 0; p < nplan; ++p) {
    const int iters = plan[3 * p], start = plan[3 * p + 1], end = plan[3 * p + 2];
    const int n = end - start, per = (n + kDhtvSlices - 1) / kDhtvSlices;
    for (int it = 0; it < iters; ++it, ++idx) {
      // ---- phase A: partial[slice][k][t] = sum over the slice's bins ----
      for (int e = gtid; e < kDhtvSlices * K * T; e += gthreads) {
        const int sl = e / (K * T), i = e - sl * (K * T);
        const int k = i / T, t = i - k * T;
        const int f0 = start + sl * per, f1 = min(end, f0 + per);
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int f = f0;
        for (; f + 3 < f1; f += 4) {
          s0 += feat[((size_t)k * F + f) * T + t];
          s1 += feat[((size_t)k * F + f + 1) * T + t];
          s2 += feat[((size_t)k * F + f + 2) * T + t];
          s3 += feat[((size_t)k * F + f + 3) * T + t];
        }
        for (; f < f1; ++f) s0 += feat[((size_t)k * F + f) * T + t];
        partial[(size_t)sl * K * T + i] = (s0 + s1) + (s2 + s3);
      }
      DH_PH(0);  // phase A
      grid_barrier(bar, generation);
      DH_PH(1);  // barrier 1
      // ---- phase B: one CTA per bin; CTAs without a bin skip the centroid ----
      if ((int)blockIdx.x < n) {
        const double inv_n = 1.0 / (double)n;
#pragma unroll 2
        for (int i = tid; i < K * T; i += blockDim.x) {
          double v[kDhtvSlices];
#pragma unroll
          for (int sl = 0; sl < kDhtvSlices; ++sl) v[sl] = __ldcg(partial + (size_t)sl * K * T + i);
          double s = 0.0;
#pragma unroll
          for (int sl = 0; sl < kDhtvSlices; ++sl) s += v[sl];
          cent[i] = s * inv_n;
        }
        __syncthreads();
        DH_PH(2);  // centroid combine
        if (metric == 1) {
          for (int k = 0; k < K; ++k) {
            double s = 0.0;
            if (tid < 128)
              for (int t = tid; t < T; t += 128) { const double c = cent[k * T + t]; s += c * c; }
            const double nn = sqrt(block_sum_first128(s, red));
            if (tid == 0) cnorm[k] = fmax(nn, kTiny);
          }
          __syncthreads();
          for (int i = tid; i < K * T; i += blockDim.x) cent[i] = cent[i] / cnorm[i / T];
          __syncthreads();
        }
        DH_PH(3);  // centroid norms
        for (int f = start + blockIdx.x; f < end; f += gridDim.x) {
          // score[kr][km] = <centroid kr, feature km of this bin> by warp (kr, km): 16 values per lane at a time with
          // every load in flight; the sum runs over t in ascending order per lane, then the usual warp reduction
          for (int pair = warp; pair < K * K; pair += nwarps) {
            const int kr = pair / K, km = pair - kr * K;
            const double* __restrict__ row = feat + ((size_t)km * F + f) * T;
            double sacc = 0.0;
            for (int c0 = 0; c0 < T; c0 += 512) {
              double v[16];
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int t = c0 + lane + 32 * j;
                v[j] = t < T ? __ldcg(row + t) : 0.0;
              }
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int t = c0 + lane + 32 * j;
                if (t < T) {
                  if (metric == 2) { const double dlt = v[j] - cent[kr * T + t]; sacc += dlt * dlt; }
                  else sacc += v[j] * cent[kr * T + t];
                }
              }
            }
            sacc = warp_sum(sacc);
            if (metric == 2) sacc = -sqrt(sacc);  // the minus turns the distance into a similarity (:412-418)
            if (lane == 0) score_s[pair] = sacc;
          }
          __syncthreads();
          DH_PH(4);  // scores
          if (tid == 0) {
            double sc[kDhtvMaxK * kDhtvMaxK];
            int perm[kDhtvMaxK];
            for (int i = 0; i < K * K; ++i) sc[i] = score_s[i];
            dhtv_assign(sc, K, optimal, perm);
            bool ident = true;
            for (int k = 0; k < K; ++k) { perm_s[k] = perm[k]; ident = ident && perm[k] == k; }
            ident_s = ident ? 1 : 0;
            if (!ident) {
              long long mv[kDhtvMaxK];
              for (int k = 0; k < K; ++k) mv[k] = mapping[(size_t)k * F + f];
              for (int k = 0; k < K; ++k) mapping[(size_t)k * F + f] = mv[perm[k]];
              changed[idx] = 1;
            }
          }
          __syncthreads();
          DH_PH(5);  // assignment
          if (!ident_s) {
            for (int t = tid; t < T; t += blockDim.x) {
              double v[kDhtvMaxK];
              for (int k = 0; k < K; ++k) v[k] = feat[((size_t)k * F + f) * T + t];
              for (int k = 0; k < K; ++k) feat[((size_t)k * F + f) * T + t] = v[perm_s[k]];
            }
          }
          __syncthreads();
        }
      }
      DH_PH(6);  // permutation / rest of phase B
      grid_barrier(bar, generation);
      DH_PH(7);  // barrier 2
      if (__ldcg(changed + idx) == 0) {  // nothing moved: the segment has converged (:352-353)
        idx += iters - it;
        break;
      }
    }
  }
}

// ---- the whole plan in ONE thread-block cluster, features in (distributed) shared memory ----------------------
// A segment of the reference's plan is ~100 bins wide (stft_size 1024: 20 segments of 100-120 bins, 58 iterations),
// i.e. K T doubles x 120 = 1.4 MB: it fits into the shared memory of a 16-CTA cluster.  CTA r owns a contiguous run
// of the segment's bins, keeps their feature rows in its shared memory for all iterations of the segment and writes
// the permuted rows back once.  Per iteration: local partial sums -> cluster barrier -> reduce-scatter of the
// centroid over DSMEM (CTA r adds slice r of the C partial sums in rank order and stores it into every CTA's copy)
// -> cluster barrier -> norms, K^2 scores per owned bin (one warp per (bin, mask class), operands in shared memory),
// warp-parallel greedy assignment, in-place permutation, "changed" flags exchanged over DSMEM, the partial sums of the
// next iteration (only where a row moved) -> cluster barrier.  Two cluster barriers per iteration instead of two grid
// barriers, no L2 round trip and no thread-local array inside an iteration (a cluster barrier invalidates the L1).
// Same score arithmetic as dhtv_coop_kernel up to <x, c/|c|> = <x, c>/|c|; the bins are added into the centroid by
// owner.  Mappings are identical wherever no decision lies within rounding of a tie, and on exact ties
// (tests/test_permutation_gpu.py::test_dhtv_every_kernel_matches_the_oracle).
constexpr int kDhtvClThreads = 512;
constexpr int kDhtvClMaxLocal = 16;  // bins one CTA may own (static score / permutation tables)
static_assert(kDhtvClMaxLocal <= kDhtvClThreads / 32, "one warp per owned bin in the assignment");

__device__ __forceinline__ void dhtv_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t dhtv_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t dhtv_map_cta(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void dhtv_st_remote_u32(uint32_t addr, int v) {
  asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// KC = number of classes at compile time (2, 3, 4: clean unrolled code), 0 = any K <= 9 at run time
template <int KC>
__global__ void __launch_bounds__(kDhtvClThreads, 1) dhtv_cluster_kernel(
    double* __restrict__ feat, const int* __restrict__ plan, int nplan, int Krt, int F, int T,
    long long* __restrict__ mapping, int metric, int optimal) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int K = KC > 0 ? KC : Krt;
  constexpr int KU = KC > 0 ? KC : kDhtvMaxK;  // unroll bound of the per-class loops
  const int KT = K * T;
  double* cent = reinterpret_cast<double*>(smem_raw);  // [K][T] centroid (mean, not normalised), complete in every CTA
  double* part = cent + KT;                            // [K][T] sum over this CTA's bins
  double* rows = part + KT;                            // [local bin][K][T]
  __shared__ double cnorm[kDhtvMaxK];
  __shared__ double score_s[kDhtvClMaxLocal][kDhtvMaxK * kDhtvMaxK];
  __shared__ long long map_s[kDhtvClMaxLocal][kDhtvMaxK];  // the owned bins' columns of the mapping
  __shared__ int perm_s[kDhtvClMaxLocal][kDhtvMaxK];
  __shared__ int ident_s[kDhtvClMaxLocal];
  __shared__ int dirty_s[kDhtvClMaxLocal];
  __shared__ int flags_s[16];
  uint32_t C, r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(C));
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const uint32_t flags_a = dhtv_smem_addr(flags_s);
  // generic pointers into every CTA's partial sum / centroid (ordinary loads and stores: the compiler keeps all the
  // remote loads of one element in flight)
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const double* rpart[16];
  double* rcent[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    rpart[c] = cluster.map_shared_rank(part, c < (int)C ? c : 0);
    rcent[c] = cluster.map_shared_rank(cent, c < (int)C ? c : 0);
  }
#ifdef PBB_PHASE_TIMING
  long long _tp = clock64();
#endif
  const int sl = (KT + (int)C - 1) / (int)C;  // centroid slice reduced by one CTA
  for (int p = 0; p < nplan; ++p) {
    const int iters = plan[3 * p], start = plan[3 * p + 1], end = plan[3 * p + 2];
    const int n = end - start, per = (n + (int)C - 1) / (int)C;
    const int f0 = start + (int)r * per, f1 = min(end, f0 + per);
    const int nloc = max(0, f1 - f0);
    // own rows -> shared memory: warp w takes rows (j, k) = w, w + nwarps, ..., four loads per lane in flight
    for (int jk = warp; jk < nloc * K; jk += nwarps) {
      const int j = jk / K, k = jk - j * K;
      const double* __restrict__ src = feat + ((size_t)k * F + f0 + j) * T;
      double* __restrict__ dst = rows + j * KT + k * T;
      for (int c0 = 0; c0 < T; c0 += 512) {  // 16 loads per lane in flight: one L2 round trip per 512 frames of a row
        double v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int t = c0 + lane + 32 * q;
          v[q] = t < T ? __ldcg(src + t) : 0.0;
        }
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int t = c0 + lane + 32 * q;
          if (t < T) dst[t] = v[q];
        }
      }
    }
    if (tid < nloc * K) map_s[tid / K][tid % K] = __ldcg(mapping + (size_t)(tid % K) * F + f0 + tid / K);
    if (tid < kDhtvClMaxLocal) dirty_s[tid] = 0;
    __syncthreads();
    DH_PH(0);  // segment load
    const double inv_n = 1.0 / (double)n;
    auto partial_sums = [&]() {
      for (int i = tid; i < KT; i += blockDim.x) {
        double s = 0.0;  // owned bins in ascending order; four loads in flight
        int j = 0;
        for (; j + 4 <= nloc; j += 4) {
          const double a0 = rows[j * KT + i], a1 = rows[(j + 1) * KT + i], a2 = rows[(j + 2) * KT + i],
                       a3 = rows[(j + 3) * KT + i];
          s += a0; s += a1; s += a2; s += a3;
        }
        for (; j < nloc; ++j) s += rows[j * KT + i];
        part[i] = s;
      }
    };
    if (iters > 0) partial_sums();
    DH_PH(1);  // local partial sums
    dhtv_cluster_sync();  // every CTA's partial sum is complete
    for (int it = 0; it < iters; ++it) {
      for (int i = (int)r * sl + tid; i < min(KT, ((int)r + 1) * sl); i += blockDim.x) {
        double v[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) v[c] = c < (int)C ? rpart[c][i] : 0.0;
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < 16; ++c) s += v[c];  // rank order (the zeros beyond C change nothing)
        s *= inv_n;
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (c < (int)C) rcent[c][i] = s;
      }
      DH_PH(2);  // reduce-scatter + broadcast
      dhtv_cluster_sync();  // the centroid is complete in every CTA
      DH_PH(3);  // cluster barrier 2
      // cos: ||centroid_k|| by the LAST warps (they have the fewest score items), applied to the scores afterwards --
      // <x, c / ||c||> = <x, c> / ||c||, one division per score instead of a pass over the centroid
      if (metric == 1 && warp >= nwarps - K) {
        const int k = warp - (nwarps - K);
        double s = 0.0;
#pragma unroll 4
        for (int t = lane; t < T; t += 32) { const double c = cent[k * T + t]; s += c * c; }
        s = warp_sum(s);
        if (lane == 0) cnorm[k] = fmax(sqrt(s), kTiny);
      }
      // scores of every owned bin.  Per (kr, km): sum over t in ascending order per lane, then the warp reduction --
      // the order of the other DHTV kernels.  The pass is bound by shared-memory bandwidth, so for K <= 4 one warp
      // takes a whole bin (K feature rows and K centroid rows read once, K^2 accumulators); the generic kernel takes
      // one (bin, mask class) row per warp with K accumulators.
      if constexpr (KC > 0) {
        for (int j = warp; j < nloc; j += nwarps) {
          const double* __restrict__ rowj = rows + j * KT;
          double sacc[KC][KC];
#pragma unroll
          for (int kr = 0; kr < KC; ++kr)
#pragma unroll
            for (int km = 0; km < KC; ++km) sacc[kr][km] = 0.0;
#pragma unroll 2
          for (int t = lane; t < T; t += 32) {
            double x[KC], c[KC];
#pragma unroll
            for (int k = 0; k < KC; ++k) { x[k] = rowj[k * T + t]; c[k] = cent[k * T + t]; }
#pragma unroll
            for (int kr = 0; kr < KC; ++kr)
#pragma unroll
              for (int km = 0; km < KC; ++km) {
                if (metric == 2) { const double dlt = x[km] - c[kr]; sacc[kr][km] += dlt * dlt; }
                else sacc[kr][km] += x[km] * c[kr];
              }
          }
#pragma unroll
          for (int kr = 0; kr < KC; ++kr)
#pragma unroll
            for (int km = 0; km < KC; ++km) {
              double v = warp_sum(sacc[kr][km]);
              if (metric == 2) v = -sqrt(v);
              if (lane == 0) score_s[j][kr * KC + km] = v;
            }
        }
      } else {
      for (int item = warp; item < nloc * K; item += nwarps) {
        const int j = item / K, km = item - j * K;
        const double* __restrict__ row = rows + j * KT + km * T;
        double sacc[KU];
#pragma unroll
        for (int kr = 0; kr < KU; ++kr) sacc[kr] = 0.0;
        if (metric == 2) {
#pragma unroll 4
          for (int t = lane; t < T; t += 32) {
            const double x = row[t];
#pragma unroll
            for (int kr = 0; kr < KU; ++kr)
              if (kr < K) { const double dlt = x - cent[kr * T + t]; sacc[kr] += dlt * dlt; }
          }
        } else {
#pragma unroll 4
          for (int t = lane; t < T; t += 32) {
            const double x = row[t];
#pragma unroll
            for (int kr = 0; kr < KU; ++kr)
              if (kr < K) sacc[kr] += x * cent[kr * T + t];
          }
        }
#pragma unroll
        for (int kr = 0; kr < KU; ++kr) {
          if (kr < K) {
            double v = warp_sum(sacc[kr]);
            if (metric == 2) v = -sqrt(v);
            if (lane == 0) score_s[j][kr * K + km] = v;
          }
        }
      }
      }
      __syncthreads();
      DH_PH(4);  // norms + scores
      int moved = 0;
      if (warp < nloc) {
        // one warp per owned bin (everything in shared memory / registers: the cluster barrier invalidates the L1, a
        // thread-local array would cost an L2 round trip per line and iteration)
        const int j = warp;
        double* sc = score_s[j];
        int* perm = perm_s[j];
        if (metric == 1)
          for (int i = lane; i < K * K; i += 32) sc[i] = sc[i] / cnorm[i / K];
        __syncwarp();
        if (optimal) {
          if (lane == 0) dhtv_assign(sc, K, 1, perm);
        } else {
          // greedy (:525-553): K times the largest remaining score, first one in row-major order on ties; the lanes
          // hold entries lane, lane + 32, lane + 64 (K^2 <= 81)
          double e[3];
          bool alive[3];
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            const int i = lane + 32 * q;
            alive[q] = i < K * K;
            e[q] = alive[q] ? sc[i] : 0.0;
          }
          for (int round = 0; round < K; ++round) {
            double bv = 0.0;
            int bi = 1 << 30;  // no candidate
#pragma unroll
            for (int q = 0; q < 3; ++q)
              if (alive[q] && (bi == (1 << 30) || e[q] > bv)) { bv = e[q]; bi = lane + 32 * q; }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
              const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
              const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
              // the candidate with the smaller index wins unless the other one is strictly larger (scan order of the
              // reference: a later entry replaces the best only if it is greater)
              const bool take = oi != (1 << 30) && (bi == (1 << 30) || (oi < bi ? !(bv > ov) : ov > bv));
              if (take) { bv = ov; bi = oi; }
            }
            const int row = bi / K, col = bi - row * K;
            if (lane == 0) perm[row] = col;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
              const int i = lane + 32 * q;
              if (i / K == row || i % K == col) alive[q] = false;
            }
          }
        }
        __syncwarp();
        bool ident = true;
        for (int k = 0; k < K; ++k) ident = ident && perm[k] == k;
        if (lane == 0) ident_s[j] = ident ? 1 : 0;
        if (!ident) {
          const long long m = lane < K ? map_s[j][perm[lane]] : 0;
          __syncwarp();
          if (lane < K) map_s[j][lane] = m;
          if (lane == 0) dirty_s[j] = 1;
          moved = 1;
        }
      }
      moved = __syncthreads_or(moved);
      DH_PH(5);  // assignment
      for (int j = 0; j < nloc; ++j) {
        if (ident_s[j]) continue;
        for (int t = tid; t < T; t += blockDim.x) {
          double v[KU];
#pragma unroll
          for (int k = 0; k < KU; ++k) v[k] = (KC > 0 || k < K) ? rows[j * KT + k * T + t] : 0.0;
#pragma unroll
          for (int k = 0; k < KU; ++k) {
            if (KC > 0 || k < K) {
              const int src = perm_s[j][k];
              double x = v[0];
#pragma unroll
              for (int q = 1; q < KU; ++q) x = src == q ? v[q] : x;  // register select instead of a local array
              rows[j * KT + k * T + t] = x;
            }
          }
        }
      }
      if (tid < (int)C) dhtv_st_remote_u32(dhtv_map_cta(flags_a + 4u * r, (uint32_t)tid), moved);
      DH_PH(6);  // permutation
      // the next iteration's partial sum goes in front of the same barrier (only if a row of this CTA moved: it is
      // a sum over the owned rows, nothing else); everybody is past the reduce-scatter that read the old one
      if (moved && it + 1 < iters) {
        __syncthreads();
        partial_sums();
      }
      DH_PH(1);
      dhtv_cluster_sync();  // flags and partial sums of every CTA have arrived; rows / tables are final
      DH_PH(7);  // cluster barrier
#ifdef PBB_PHASE_TIMING
      if (blockIdx.x == 0 && tid == 0) g_dhtv_iters += 1;
#endif
      int any = 0;
      for (uint32_t c = 0; c < C; ++c) any |= flags_s[c];
      if (!any) break;  // nothing moved anywhere: the segment has converged (:352-353); uniform over the cluster
    }
    // the segment's permuted rows and mapping columns go back to global memory for the owners of the next segment
    for (int jk = warp; jk < nloc * K; jk += nwarps) {
      const int j = jk / K, k = jk - j * K;
      if (!dirty_s[j]) continue;
      double* __restrict__ dst = feat + ((size_t)k * F + f0 + j) * T;
      const double* __restrict__ src = rows + j * KT + k * T;
      for (int t = lane; t < T; t += 32) __stcg(dst + t, src[t]);
    }
    if (tid < nloc * K && dirty_s[tid / K]) mapping[(size_t)(tid % K) * F + f0 + tid / K] = map_s[tid / K][tid % K];
    __threadfence();
    dhtv_cluster_sync();
  }
}

__global__ void apply_mapping_kernel(const double* __restrict__ mask, const long long* __restrict__ mapping, int K,
                                     int F, int T, double* __restrict__ out) {
  const int kf = blockIdx.x;  // k * F + f
  const int f = kf % F;
  const long long src = mapping[kf];
  const double* __restrict__ s = mask + ((size_t)src * F + f) * T;
  double* __restrict__ o = out + (size_t)kf * T;
  for (int t = threadIdx.x; t < T; t += blockDim.x) o[t] = s[t];
}

// ---- score matrices and assignments for Greedy / Oracle alignment ------------------
// _ScoreMatrix.multiply / cos / euclidean (:380-420): scores[f][k_ref][k_mask].  One warp
// per bin; the bin-th vector of source k starts at base + k * source_stride + f * T, which
// lets GreedyPermutationAlignment pass the two shifted views mask[:, 1:] / mask[:, :-1]
// (:702) of one array.
__global__ void __launch_bounds__(128) score_matrix_kernel(const double* __restrict__ mask,
                                                           const double* __restrict__ ref, long long mask_ss,
                                                           long long ref_ss, int K, int F, int T, int metric,
                                                           double* __restrict__ scores) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (f >= F) return;
  double nm[kDhtvMaxK], nr[kDhtvMaxK];
  for (int k = 0; k < K; ++k) { nm[k] = 1.0; nr[k] = 1.0; }
  if (metric == 1) {  // cos: both sides L2-normalised over time (:358-377)
    for (int k = 0; k < K; ++k) {
      const double* __restrict__ a = mask + k * mask_ss + (size_t)f * T;
      const double* __restrict__ b = ref + k * ref_ss + (size_t)f * T;
      double sa = 0.0, sb = 0.0;
      for (int t = lane; t < T; t += 32) { sa += a[t] * a[t]; sb += b[t] * b[t]; }
      nm[k] = fmax(sqrt(warp_sum(sa)), kTiny);
      nr[k] = fmax(sqrt(warp_sum(sb)), kTiny);
    }
  }
  for (int kr = 0; kr < K; ++kr)
    for (int km = 0; km < K; ++km) {
      const double* __restrict__ a = mask + km * mask_ss + (size_t)f * T;
      const double* __restrict__ b = ref + kr * ref_ss + (size_t)f * T;
      double s = 0.0;
      if (metric == 2) {
        for (int t = lane; t < T; t += 32) { const double d = a[t] - b[t]; s += d * d; }
        s = -sqrt(warp_sum(s));  // the minus turns the distance into a similarity (:412-418)
      } else {
        for (int t = lane; t < T; t += 32) s += (a[t] / nm[km]) * (b[t] / nr[kr]);
        s = warp_sum(s);
      }
      if (lane == 0) scores[((size_t)f * K + kr) * K + km] = s;
    }
}

// _mapping_from_score_matrix (:458-590), one thread per bin: dhtv_assign on finite scores.
__global__ void mapping_from_score_kernel(const double* __restrict__ scores, int F, int K, int optimal,
                                          long long* __restrict__ mapping, int* __restrict__ status) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double sc[kDhtvMaxK * kDhtvMaxK];
  bool finite = true;
  for (int i = 0; i < K * K; ++i) {
    sc[i] = scores[(size_t)f * K * K + i];
    finite = finite && isfinite(sc[i]);
  }
  if (!finite) {  // ValueError('score matrix is infeasible') (:511-513)
    atomicCAS(status, 0, f + 1);
    for (int k = 0; k < K; ++k) mapping[(size_t)k * F + f] = k;
    return;
  }
  int out[kDhtvMaxK];
  dhtv_assign(sc, K, optimal, out);
  for (int k = 0; k < K; ++k) mapping[(size_t)k * F + f] = out[k];
}

// GreedyPermutationAlignment.calculate_mapping (:700-712): bin 0 is the identity, bins
// 1..F-1 hold the pairwise mappings to their lower neighbour; chain them bottom up,
// mapping[:, f] = mapping[mapping[:, f-1], f].  Sequential in f by definition; K lanes.
__global__ void chain_mapping_kernel(const long long* __restrict__ pair, int K, int F, long long* __restrict__ mapping) {
  const int k = threadIdx.x;
  __shared__ long long prev[kDhtvMaxK];
  if (k < K) { prev[k] = k; mapping[(size_t)k * F] = k; }
  __syncthreads();
  for (int f = 1; f < F; ++f) {
    long long v = 0;
    if (k < K) v = pair[(size_t)prev[k] * (F - 1) + (f - 1)];
    __syncthreads();
    if (k < K) { prev[k] = v; mapping[(size_t)k * F + f] = v; }
    __syncthreads();
  }
}

// ---- host side of pbb_dhtv_mapping_ex ----------------------------------------------------------------------------

// One checked alignment and its `centroid` scratch: kDhtvSlices * K * T doubles of partial sums, then the int
// "changed" flags (one per iteration and a spare), the grid-barrier counter and the device copy of the plan.
struct DhtvCall {
  double* features;
  long long* mapping;
  int nplan, K, F, T, metric, algorithm;
  int total_iters, widest;
  double* partial;
  int* changed;
  unsigned* bar;
  int* plan_dev;
};

// Checks the arguments and the HOST plan, and fills c but its scratch pointers: total_iters = planned iterations of
// all segments, widest = bins of the widest segment (at least 1).
static int check_dhtv_args(const double* mask, int K, int F, int T, const int* plan, int nplan, double* features,
                           const double* centroid, long long* mapping, int metric, int algorithm, DhtvCall* c) {
  PBB_CHECK_ARG(mask != nullptr, 1, "mask is null");
  PBB_CHECK_ARG(metric >= 0 && metric <= 2, 10, "metric: 0 multiply, 1 cos, 2 euclidean");
  PBB_CHECK_ARG(algorithm == 0 || algorithm == 1, 11, "algorithm: 0 greedy, 1 optimal");
  PBB_CHECK_ARG(K > 0 && K <= kDhtvMaxK, 2, "need 0 < K < 10 (permutation_alignment.py:200)");
  PBB_CHECK_ARG(F > 0, 3, "F must be positive");
  PBB_CHECK_ARG(T > 0, 4, "T must be positive");
  PBB_CHECK_ARG(plan != nullptr && nplan > 0 && nplan <= 4096, 5, "alignment plan: HOST array of (iterations, start, end)");
  PBB_CHECK_ARG(features && centroid, 7, "scratch is null (pbb_dhtv_scratch_doubles)");
  PBB_CHECK_ARG(mapping != nullptr, 9, "mapping is null");
  PBB_CHECK_ARG((size_t)K * T * sizeof(double) <= 200 * 1024, 4, "K * T too large for the shared-memory centroid");
  int total_iters = 0, widest = 1;
  for (int p = 0; p < nplan; ++p) {
    PBB_CHECK_ARG(plan[3 * p] >= 0 && plan[3 * p + 1] >= 0 && plan[3 * p + 2] <= F && plan[3 * p + 1] < plan[3 * p + 2],
                  5, "alignment plan entry out of range");
    total_iters += plan[3 * p];
    if (plan[3 * p + 2] - plan[3 * p + 1] > widest) widest = plan[3 * p + 2] - plan[3 * p + 1];
  }
  *c = DhtvCall{features, mapping, nplan, K, F, T, metric, algorithm, total_iters, widest};
  return 0;
}

#ifdef PBB_PHASE_TIMING
// Prints and clears the cycles the kernel that just ran on st spent in each of its 8 phases (DH_PH).
static void print_dhtv_phases(cudaStream_t st, const char* tag, const char* const (&names)[8]) {
  unsigned long long ph[8], zero[8] = {0};
  cudaStreamSynchronize(st);
  cudaMemcpyFromSymbol(ph, g_dhtv_phase, sizeof(ph));
  cudaMemcpyToSymbol(g_dhtv_phase, zero, sizeof(zero));
  for (int i = 0; i < 8; ++i) fprintf(stderr, "[%s] %-26s %10llu cycles\n", tag, names[i], ph[i]);
}
#endif

// dhtv_cluster_kernel, when the widest segment fits one thread-block cluster and a cluster of 16 (non-portable size)
// or 8 CTAs can be scheduled.  *launched stays false when it does not apply.
static int launch_dhtv_cluster(const DhtvCall& c, cudaStream_t st, bool* launched) {
  static int cluster_ctas = -1;  // 16 (non-portable size), 8, or 0 = not available
  for (int C = cluster_ctas < 0 ? 16 : cluster_ctas; C >= 8; C /= 2) {
    const int per = (c.widest + C - 1) / C;
    const size_t smem = (size_t)(2 + per) * c.K * c.T * sizeof(double);
    if (per > kDhtvClMaxLocal || smem > 200 * 1024) break;
    using ClusterKern = void (*)(double*, const int*, int, int, int, int, long long*, int, int);
    const ClusterKern kern = c.K == 2 ? dhtv_cluster_kernel<2> : c.K == 3 ? dhtv_cluster_kernel<3>
                             : c.K == 4 ? dhtv_cluster_kernel<4> : dhtv_cluster_kernel<0>;
    PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if (C > 8) PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    const ClusterLaunch cl(C, kDhtvClThreads, smem, C, st);
    if (cluster_ctas < 0) {
      int nclusters = 0;
      if (cudaOccupancyMaxActiveClusters(&nclusters, kern, &cl.cfg) != cudaSuccess || nclusters < 1) {
        (void)cudaGetLastError();
        if (C == 8) cluster_ctas = 0;
        continue;  // try the portable size
      }
      cluster_ctas = C;
    }
    PBB_TRY(launch_ex("dhtv_cluster_kernel", cl.cfg, kern, c.features, c.plan_dev, c.nplan, c.K, c.F, c.T, c.mapping,
                      c.metric, c.algorithm));
    *launched = true;
#ifdef PBB_PHASE_TIMING
    print_dhtv_phases(st, "dhtv cluster", {"segment load (+store)", "partial sums", "barrier 1 + reduce-scatter",
                                           "cluster barrier 2", "norms + scores", "assignment", "permutation",
                                           "cluster barrier 3"});
    unsigned long long its = 0, z = 0;
    cudaMemcpyFromSymbol(&its, g_dhtv_iters, sizeof(its));
    cudaMemcpyToSymbol(g_dhtv_iters, &z, sizeof(z));
    fprintf(stderr, "[dhtv cluster] iterations executed %llu of %d planned\n", its, c.total_iters);
#endif
    return 0;
  }
  return 0;
}

// dhtv_coop_kernel: one CTA per bin of the widest segment, as many as can be resident.
static int launch_dhtv_coop(const DhtvCall& c, int dev, cudaStream_t st) {
  const size_t smem = (size_t)c.K * c.T * sizeof(double);
  PBB_CUDA(cudaFuncSetAttribute(dhtv_coop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  int per_sm = 0, sms = 0;
  int warps = c.K * c.K < kDhtvCoopMaxWarps ? c.K * c.K : kDhtvCoopMaxWarps;
  if (warps < 4) warps = 4;  // the centroid norms are summed by the first 128 threads
  const int threads = 32 * warps;
  PBB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dhtv_coop_kernel, threads, smem));
  PBB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int grid = c.widest;
  if (grid > per_sm * sms) grid = per_sm * sms;
  if (grid < 1) grid = 1;
  const CoopLaunch cl(grid, threads, smem, st);
  PBB_TRY(launch_ex("dhtv_coop_kernel", cl.cfg, dhtv_coop_kernel, c.features, c.partial, c.changed, c.plan_dev, c.nplan,
                    c.K, c.F, c.T, c.mapping, c.bar, c.metric, c.algorithm));
#ifdef PBB_PHASE_TIMING
  print_dhtv_phases(st, "dhtv", {"phase A", "barrier 1", "centroid combine", "centroid norms", "scores", "assignment",
                                 "permute/rest", "barrier 2"});
#endif
  return 0;
}

}  // namespace pbb

using namespace pbb;

extern "C" {

int pbb_dhtv_mapping(const double* mask, int K, int F, int T, const int* plan, int nplan, double* features,
                     double* centroid, long long* mapping, void* stream) {
  return pbb_dhtv_mapping_ex(mask, K, F, T, plan, nplan, features, centroid, mapping, 1, 0, stream);
}

int pbb_dhtv_mapping_ex(const double* mask, int K, int F, int T, const int* plan, int nplan, double* features,
                        double* centroid, long long* mapping, int metric, int algorithm, void* stream) {
  DhtvCall c;
  if (int rc = check_dhtv_args(mask, K, F, T, plan, nplan, features, centroid, mapping, metric, algorithm, &c)) return rc;
  // segments too wide for a cluster run on dhtv_coop_kernel, which needs a cooperative launch (every H100 has it)
  int dev = 0, coop = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  PBB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) { set_error("DHTV alignment: device %d does not support cooperative launch", dev); return 1; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  c.partial = centroid;
  c.changed = reinterpret_cast<int*>(centroid + (size_t)kDhtvSlices * K * T);
  c.bar = reinterpret_cast<unsigned*>(c.changed + c.total_iters + 1);  // zeroed with the flags
  c.plan_dev = c.changed + c.total_iters + 2;
  PBB_CUDA(cudaMemsetAsync(c.changed, 0, (size_t)(c.total_iters + 2) * sizeof(int), st));
  if (metric == 1)
    PBB_TRY(launch_kernel("dhtv_normalize_kernel", dhtv_normalize_kernel, K * F, 128, 0, st, mask, features, K * F, T));
  else
    PBB_CUDA(cudaMemcpyAsync(features, mask, (size_t)K * F * T * sizeof(double), cudaMemcpyDeviceToDevice, st));
  PBB_TRY(launch_kernel("dhtv_init_mapping_kernel", dhtv_init_mapping_kernel, (K * F + 255) / 256, 256, 0, st, mapping,
                        K, F));
  PBB_CUDA(cudaMemcpyAsync(c.plan_dev, plan, (size_t)3 * nplan * sizeof(int), cudaMemcpyHostToDevice, st));
  // The reference's plans (~100-bin segments) fit a cluster.  PBB_DHTV_COOP=1 keeps the grid-barrier kernel (A/B).
  static const bool no_cluster = getenv("PBB_DHTV_COOP") != nullptr;
  bool launched = false;
  if (int rc = no_cluster ? 0 : launch_dhtv_cluster(c, st, &launched)) return rc;
  return launched ? 0 : launch_dhtv_coop(c, dev, st);
}

// doubles of `centroid` scratch pbb_dhtv_mapping needs
size_t pbb_dhtv_scratch_doubles(int K, int T, const int* plan, int nplan) {
  size_t iters = 0;
  for (int p = 0; p < nplan; ++p) iters += (size_t)plan[3 * p];
  // partial sums, the per-iteration "changed" flags, the device copy of the plan
  return (size_t)kDhtvSlices * K * T + (iters + 3) / 2 + 2 + ((size_t)3 * nplan + 1) / 2 + 1;
}

int pbb_apply_mapping(const double* mask, const long long* mapping, int K, int F, int T, double* out,
                      void* stream) {
  PBB_CHECK_ARG(mask != nullptr, 1, "mask is null");
  PBB_CHECK_ARG(mapping != nullptr, 2, "mapping is null");
  PBB_CHECK_ARG(K > 0 && K < 20 && F > 0 && T > 0, 3, "bad shape (K < 20, permutation_alignment.py:102)");
  PBB_CHECK_ARG(out != nullptr, 6, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("apply_mapping_kernel", apply_mapping_kernel, K * F, 128, 0, st, mask, mapping, K, F, T, out);
}

int pbb_score_matrix(const double* mask, const double* reference, long long mask_source_stride,
                     long long reference_source_stride, int K, int F, int T, int metric, double* scores,
                     void* stream) {
  PBB_CHECK_ARG(mask != nullptr, 1, "mask is null");
  PBB_CHECK_ARG(reference != nullptr, 2, "reference mask is null");
  PBB_CHECK_ARG(K > 0 && K <= kDhtvMaxK, 5, "need 0 < K < 10 (permutation_alignment.py:690)");
  PBB_CHECK_ARG(F > 0 && T > 0, 6, "F and T must be positive");
  PBB_CHECK_ARG(metric >= 0 && metric <= 2, 8, "metric: 0 multiply, 1 cos, 2 euclidean");
  PBB_CHECK_ARG(scores != nullptr, 9, "scores is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("score_matrix_kernel", score_matrix_kernel, (F + 3) / 4, 128, 0, st, mask, reference,
                       mask_source_stride, reference_source_stride, K, F, T, metric, scores);
}

int pbb_mapping_from_score_matrix(const double* scores, int F, int K, int algorithm, long long* mapping,
                                  int* status, void* stream) {
  PBB_CHECK_ARG(scores != nullptr, 1, "scores is null");
  PBB_CHECK_ARG(F > 0, 2, "F must be positive");
  PBB_CHECK_ARG(K > 0 && K <= kDhtvMaxK, 3, "need 0 < K < 10");
  PBB_CHECK_ARG(algorithm == 0 || algorithm == 1, 4, "algorithm: 0 greedy, 1 optimal");
  PBB_CHECK_ARG(mapping != nullptr, 5, "mapping is null");
  PBB_CHECK_ARG(status != nullptr, 6, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("mapping_from_score_kernel", mapping_from_score_kernel, (F + 63) / 64, 64, 0, st, scores, F, K,
                       algorithm, mapping, status);
}

int pbb_chain_mapping(const long long* pair_mapping, int K, int F, long long* mapping, void* stream) {
  PBB_CHECK_ARG(pair_mapping != nullptr || F == 1, 1, "pair mapping is null");
  PBB_CHECK_ARG(K > 0 && K <= kDhtvMaxK, 2, "need 0 < K < 10");
  PBB_CHECK_ARG(F > 0, 3, "F must be positive");
  PBB_CHECK_ARG(mapping != nullptr, 4, "mapping is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("chain_mapping_kernel", chain_mapping_kernel, 1, 32, 0, st, pair_mapping, K, F, mapping);
}

}  // extern "C"
