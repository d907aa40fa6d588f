// "Sticky bins": the cACGMM fit of FEW bins (D = 8, lean variant), one thread-block cluster per bin for ALL iterations.
//
// em_ws_kernel hands (bin, iteration) tasks to whichever CTA is free; the model and the dependency flag of a bin
// travel through L2 between iterations.  With fewer bins than CTA slots (a rank's shard of a bin-sharded utterance,
// short STFTs) that chain -- sweep, partial sums, update, publish, poll, model load: ~13 us per iteration on an
// H100 -- is all there is, and most SMs idle.  Here a cluster of S = 1, 2 or 4 CTAs keeps ONE bin from the first to
// the last iteration:
//   * CTA p of the cluster holds the ring stages [p n / S, (p + 1) n / S) of the bin's staged observation in shared
//     memory for the whole fit (at most kWsStages of them, copied in once at the start by stage_g2s);
//   * per iteration its four EM warps sweep those frames (the hot loop of em_ws_kernel, unchanged) and leave the
//     scatter sums in shared memory -> cluster barrier -> the update warps of CTA 0 add the S partial sums in rank
//     order through DSMEM (bit-reproducible), update the model (cacg_update_class, unchanged) and store it into
//     every CTA's model buffer through DSMEM -> cluster barrier -> every CTA's EM warps start the next sweep.
// No tickets, no flags, no partial sums through L2, no re-streaming of the observation; the E / M arithmetic, the
// update and therefore the results are those of em_ws_kernel with the frame split (same summation order over the
// parts).  The host uses it when the device runs all F clusters of S CTAs at once (cudaOccupancyMaxActiveClusters)
// and a part fits the ring (n / S <= kWsStages); otherwise em_ws_kernel runs.
#pragma once
#include <cooperative_groups.h>

#include "em_ws.cuh"

namespace pbb {

// Register budget of the EM warps (the helpers get 256 - this), multiple of 8.  200 / 56 instead of em_ws_kernel's
// 208 / 48: the update warps spill less, and a spill reload behind a cluster barrier (which invalidates the L1) is
// an L2 round trip.
constexpr int kStickyEmRegs = 200;

__device__ __forceinline__ void sticky_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

template <int K, typename CT>
__global__ void __launch_bounds__(256, 2) em_sticky_kernel(const PersistArgs a) {
  constexpr int D = 8;
  using SM = WsSmem<D, K, CT>;
  using G = GroupDims<D>;
  constexpr int NS = D * D, M = D / 2, NSG = G::NSG;
  constexpr int NU = K < 3 ? K : 3;  // updater warps
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(smem_raw);
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int S = (int)cluster.num_blocks(), part = (int)cluster.block_rank();
  const int bin = blockIdx.x / S;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int zs = a.zs;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  const int c0 = part * nchunks / S, c1 = (part + 1) * nchunks / S;  // this CTA's ring stages (c1 - c0 <= kWsStages)

  for (int s = tid; s < NS; s += blockDim.x) sm.tab[s] = slot_pack(D, s);
  if (tid == 0) {
    for (int s = 0; s < kWsStages; ++s) mbar_init(&sm.full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    // the part's observation: resident for the whole fit
    const CT* __restrict__ zbase = reinterpret_cast<const CT*>(a.z);
    for (int c = c0; c < c1; ++c) stage_g2s<D>(sm.zbuf[c - c0], zbase, bin, nchunks, c, &sm.full[c - c0]);
  }

  if (warp < M) {
    // =============================== EM warps ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kStickyEmRegs));
    const int g = warp;
#pragma unroll 1
    for (int it = 0; it < a.iterations; ++it) {
      const bool mstep_only = a.first_is_m && it == 0;
      double acc[K * NSG];
#pragma unroll
      for (int i = 0; i < K * NSG; ++i) acc[i] = 0.0;
      double sg[K];
#pragma unroll
      for (int k = 0; k < K; ++k) sg[k] = 0.0;
#pragma unroll 1
      for (int c = c0; c < c1; ++c) {
        const int st = c - c0;
        mbar_wait(&sm.full[st], 0u);  // completes once; later iterations pass straight through
        ws_stage<K, CT>(a, sm, 0, g, bin, st, c, lane, mstep_only, acc, sg);
      }
      ws_task_end<K, CT>(a, sm, 0, g, c1, nchunks, lane, mstep_only, sg);
      warp_reduce_halving<K * NSG>(acc, lane);
      store_group_sums<D, K>(acc, g, lane, sm.S[0]);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double v = warp_sum(sg[k]);
        if (lane == 0) sm.sgp[0][g][k] = v;
      }
      sticky_cluster_sync();  // (1) every part's sums are complete
      sticky_cluster_sync();  // (2) CTA 0 has stored the new model into every CTA's shared memory
      if (it + 1 < a.iterations) {
        // weights and ew from the raw scalars (sum of gamma, log det), as the producer warp of em_ws_kernel does
        if (tid < K) sm.ew[0][tid] = lean_ew<K>(sm.S[1][tid][NS], sm.ld[tid], sm.ld, a.weight_mode, a.T);
        asm volatile("bar.sync 1, %0;" ::"n"(32 * M) : "memory");
      }
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(256 - kStickyEmRegs));
    const int u = warp - M - 1;  // updater index (warp M only keeps the barriers company)
#pragma unroll 1
    for (int it = 0; it < a.iterations; ++it) {
      sticky_cluster_sync();  // (1)
      if (part == 0 && u >= 0 && u < NU) {
        const bool last_it = it == a.iterations - 1;
        // sums over the parts in rank order (fixed: the result does not depend on timing); sum of gamma = the four
        // groups' shares of every part
        for (int k = u; k < K; k += NU) {
          for (int i = lane; i < NS + 1; i += 32) {
            double v = 0.0;
            for (int p = 0; p < S; ++p) {
              if (i < NS) {
                v += *cluster.map_shared_rank(&sm.S[0][k][i], p);
              } else {
                const double* sp = cluster.map_shared_rank(&sm.sgp[0][0][k], p);
                v += (sp[0] + sp[K]) + (sp[2 * K] + sp[3 * K]);
              }
            }
            sm.S[1][k][i] = v;
          }
        }
        __syncwarp();
        if (last_it) {
          // leave the raw sums for cacg_update_kernel (reference-exact eigendecomposition)
          double* __restrict__ po = a.part + (size_t)bin * K * (NS + 1);
          for (int k = u; k < K; k += NU)
            for (int i = lane; i < NS + 1; i += 32) po[k * (NS + 1) + i] = sm.S[1][k][i];
        } else {
          for (int k = u; k < K; k += NU) {
            // the class model goes to a staging row in this CTA's shared memory, then into every CTA's model buffer
            // through DSMEM: no L2 round trip between the update and the next sweep
            cacg_update_class<D, false>(a, bin, k, K, lane, sm.A[k], sm.V[k], sm.lam[k], sm.S[1][k], sm.tab, &sm.ld[k],
                                        &sm.coef[1][k][0]);
            __syncwarp();
            const double c0v = sm.coef[1][k][lane], c1v = sm.coef[1][k][lane + 32];
            const double ldk = sm.ld[k], sgam = sm.S[1][k][NS];
            for (int p = 0; p < S; ++p) {
              double* rc = cluster.map_shared_rank(&sm.coef[0][k][0], p);
              rc[lane] = c0v;
              rc[lane + 32] = c1v;
              if (lane == 0 && p != 0) {
                *cluster.map_shared_rank(&sm.ld[k], p) = ldk;
                *cluster.map_shared_rank(&sm.S[1][k][NS], p) = sgam;
              }
            }
          }
        }
      }
      sticky_cluster_sync();  // (2)
    }
  }
}

}  // namespace pbb
