// Warp-specialised persistent cACGMM EM kernel (D = 8 microphones, lean variant).
//
// Same task model, numerics and global protocol as em_persistent.cuh (task = one EM iteration
// of one bin, atomic tickets, per-bin release/acquire flags, Gauss-Jordan model update with the
// Jacobi fallback), but the CTA is split into two warpgroups with different jobs and register
// budgets (setmaxnreg), so that everything that is not E-step / M-step arithmetic leaves the
// critical path of the four slot-group warps:
//
//   warpgroup 0, warps 0..3  "EM"       the hot loop of em_persistent.cuh, nothing else: wait for a
//                                       staged model, consume ring stages, reduce, hand the scatter
//                                       sums over and start the next task immediately
//   warpgroup 1, warp  4     "producer" tickets, task order, dependency flags, model -> shared
//                                       memory, 1-D TMA bulk copies of the observation chunks into
//                                       a 3-stage ring, always up to three chunks ahead
//   warpgroup 1, warps 5..7  "update"   one class each: scatter sums -> inverse -> coefficients in
//                                       L2, then the bin's flag; runs while the EM warps are
//                                       already busy with the next task
//
// All hand-overs are shared-memory mbarriers (full/empty pairs); the E-step exchange of the four
// EM warps is named barrier 1, the updaters meet on named barrier 2.  The per-bin flag release
// keeps the cross-CTA protocol of em_persistent.cuh.
//
// Frame split (PersistArgs::tsplit = S > 1, chosen by the host when there are fewer bins than CTA slots): a task is
// one EM iteration of one bin over the ring stages [p * nchunks / S, (p + 1) * nchunks / S), S consecutive tickets per
// (bin, iteration).  Every part leaves its scatter sums in tpart[bin][p]; the part that arrives last (tcount[bin],
// one atomic per part) adds the S partial sums in the order p = 0 .. S-1 -- so the result does not depend on which
// CTA that was -- and updates the model as before.  This shortens the per-bin dependency chain (the E / M sweep is
// the longest link) at the price of one more L2 round trip per iteration.
#pragma once
#include "em_persistent.cuh"

namespace pbb {

constexpr int kWsLead = 2;  // chunks the EM warps have left when the producer takes the next ticket
constexpr int kWsStages = 3;
constexpr int kWsEmRegs = 208;  // 128 threads x 208 + 128 threads x 48 = 32768 = 256 x 128
constexpr int kWsHelperRegs = 256 - kWsEmRegs;

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// mbarrier wait for the helper warps: they are latency tolerant, so they poll at a low rate
// instead of competing with the EM warps of their scheduler for issue slots
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, unsigned ns) {
  while (true) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(ns);
  }
}

template <int D, int K, typename CT>
struct WsSmem {
  static constexpr int NS = D * D;
  static constexpr int M = D / 2;
  static constexpr int ROWS = stage_rows(D);
  CT zbuf[kWsStages][ROWS][kStageFrames];
  double2 A[K][NS];       // updaters: scatter matrix / inverse
  double2 V[K][NS];       // updaters: eigenvectors (Jacobi fallback)
  double coef[2][K][NS];  // model of the current / next task (producer writes, EM reads)
  double xq[2][M][2 * K][32];
  double cwx[K][64];       // gamma / q per (class, frame of the step)
  double sgp[2][M][K];     // sum of gamma per slot-group warp
  double S[2][K][NS + 1];  // scatter sums of the last / second last task (EM writes, updaters read)
  double lam[K][D];
  double ld[K];
  alignas(16) double ew[2][4];
  int tab[NS];
  int desc[2][4];    // per model buffer: bin, iteration, part (bin < 0: no more tasks)
  int sdesc[2][4];   // per S buffer: bin, iteration, part
  int tlast;         // frame split: this CTA delivered the last part of the iteration
  uint64_t full[kWsStages], empty[kWsStages];
  uint64_t model_full[2], model_empty[2];
  uint64_t s_full[2], s_empty[2];
};

// EM warp g's share of one ring stage st (chunk c of the bin) in em_ws_kernel and em_sticky_kernel, model buffer mb.
// The E + M sweep computes the posterior once per frame (lean_chunk2_split: -3 % on C2), so sg counts the frames
// this warp evaluated; in the odd tail step of a short last chunk every group evaluates all 32 frames and only group
// 0 counts them.  The M-step-only pass counts gamma in every group (ws_task_end keeps group 0's).
template <int K, typename CT>
__device__ __forceinline__ void ws_stage(const PersistArgs& a, WsSmem<8, K, CT>& sm, int mb, int g, int bin, int st,
                                         int c, int lane, bool mstep_only,
                                         double (&acc)[K * GroupDims<8>::NSG], double (&sg)[K]) {
  constexpr int D = 8;
  const int t_chunk = c * kStageFrames;
  const int nsteps = (min(kStageFrames, a.zs - t_chunk)) >> 5;
  int buf = 0;
  if (!mstep_only) {
    lean_chunk2_split<D, K, CT>(sm, mb, g, st, nsteps >> 1, lane, a.aff_eps, acc, sg);
    if (nsteps & 1) {
      double sgt[K];
#pragma unroll
      for (int k = 0; k < K; ++k) sgt[k] = 0.0;
      lean_step<D, K, CT, 0, true>(sm, mb, g, st, nsteps - 1, lane, buf, a.aff_eps, acc, sgt);
#pragma unroll
      for (int k = 0; k < K; ++k) sg[k] += g == 0 ? sgt[k] : 0.0;
    }
  } else {
    general_chunk<D, K, CT, false>(a, sm, g, bin, st, t_chunk, nsteps, lane, buf, true, true, acc, sg);
  }
}

// End of EM warp g's sweep of stages [.., c1): every padded frame was counted once, by whichever warp evaluated it,
// so group 0 takes them out; the M-step-only pass keeps group 0's sum of gamma only.
template <int K, typename CT>
__device__ __forceinline__ void ws_task_end(const PersistArgs& a, const WsSmem<8, K, CT>& sm, int mb, int g, int c1,
                                            int nchunks, int lane, bool mstep_only, double (&sg)[K]) {
  if (!mstep_only && a.zs > a.T && c1 == nchunks) {
    double gp[K];
    padded_gamma<8, K, 0>(sm, mb, a.aff_eps, gp);
    const int npad_lane = (g == 0 && lane >= 32 - (a.zs - a.T)) ? 1 : 0;
#pragma unroll
    for (int k = 0; k < K; ++k) sg[k] -= npad_lane ? gp[k] : 0.0;
  }
  if (mstep_only && g != 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) sg[k] = 0.0;
  }
}

template <int K, typename CT>
__global__ void __launch_bounds__(256, 2) em_ws_kernel(const PersistArgs a) {
  constexpr int D = 8;
  using SM = WsSmem<D, K, CT>;
  using G = GroupDims<D>;
  constexpr int NS = D * D, M = D / 2, NSG = G::NSG;
  constexpr int NU = K < 3 ? K : 3;  // updater warps
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int F = a.F, T = a.T, zs = a.zs;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  const int S = a.tsplit > 1 ? a.tsplit : 1;  // parts per (bin, iteration); the host keeps S <= nchunks
  const int total = a.iterations * F * S;

  for (int s = tid; s < NS; s += blockDim.x) sm.tab[s] = slot_pack(D, s);
  if (tid == 0) {
    for (int s = 0; s < kWsStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], M); }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&sm.model_full[s], 1);
      mbar_init(&sm.model_empty[s], M);
      mbar_init(&sm.s_full[s], M);
      mbar_init(&sm.s_empty[s], NU);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < M) {
    // =============================== EM warps ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWsEmRegs));
    const int g = warp;
    unsigned chunk_cnt = 0;
#ifdef PBB_PHASE_TIMING
    long long _tp = clock64();
#endif
#pragma unroll 1
    for (unsigned n = 0;; ++n) {
      const int mb = n & 1;
      mbar_wait(&sm.model_full[mb], (n >> 1) & 1u);
      PBB_PH(0);  // wait for the staged model
      const int bin = sm.desc[mb][0], it = sm.desc[mb][1], part = sm.desc[mb][2];
      const int c0 = part * nchunks / S, c1 = (part + 1) * nchunks / S;
      if (bin < 0) {
        // no more tasks: tell the updaters
        const int sb = n & 1;
        mbar_wait(&sm.s_empty[sb], ((n >> 1) & 1u) ^ 1u);
        if (lane == 0) {
          if (g == 0) sm.sdesc[sb][0] = -1;
          mbar_arrive(&sm.s_full[sb]);
        }
        break;
      }
      const bool mstep_only = a.first_is_m && it == 0;
      double acc[K * NSG];
#pragma unroll
      for (int i = 0; i < K * NSG; ++i) acc[i] = 0.0;
      double sg[K];
#pragma unroll
      for (int k = 0; k < K; ++k) sg[k] = 0.0;
#pragma unroll 1
      for (int c = c0; c < c1; ++c) {
        const int st = chunk_cnt % kWsStages;
        mbar_wait(&sm.full[st], (chunk_cnt / kWsStages) & 1u);
        PBB_PH(2);  // TMA wait
        ws_stage<K, CT>(a, sm, mb, g, bin, st, c, lane, mstep_only, acc, sg);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[st]);
        ++chunk_cnt;
        PBB_PH(3);  // EM steps
      }
      ws_task_end<K, CT>(a, sm, mb, g, c1, nchunks, lane, mstep_only, sg);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.model_empty[mb]);  // done with this task's model

      warp_reduce_halving<K * NSG>(acc, lane);
      const int sb = n & 1;
      PBB_PH(4);  // reduce
      mbar_wait(&sm.s_empty[sb], ((n >> 1) & 1u) ^ 1u);  // updaters are done with task n - 2
      PBB_PH(5);  // wait for the S buffer
      store_group_sums<D, K>(acc, g, lane, sm.S[sb]);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double v = warp_sum(sg[k]);
        if (lane == 0) sm.sgp[sb][g][k] = v;
      }
      if (g == 0 && lane == 0) { sm.sdesc[sb][0] = bin; sm.sdesc[sb][1] = it; sm.sdesc[sb][2] = part; }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.s_full[sb]);
      PBB_PH(6);  // hand-over
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWsHelperRegs));
    if (warp == M) {
      // =============================== producer ===============================
      const CT* __restrict__ zbase = reinterpret_cast<const CT*>(a.z);
      unsigned chunk_cnt = 0;
#pragma unroll 1
      for (unsigned n = 0;; ++n) {
        const int mb = n & 1;
        int t = 0;
        if (lane == 0) t = atomicAdd(a.ticket, 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        int bin = -1, it = 0, part = 0;
        if (t < total) decode_task(a, t, S, order_entry(a, t, S), bin, it, part);
        const int c0 = part * nchunks / S, ncp = (part + 1) * nchunks / S - c0;  // this task's ring stages
        const bool mstep_only = a.first_is_m && it == 0;
        int issued = 0;  // chunks of this task already requested (lane 0)
        auto issue_chunks = [&](int upto, bool blocking) {
          // lane 0: request chunks [issued, upto) of this task; non-blocking stops at a busy stage
          while (issued < upto) {
            const int st = chunk_cnt % kWsStages;
            const uint32_t par = ((chunk_cnt / kWsStages) & 1u) ^ 1u;
            if (blocking) {
              mbar_wait_relaxed(&sm.empty[st], par, 100);
            } else {
              uint32_t done;
              asm volatile(
                  "{\n"
                  ".reg .pred p;\n"
                  "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
                  "selp.u32 %0, 1, 0, p;\n"
                  "}\n"
                  : "=r"(done)
                  : "r"(smem_u32(&sm.empty[st])), "r"(par)
                  : "memory");
              if (!done) break;
            }
            stage_g2s<D>(sm.zbuf[st], zbase, bin, nchunks, c0 + issued, &sm.full[st]);
            ++chunk_cnt;
            ++issued;
          }
        };
        if (bin >= 0 && lane == 0) {
          // streamed upload: the bin's observation is in place once flags[bin] >= 0 (stream_load_kernel), which a
          // task of any iteration may see before; the staged rows were written with ordinary stores by another
          // CTA, so order them before this CTA's async-proxy (TMA) reads
          bool z_ready = !a.wait_load;
          if (!z_ready && ld_acquire_gpu(a.flags + bin) >= 0) {
            asm volatile("fence.proxy.async;" ::: "memory");
            z_ready = true;
          }
          // the observation does not depend on the model: request what fits into the ring right away, so
          // that the copy overlaps the flag / model round trips below
          if (z_ready) issue_chunks(ncp, false);
          // dependency: the bin's previous iteration (or its arrival, streamed upload)
          if (mstep_only) {
            if (a.wait_load) while (ld_acquire_gpu(a.flags + bin) < 0) __nanosleep(200);
          } else {
            while (ld_acquire_gpu(a.flags + bin) < it) {
              if (z_ready) issue_chunks(ncp, false);  // keep the ring filled while the dependency is still executing
              __nanosleep(40);
            }
          }
          if (!z_ready) asm volatile("fence.proxy.async;" ::: "memory");
        }
        __syncwarp();
        mbar_wait_relaxed(&sm.model_empty[mb], ((n >> 1) & 1u) ^ 1u, 100);  // EM warps are done with task n - 2
        if (bin >= 0 && !mstep_only) {
          const double* __restrict__ cf = a.coef + (size_t)bin * K * NS;
          for (int i = lane; i < K * NS; i += 32) (&sm.coef[mb][0][0])[i] = __ldcg(cf + i);
          if (lane < K) {
            // weights and ew from the published raw scalars (sum of gamma, log det)
            double ld[K];
#pragma unroll
            for (int j = 0; j < K; ++j) ld[j] = __ldcg(a.ld + (size_t)bin * 4 + j);
            sm.ew[mb][lane] = lean_ew<K>(__ldcg(a.ew + (size_t)bin * 4 + lane), __ldcg(a.ld + (size_t)bin * 4 + lane),
                                         ld, a.weight_mode, T);
          }
        }
        if (lane == 0) { sm.desc[mb][0] = bin; sm.desc[mb][1] = it; sm.desc[mb][2] = part; }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.model_full[mb]);
        if (bin < 0) break;
        if (lane == 0) {
          issue_chunks(ncp, true);
          // Do not take the next ticket too early: with two tickets per CTA in flight the grid holds
          // more tasks than there are bins and most dependencies are still executing.  Wait until the
          // EM warps have ~2 chunks left (enough to hide ticket, flag and model latency).
          const unsigned x = chunk_cnt - (unsigned)(ncp >= kWsLead + 1 ? kWsLead + 1 : ncp);
          mbar_wait_relaxed(&sm.empty[x % kWsStages], (x / kWsStages) & 1u, 100);
        }
        __syncwarp();
      }
    } else if (warp - M - 1 < NU) {
      // =============================== updaters ===============================
      const int u = warp - M - 1;
#ifdef PBB_PHASE_TIMING
      long long _tp = clock64();
#undef PBB_PH
#define PBB_PH(i) do { if (u == 0 && lane == 0) { long long _t = clock64(); atomicAdd(&a.phase[i], (unsigned long long)(_t - _tp)); _tp = _t; } } while (0)
#endif
#pragma unroll 1
      for (unsigned n = 0;; ++n) {
        const int sb = n & 1;
        mbar_wait_relaxed(&sm.s_full[sb], (n >> 1) & 1u, 100);
        PBB_PH(7);  // updater idle
        const int bin = sm.sdesc[sb][0], it = sm.sdesc[sb][1];
        if (bin < 0) break;
        const bool last_it = it == a.iterations - 1;
        // sum of gamma = the four groups' shares, added in a fixed order
        for (int k = u; k < K; k += NU)
          if (lane == 0)
            sm.S[sb][k][NS] = (sm.sgp[sb][0][k] + sm.sgp[sb][1][k]) + (sm.sgp[sb][2][k] + sm.sgp[sb][3][k]);
        __syncwarp();
        if (last_it && S == 1) asm volatile("bar.sync 2, %0;" ::"n"(NU * 32) : "memory");
        if (S > 1) {
          // frame split: leave this part's sums in L2; whoever delivers the last part adds them up in a fixed order
          const int part = sm.sdesc[sb][2];
          constexpr int kRow = K * (NS + 1);
          double* __restrict__ tp = a.tpart + ((size_t)bin * S + part) * kRow;
          for (int k = u; k < K; k += NU)
            for (int i = lane; i < NS + 1; i += 32) __stcg(tp + k * (NS + 1) + i, sm.S[sb][k][i]);
          __threadfence();
          asm volatile("bar.sync 2, %0;" ::"n"(NU * 32) : "memory");
          if (u == 0 && lane == 0) sm.tlast = split_last_part(a, bin, it, S);
          asm volatile("bar.sync 2, %0;" ::"n"(NU * 32) : "memory");
          if (!sm.tlast) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.s_empty[sb]);
            continue;  // (tlast is rewritten behind the next task's first updater barrier: everyone has read it by then)
          }
          for (int k = u; k < K; k += NU)
            for (int i = lane; i < NS + 1; i += 32) sm.S[sb][k][i] = split_sum<D, K>(a, bin, S, k * (NS + 1) + i);
          __syncwarp();
          if (last_it) asm volatile("bar.sync 2, %0;" ::"n"(NU * 32) : "memory");
        }
        if (last_it) {
          // leave the raw sums for cacg_update_kernel (reference-exact eigendecomposition)
          double* __restrict__ po = a.part + (size_t)bin * K * (NS + 1);
          for (int i = u * 32 + lane; i < K * (NS + 1); i += NU * 32) po[i] = (&sm.S[sb][0][0])[i];
        } else {
          for (int k = u; k < K; k += NU)
            cacg_update_class<D, false>(a, bin, k, K, lane, sm.A[k], sm.V[k], sm.lam[k], sm.S[sb][k], sm.tab, &sm.ld[k]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.s_empty[sb]);  // S[sb] may be overwritten
        if (!last_it) {
          // every updater's model stores are ordered before the single cumulative release
          asm volatile("bar.sync 2, %0;" ::"n"(NU * 32) : "memory");
          if (u == 0 && lane == 0) st_release_gpu(a.flags + bin, it + 1);
        }
        PBB_PH(1);  // updater busy
      }
    }
  }
}

}  // namespace pbb
