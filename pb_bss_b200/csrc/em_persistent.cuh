// Persistent cACGMM EM kernel: all EM iterations of a fit in ONE launch.
//
// Work unit ("task") = one EM iteration of one frequency bin: E-step with the
// bin's current model fused with the M-step accumulation over all T frames,
// then the model update of that bin.  Tasks are handed out in iteration-major
// order by an atomic ticket counter; bins are independent, so the only
// dependency is task (bin, it) -> (bin, it + 1), tracked by a per-bin
// release/acquire flag in L2.  Because a task only ever waits for a LOWER
// ticket, and tickets are only held by running CTAs, the schedule cannot
// deadlock, needs no grid-wide barrier and balances itself to within one task
// (F = 513 bins do not divide 132 SMs; 51300 tasks do).
//
// Inside a task the CTA is D/2 warps; warp g owns slot group g (common.cuh) and
// lane = frame.  The observation rows of the bin stream from L2 into a 2-stage
// shared-memory ring with 1-D TMA bulk copies (cp.async.bulk + mbarrier
// complete_tx), prefetched one 128-frame chunk ahead -- across task boundaries,
// so the next bin's first chunk arrives while this bin's model is updated.
//
// Model update per (bin, class): the E-step only needs B^{-1} and log det B up
// to a common scale (log_pdf = -D log q - log det is invariant to B -> s B,
// and gamma/q rescales the next scatter matrix by the same s), so intermediate
// iterations invert the trace-normalised scatter matrix by Gauss-Jordan
// elimination (HPD: no pivoting) instead of an eigendecomposition.  That is
// exact unless the reference would floor an eigenvalue
// (complex_angular_central_gaussian.py:111-126); the bound
// lambda_min / lambda_max >= 1 / (tr(A) tr(A^{-1})) > floor proves it would
// not.  If the bound fails (cond > ~1e9) the warp falls back to the Jacobi
// eigensolver with the reference's normalise-and-floor semantics.  The last
// iteration always leaves the raw scatter sums for cacg_update_kernel, which
// produces the reference-exact eigenvectors / eigenvalues / weights.
#pragma once
#include "common.cuh"
#include "em_kernels.cuh"
#include "heig.cuh"

namespace pbb {

#ifdef PBB_PHASE_TIMING
#define PBB_PH(i) do { if (tid == 0) { long long _t = clock64(); atomicAdd(&a.phase[i], (unsigned long long)(_t - _tp)); _tp = _t; } } while (0)
#else
#define PBB_PH(i) do { } while (0)
#endif

struct PersistArgs {
  const void* z;   // staged layout (F, nchunks, D, kStageFrames): the channel rows of a ring stage are one
                   // contiguous block (zero padded), see normalize_staged_kernel and stage_g2s
  int zs;          // padded frame count, multiple of 32
  int F, T;
  int iterations;  // EM iterations in this launch
  int first_is_m;  // iteration 0 is an M-step from aff_in with q = 1 (cacgmm.py:206-228)
  int user_model;  // iteration 0 uses a user supplied model: log-domain softmax
  int softmax_fast;
  const double* aff_in;     // (F, K, T)
  const double* saliency;   // (F, T) or null      [FULL]
  const uint8_t* activity;  // (F, K, T) or null   [FULL]
  double aff_eps;
  double eigenvalue_floor;
  int covariance_norm;
  int weight_mode;
  double* coef;  // (F, K, NS)   model state, updated in place
  double* ld;    // (F, K)
  double* w;     // (F, K)
  double* ew;    // (F, K)
  double* part;  // (F, K, NS + 1) raw scatter sums of the last iteration
  int* flags;    // (F) number of model updates published for the bin
  int* ticket;   // (1)
  const int* dead;  // (F) bin has an all-zero observation frame (set by normalize_staged_kernel)
  int* status;
  CwSpline spline;  // complex Watson only: inverse hypergeometric ratio (model_kind 1)
  int wave_c;      // task order: 0 = iteration-major; c > 0 = rounds, c bins join per round (decode_ticket)
  int wait_load;   // streamed upload: the bin's first task waits for flags[bin] >= 0 (stream_load_kernel)
  const int* order;  // optional explicit task order: order[ticket] = bin | iteration << 16 (host-built, api_cacgmm.cu)
  unsigned long long* phase;  // debug: per-phase cycle sums (PBB_PHASE_TIMING builds)
  int tsplit;      // em_ws_kernel: parts (ranges of ring stages) one EM iteration of a bin is split into, 0 / 1 = none
  double* tpart;   // (F, tsplit, K, NS + 1) scatter sums per part
  int* tcount;     // (F) parts delivered so far, zero at launch
};

// ---- PTX helpers --------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

constexpr int kStageFrames = 128;  // frames per ring stage (4 steps of 32)

// One ring stage of the staged observation into shared memory, all copies completing on `bar` (armed here for the
// whole stage).  Global memory holds the D channel rows of each (bin, chunk) only, so that the observation the fit
// re-reads every iteration stays small enough for L2; the stage in shared memory has stage_rows(D) rows.  One bulk
// copy brings the channel rows, then one per repeated row (common.cuh) copies its channel row again -- from the L2
// lines the first copy has just brought in.
template <int D, typename CT>
__device__ __forceinline__ void stage_g2s(CT (*dst)[kStageFrames], const CT* z, int bin, int nchunks, int chunk,
                                          uint64_t* bar) {
  constexpr int ROWS = stage_rows(D);
  constexpr uint32_t kRowBytes = kStageFrames * sizeof(CT);
  const CT* src = z + ((size_t)bin * nchunks + chunk) * (D * kStageFrames);
  mbar_expect_tx(bar, ROWS * kRowBytes);
  bulk_g2s(dst[0], src, D * kRowBytes, bar);
#pragma unroll
  for (int r = D; r < ROWS; ++r) bulk_g2s(dst[r], src + row_channel(D, r) * kStageFrames, kRowBytes, bar);
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// reciprocal without the slow-path branches of 1.0 / x: hardware seed + 2 Newton
// steps; exact to ~1 ulp for normal, finite x (here 1e-300 < x < 1e300).
__device__ __forceinline__ double fast_rcp(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  return r;
}

// ---- task order ------------------------------------------------------------------
// wave_c == 0: iteration-major, ticket = it * F + bin.
// wave_c = c > 0 (streamed upload): the bins arrive over PCIe in ascending order while the
// kernel runs, so they join the schedule c at a time, one group per round, and every round
// advances all joined bins by one iteration: round r holds (bin b, iteration r - b / c) for
// b in [min(F, c max(0, r - I + 1)), min(F, c (r + 1))).  Bins that arrived early run ahead
// instead of every CTA queueing behind the link.  Tickets before round r:
// H(r) - H(max(0, r - I)) with H(r) = sum_{j < r} min(F, c (j + 1)).  A task still only
// depends on a lower ticket ((b, it - 1) is one round earlier).
__device__ __forceinline__ long long wave_h(long long r, int F, int c) {
  const long long m = F / c;
  const long long n = r < m ? r : m;
  return (long long)c * n * (n + 1) / 2 + (r - n) * (long long)F;
}
__device__ __forceinline__ long long wave_prefix(int r, int F, int I, int c) {
  return wave_h(r, F, c) - wave_h(r > I ? r - I : 0, F, c);
}
__device__ __forceinline__ void decode_ticket(int t, int F, int I, int c, int& bin, int& it) {
  if (c == 0) {
    it = t / F;
    bin = t - it * F;
    return;
  }
  int lo = 0, hi = I + (F + c - 1) / c - 1;  // last round r with wave_prefix(r) <= t
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (wave_prefix(mid, F, I, c) <= (long long)t) lo = mid; else hi = mid;
  }
  const long long first = (long long)c * (lo - I + 1 > 0 ? lo - I + 1 : 0);
  bin = (int)(first < F ? first : F) + (int)(t - wave_prefix(lo, F, I, c));
  it = lo - bin / c;
}
// Task of ticket t: S consecutive tickets per (bin, iteration) (frame split), part = t mod S.  With the explicit order
// table, ord = order_entry(a, t, S) = bin | iteration << 16 (loaded by the caller, which may issue it early).
__device__ __forceinline__ int order_entry(const PersistArgs& a, int t, int S) {
  return a.order != nullptr ? __ldcg(a.order + t / S) : 0;
}
__device__ __forceinline__ void decode_task(const PersistArgs& a, int t, int S, int ord, int& bin, int& it, int& part) {
  const int tt = t / S;
  part = t - tt * S;
  if (a.order != nullptr) {
    bin = ord & 0xffff;
    it = ord >> 16;
  } else {
    decode_ticket(tt, a.F, a.iterations, a.wave_c, bin, it);
  }
}

__device__ __forceinline__ double2 lds_cplx(const double2* p) { return *p; }
__device__ __forceinline__ double2 lds_cplx(const float2* p) {
  const float2 v = *p;
  return make_double2((double)v.x, (double)v.y);
}

constexpr int kStages = 2;

template <int D, int K, typename CT>
struct PersistSmem {
  static constexpr int NS = D * D;
  static constexpr int M = D / 2;
  static constexpr int ROWS = stage_rows(D);  // channels + repeated rows, see common.cuh
  CT zbuf[kStages][ROWS][kStageFrames];
  double2 A[K][NS];     // scatter matrix / its inverse
  double2 V[K][NS];     // eigenvectors (Jacobi fallback only)
  double2 W[K][NS];     // complex Watson: second scratch of the top-eigenpair iteration
  double coef[2][K][NS];  // E-step form of the bin's model (double buffered: next task's model is prefetched)
  double xq[2][M][2 * K][32];  // partial quadratic forms, up to 2 frames per lane
  double S[K][NS + 1];  // scatter sums + sum of gamma
  alignas(16) double rot[K][((D + 1) / 2) * 6];
  double lam[K][D];
  double ld[K], w[K];
  alignas(16) double ew[2][4];  // w_k exp(ld_min - ld_k) of the current / prefetched model
  alignas(16) double raw[2][8];  // lean variant: published (sum gamma_k, ld_k), padded to 4 + 4, cp.async target
  uint64_t full[kStages];
  int tab[NS];
  int tick[8];            // [0] first ticket; [1..4] next ticket, its bin, iteration, part; [5] frame split: last part
  int ready;              // the next task's model was already published when probed
};

template <int D>
struct GroupDims {
  static constexpr int NSG = group_shape(D).nsg, NLOC = group_shape(D).nloc, NS = D * D;
  static constexpr int NFULL = group_shape(D).nfull, HALF = group_shape(D).half, M = D / 2;
};

// psi slots of one group from its NLOC local channels (order: group_local_slot)
template <int D>
__device__ __forceinline__ void group_psi(const double2 (&x)[GroupDims<D>::NLOC], double (&psi)[GroupDims<D>::NSG]) {
  using G = GroupDims<D>;
  psi[0] = x[0].x * x[0].x + x[0].y * x[0].y;
  psi[1] = x[1].x * x[1].x + x[1].y * x[1].y;
  psi[2] = x[0].x * x[1].x + x[0].y * x[1].y;
  psi[3] = x[0].x * x[1].y - x[0].y * x[1].x;
#pragma unroll
  for (int j = 0; j < G::NFULL; ++j) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const double2 u = x[q / 2], v = x[2 + 2 * j + (q % 2)];
      psi[4 + 8 * j + 2 * q] = u.x * v.x + u.y * v.y;
      psi[4 + 8 * j + 2 * q + 1] = u.x * v.y - u.y * v.x;
    }
  }
  if (G::HALF) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const double2 u = x[h], v = x[2 + 2 * G::NFULL + h];
      psi[4 + 8 * G::NFULL + 2 * h] = u.x * v.x + u.y * v.y;
      psi[4 + 8 * G::NFULL + 2 * h + 1] = u.x * v.y - u.y * v.x;
    }
  }
}

// ---- posterior of one frame, product form -------------------------------------
// gamma_k ~ ew_k / q_k^D  =  ew_k * (prod_{j != k} q_j)^D / (prod_j q_j)^D : no
// logarithm, exponential, minimum or per-class division.  The host enables it
// only when (K-1) * D * log10(1/floor) < 290 so the products stay in range;
// q_k lies in [1/D, 1/floor] after the update's trace normalisation.  A frame
// whose observation is the zero vector has every q_k = 0; the reference floors
// those at `tiny` (cacg.py:198), which makes all classes equal -- reproduced by
// mapping such a frame to q_k = 1.
// Outputs gamma_k (clipped, mixture_model_utils.py:50-53) and
// cw_k = gamma_k / q_k (cacg.py:316-325).
template <int D, int K>
__device__ __forceinline__ void softmax_product(double (&q)[K], const double* __restrict__ ew, double eps,
                                                double (&gam)[K], double (&cw)[K]) {
  const bool dead = q[0] < 1e-200;
#pragma unroll
  for (int k = 0; k < K; ++k) q[k] = dead ? 1.0 : q[k];
  double P[K];
  if constexpr (K == 2) {
    P[0] = q[1]; P[1] = q[0];
  } else if constexpr (K == 3) {
    P[0] = q[1] * q[2]; P[1] = q[0] * q[2]; P[2] = q[0] * q[1];
  } else {
    const double q01 = q[0] * q[1], q23 = q[2] * q[3];
    P[0] = q[1] * q23; P[1] = q[0] * q23; P[2] = q01 * q[3]; P[3] = q01 * q[2];
  }
  double b[K];
  double S = 1e-300;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    b[k] = ew[k] * ipow<D>(P[k]);
    S += b[k];
  }
  const double rS = fast_rcp(S);
  const double rQ = fast_rcp(q[0] * P[0]);
  const double hi = 1.0 - eps;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double g = b[k] * rS;
    if (eps != 0.0) {
      g = g < eps ? eps : g;
      g = g > hi ? hi : g;
    }
    gam[k] = g;
    cw[k] = g * (P[k] * rQ);
  }
}

// Complex Watson posterior (complex_watson.py:73-87 + mixture_model_utils.py:7-55, eps = 0):
// log_pdf_k = kappa_k |m_k^H z|^2 - log c(kappa_k); q_k arrives as the slot form of m m^H.
// The M-step weight is gamma itself (complex_watson.py:307-312 has no 1/q).
template <int K>
__device__ __forceinline__ void softmax_watson(const double (&q)[K], const double* __restrict__ kappa,
                                               const double* __restrict__ lognorm, const double* __restrict__ w,
                                               double (&gam)[K], double (&cw)[K]) {
  double lp[K];
  double m = -INFINITY;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    lp[k] = fma(kappa[k], q[k], -lognorm[k]);
    m = lp[k] > m ? lp[k] : m;
  }
  double den = 0.0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    gam[k] = exp(lp[k] - m) * w[k];
    den += gam[k];
  }
  const double inv = 1.0 / fmax(den, kTiny);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    gam[k] *= inv;
    cw[k] = gam[k];
  }
}

// Hot loop of the lean variant: E-step + M-step of one ring stage for slot
// group g.  All warps run the same instructions (one loop body in the L0
// instruction cache); the staged rows are laid out so that the group's local
// channels are rows 2g .. 2g+NLOC-1, i.e. one base register plus immediates.
// No per-frame masking: padded frames have z = 0, add nothing to the scatter
// sums, and their gamma is subtracted analytically by the caller.
// exchange barrier of the E-step: the whole CTA, or (NAMED) only the D/2 slot-group warps of a
// warp-specialised CTA (em_ws.cuh), which meet on named barrier 1
template <int D, bool NAMED>
__device__ __forceinline__ void em_exchange_barrier() {
  if constexpr (NAMED) asm volatile("bar.sync 1, %0;" ::"n"(32 * (D / 2)) : "memory");
  else __syncthreads();
}

// Front half of a lean step for FR = 1 or 2 frames per lane (frames zrow, zrow + 32): z loads -> psi slots ->
// this group's share of the K quadratic forms, 2K independent FMA chains per frame (coefficients cg, broadcast from
// shared memory) -> partial forms of frame f, class k stored at xw[(f K + k) 32].  The psi slots stay with the caller
// for the M-step.
template <int D, int K, int FR, typename CT>
__device__ __forceinline__ void lean_partial_forms(const CT* __restrict__ zrow, const double* __restrict__ cg,
                                                   double* __restrict__ xw, double (&psi)[FR][GroupDims<D>::NSG]) {
  using G = GroupDims<D>;
  constexpr int NSG = G::NSG, NLOC = G::NLOC, NS = G::NS;
  {
    double2 x[NLOC];
#pragma unroll
    for (int f = 0; f < FR; ++f) {
#pragma unroll
      for (int l = 0; l < NLOC; ++l) x[l] = lds_cplx(zrow + l * kStageFrames + 32 * f);
      group_psi<D>(x, psi[f]);
    }
  }
  double p0[FR][K], p1[FR][K];
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int f = 0; f < FR; ++f) { p0[f][k] = 0.0; p1[f][k] = 0.0; }
#pragma unroll
  for (int i = 0; i < NSG; i += 2) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double2 cc = *reinterpret_cast<const double2*>(cg + k * NS + i);
#pragma unroll
      for (int f = 0; f < FR; ++f) p0[f][k] = fma(cc.x, psi[f][i], p0[f][k]);
#pragma unroll
      for (int f = 0; f < FR; ++f) p1[f][k] = fma(cc.y, psi[f][i + 1], p1[f][k]);
    }
  }
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int f = 0; f < FR; ++f) xw[(f * K + k) * 32] = p0[f][k] + p1[f][k];
}

// One lean step with one frame per lane (frame 32 j + lane of the stage): the odd tail step of a short last chunk.
template <int D, int K, typename CT, int MODEL, bool NAMED = false, typename SMT>
__device__ __forceinline__ void lean_step(SMT& sm, int cb, int g, int st, int j, int lane, int& buf, double eps,
                                          double (&acc)[K * GroupDims<D>::NSG], double (&sg)[K]) {
  using G = GroupDims<D>;
  constexpr int NSG = G::NSG, M = G::M;
  double psi[1][NSG];
  lean_partial_forms<D, K, 1, CT>(&sm.zbuf[st][2 * g][0] + lane + 32 * j, &sm.coef[cb][0][g * NSG],
                                  &sm.xq[buf][g][0][lane], psi);
  em_exchange_barrier<D, NAMED>();
  const double* __restrict__ xr = &sm.xq[buf][0][0][lane];
  double q[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double v = xr[k * 32];
#pragma unroll
    for (int gg = 1; gg < M; ++gg) v += xr[(gg * 2 * K + k) * 32];
    q[k] = fabs(v);
  }
  buf ^= 1;
  double gam[K], cw[K];
  if constexpr (MODEL == 1) softmax_watson<K>(q, sm.ew[cb], sm.ld, sm.w, gam, cw);
  else softmax_product<D, K>(q, sm.ew[cb], eps, gam, cw);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    sg[k] += gam[k];
#pragma unroll
    for (int i = 0; i < NSG; ++i) acc[k * NSG + i] = fma(cw[k], psi[0][i], acc[k * NSG + i]);
  }
}

// The lean step loop with TWO frames per lane and step (frames t and t + 32):
// the coefficient loads, the barrier and the loop overhead are shared by the two
// frames, and their E-step / softmax dependency chains interleave, which is what
// keeps the fp64 pipe busy with only two warps per scheduler.
template <int D, int K, typename CT, int MODEL, bool NAMED = false, typename SMT>
__device__ __forceinline__ void lean_chunk2(SMT& sm, int cb, int g, int st, int nsteps2, int lane,
                                            int& buf, double eps, double (&acc)[K * GroupDims<D>::NSG],
                                            double (&sg)[K]) {
  using G = GroupDims<D>;
  constexpr int NSG = G::NSG, M = G::M;
  const CT* __restrict__ zrow = &sm.zbuf[st][2 * g][0] + lane;
  const double* __restrict__ cg = &sm.coef[cb][0][g * NSG];
#pragma unroll 1
  for (int j = 0; j < nsteps2; ++j, zrow += 64) {
    double psi[2][NSG];
    lean_partial_forms<D, K, 2, CT>(zrow, cg, &sm.xq[buf][g][0][lane], psi);
    em_exchange_barrier<D, NAMED>();
    const double* __restrict__ xr = &sm.xq[buf][0][0][lane];
    double qA[K], qB[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double va = xr[k * 32], vb = xr[(K + k) * 32];
#pragma unroll
      for (int gg = 1; gg < M; ++gg) {
        va += xr[(gg * 2 * K + k) * 32];
        vb += xr[(gg * 2 * K + K + k) * 32];
      }
      qA[k] = fabs(va);
      qB[k] = fabs(vb);
    }
    buf ^= 1;
    double gA[K], cA[K], gB[K], cB[K];
    if constexpr (MODEL == 1) {
      softmax_watson<K>(qA, sm.ew[cb], sm.ld, sm.w, gA, cA);
      softmax_watson<K>(qB, sm.ew[cb], sm.ld, sm.w, gB, cB);
    } else {
      softmax_product<D, K>(qA, sm.ew[cb], eps, gA, cA);
      softmax_product<D, K>(qB, sm.ew[cb], eps, gB, cB);
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
      sg[k] += gA[k] + gB[k];
#pragma unroll
      for (int i = 0; i < NSG; ++i) {
        acc[k * NSG + i] = fma(cA[k], psi[0][i], acc[k * NSG + i]);
        acc[k * NSG + i] = fma(cB[k], psi[1][i], acc[k * NSG + i]);
      }
    }
  }
}

// lean_chunk2 with the posterior computed ONCE per frame instead of once per slot group
// (warp-specialised kernel only).  After the exchange of the partial quadratic forms, warp g
// evaluates the softmax for frames 16g .. 16g+15 of the step's 64 (lanes 16-31 mirror lanes
// 0-15), publishes gamma / q per (class, frame) and a second barrier hands it to all groups.
// Saves (M - 1) / M of the softmax instructions and half of the partial-sum adds for one more
// barrier per step.  sg then holds the sum of gamma over the frames THIS WARP evaluated; the
// caller adds the groups' sums.
template <int D, int K, typename CT, typename SMT>
__device__ __forceinline__ void lean_chunk2_split(SMT& sm, int cb, int g, int st, int nsteps2, int lane, double eps,
                                                  double (&acc)[K * GroupDims<D>::NSG], double (&sg)[K]) {
  using G = GroupDims<D>;
  constexpr int NSG = G::NSG, M = G::M;
  static_assert(M == 4, "frame split assumes four slot-group warps");
  const CT* __restrict__ zrow = &sm.zbuf[st][2 * g][0] + lane;
  const double* __restrict__ cg = &sm.coef[cb][0][g * NSG];
  const int fsel = 16 * g + (lane & 15);         // frame of the step this lane evaluates
  const int fhalf = fsel >> 5, fl = fsel & 31;   // its half (A / B) and lane
#pragma unroll 1
  for (int j = 0; j < nsteps2; ++j, zrow += 64) {
    double psi[2][NSG];
    lean_partial_forms<D, K, 2, CT>(zrow, cg, &sm.xq[0][g][0][lane], psi);
    em_exchange_barrier<D, true>();
    {
      const double* __restrict__ xr = &sm.xq[0][0][fhalf * K][fl];
      double q[K];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        double v = xr[k * 32];
#pragma unroll
        for (int gg = 1; gg < M; ++gg) v += xr[(gg * 2 * K + k) * 32];
        q[k] = fabs(v);
      }
      double gm[K], cw[K];
      softmax_product<D, K>(q, sm.ew[cb], eps, gm, cw);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        sg[k] += lane < 16 ? gm[k] : 0.0;
        sm.cwx[k][fsel] = cw[k];
      }
    }
    em_exchange_barrier<D, true>();
    double cA[K], cB[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      cA[k] = sm.cwx[k][lane];
      cB[k] = sm.cwx[k][32 + lane];
    }
    // A DFMA reading three different registers issues every 3 cycles, one that finds an operand in the reuse cache
    // every 2 (scripts/microbench/fp64_operands.cu): runs of NSG instructions share gamma / q of one (class, frame)
#pragma unroll
    for (int k = 0; k < K; ++k) {
#pragma unroll
      for (int i = 0; i < NSG; ++i) acc[k * NSG + i] = fma(cA[k], psi[0][i], acc[k * NSG + i]);
#pragma unroll
      for (int i = 0; i < NSG; ++i) acc[k * NSG + i] = fma(cB[k], psi[1][i], acc[k * NSG + i]);
    }
  }
}

// General posterior (log domain or qmin-ratio form) with the reference's floors.
template <int D, int K>
__device__ __forceinline__ void softmax_general(const double (&q)[K], const double* __restrict__ ld,
                                                const double* __restrict__ w, const double* __restrict__ ew,
                                                bool fast, double eps, double (&gam)[K], double (&invq)[K]) {
  double a[K];
  if (fast) {
    double qmin = q[0];
#pragma unroll
    for (int k = 1; k < K; ++k) qmin = fmin(qmin, q[k]);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      invq[k] = fast_rcp(q[k]);
      a[k] = ew[k] * ipow<D>(qmin * invq[k]);
    }
  } else {
    double lp[K];
    double m = -INFINITY;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      lp[k] = -(double)D * log(q[k]) - ld[k];
      m = fmax(m, lp[k]);
      invq[k] = 1.0 / q[k];
    }
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] = exp(lp[k] - m) * w[k];
  }
  double den = a[0];
#pragma unroll
  for (int k = 1; k < K; ++k) den += a[k];
  const double inv = 1.0 / fmax(den, kTiny);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double g = a[k] * inv;
    if (eps != 0.0) g = fmin(fmax(g, eps), 1.0 - eps);
    gam[k] = g;
  }
}

// General step (runtime group index): M-step-only iteration 0, and the FULL
// variant (saliency, source activity mask, log-domain softmax).  Frames are
// masked individually.
template <int D, int K, typename CT, bool FULL, bool NAMED = false, typename SMT>
__device__ __forceinline__ void general_chunk(const PersistArgs& a, SMT& sm, int g, int bin,
                                              int st, int t_chunk, int nsteps, int lane, int& buf, bool mstep_only,
                                              bool fast, double (&acc)[K * GroupDims<D>::NSG], double (&sg)[K]) {
  using G = GroupDims<D>;
  constexpr int NSG = G::NSG, NLOC = G::NLOC, M = G::M, NS = G::NS;
  const int T = a.T;
  const CT* __restrict__ zb = &sm.zbuf[st][0][0];
  const CT* __restrict__ zg = zb + 2 * g * kStageFrames + lane;
#pragma unroll 1
  for (int j = 0; j < nsteps; ++j) {
    const int t = t_chunk + j * 32 + lane;
    const bool valid = t < T;
    const int tc = valid ? t : 0;
    double2 x[NLOC];
#pragma unroll
    for (int l = 0; l < NLOC; ++l) x[l] = lds_cplx(zg + l * kStageFrames + j * 32);
    double psi[NSG];
    group_psi<D>(x, psi);
    double gam[K], invq[K];
    bool done = false;
    if constexpr (FULL) {
      if (!mstep_only) {
        const double* __restrict__ cg = &sm.coef[0][0][g * NSG];
#pragma unroll
        for (int k = 0; k < K; ++k) {
          double pq = 0.0;
#pragma unroll
          for (int i = 0; i < NSG; ++i) pq = fma(cg[k * NS + i], psi[i], pq);
          sm.xq[buf][g][k][lane] = pq;
        }
        em_exchange_barrier<D, NAMED>();
        double q[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
          double v = sm.xq[buf][0][k][lane];
#pragma unroll
          for (int gg = 1; gg < M; ++gg) v += sm.xq[buf][gg][k][lane];
          q[k] = fmax(fabs(v), 10.0 * kTiny);
        }
        buf ^= 1;
        if (a.activity != nullptr) {
          // masked classes get zero posterior mass (mixture_model_utils.py:39-41)
          double ewm[K], wm[K];
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const bool on = a.activity[((size_t)bin * K + k) * T + tc] != 0;
            ewm[k] = on ? sm.ew[0][k] : 0.0;
            wm[k] = on ? sm.w[k] : 0.0;
          }
          softmax_general<D, K>(q, sm.ld, wm, ewm, fast, a.aff_eps, gam, invq);
        } else {
          softmax_general<D, K>(q, sm.ld, sm.w, sm.ew[0], fast, a.aff_eps, gam, invq);
        }
        done = true;
      }
    }
    if (!done) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        gam[k] = __ldcg(a.aff_in + ((size_t)bin * K + k) * T + tc);  // L2: may just have been streamed in
        invq[k] = 1.0;
      }
    }
    double sal = 1.0;
    if (FULL && a.saliency != nullptr) sal = a.saliency[(size_t)bin * T + tc];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double gs = valid ? gam[k] * sal : 0.0;
      const double cw = gs * invq[k];
      sg[k] += gs;
#pragma unroll
      for (int i = 0; i < NSG; ++i) acc[k * NSG + i] = fma(cw, psi[i], acc[k * NSG + i]);
    }
  }
}

// In-place inverse of a Hermitian positive definite D x D matrix in shared
// memory by Gauss-Jordan elimination without pivoting (one warp; every lane
// keeps its own entries in registers and only fetches the pivot row / column).
// Returns det(A) as the product of the pivots (the caller takes one log);
// *ok is false if a pivot is not positive / finite.
template <int D>
__device__ __forceinline__ double warp_hpd_inverse(double2* __restrict__ A, int lane, bool* ok) {
  constexpr int NS = D * D;
  constexpr int PER = (NS + 31) / 32;
  int ri[PER], ci[PER];
  double2 mine[PER];
#pragma unroll
  for (int r = 0; r < PER; ++r) {
    const int idx = lane + 32 * r;
    ri[r] = idx / D;
    ci[r] = idx - ri[r] * D;
    mine[r] = idx < NS ? A[idx] : make_double2(0.0, 0.0);
  }
  double det = 1.0;
  bool good = true;
#pragma unroll 1
  for (int j = 0; j < D; ++j) {
    const double p = A[j * D + j].x;
    good = good && (p > 0.0) && (p < 1e300);
    const double ip = fast_rcp(p);
    det *= p;
#pragma unroll
    for (int r = 0; r < PER; ++r) {
      if (lane + 32 * r < NS) {
        const int i = ri[r], k = ci[r];
        const double2 aij = A[i * D + j], ajk = A[j * D + k];
        const double sx = aij.x * ip, sy = aij.y * ip;  // a_ij / p
        // general entry: a_ik - a_ij a_jk / p
        double2 v = make_double2(mine[r].x - (sx * ajk.x - sy * ajk.y), mine[r].y - (sx * ajk.y + sy * ajk.x));
        if (k == j) v = make_double2(-sx, -sy);
        if (i == j) v = make_double2(ajk.x * ip, ajk.y * ip);
        if (i == j && k == j) v = make_double2(ip, 0.0);
        mine[r] = v;
      }
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < PER; ++r)
      if (lane + 32 * r < NS) A[lane + 32 * r] = mine[r];
    __syncwarp();
  }
  *ok = good;
  return det;
}

// Model update of one (bin, class) by one warp (cACGMM): scatter sums Sk[0..NS) + sum of gamma
// Sk[NS] -> E-step coefficients in a.coef (+ the published scalars), see the file header.
// A, V: D x D shared-memory scratch of the warp; lamk: D doubles.
template <int D, bool FULL>
__device__ __forceinline__ void cacg_update_class(const PersistArgs& a, int bin, int k, int K, int lane,
                                                  double2* __restrict__ A, double2* __restrict__ V,
                                                  double* __restrict__ lamk, const double* __restrict__ Sk,
                                                  const int* __restrict__ tab, double* __restrict__ ld_out,
                                                  double* __restrict__ coef_out = nullptr) {
  // coef_out: destination of the class's NS slot coefficients instead of a.coef (em_sticky.cuh: shared memory)
  constexpr int NS = D * D;
  double* Ad = reinterpret_cast<double*>(A);
    // L2 round trip issued first, consumed after the inversion
    const int dead_bin = a.dead == nullptr ? 0 : __ldcg(a.dead + bin);
#ifdef PBB_PHASE_TIMING
    long long _tu = clock64();
#define PBB_PHU(i) do { if (k == 0 && lane == 0) { long long _t = clock64(); atomicAdd(&a.phase[i], (unsigned long long)(_t - _tu)); _tu = _t; } } while (0)
#else
#define PBB_PHU(i) do { } while (0)
#endif
    const double scale = (double)D / fmax(Sk[NS], kTiny);
    bool bad = false;
    auto build_scaled = [&](double f) {
      for (int s = lane; s < NS; s += 32) {
        const int pk = tab[s];
        const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
        const double v = Sk[s] * f;
        bad |= !isfinite(v);
        if (kind == 0) { Ad[2 * (d * D + d)] = v; Ad[2 * (d * D + d) + 1] = 0.0; }
        else if (kind == 1) { Ad[2 * (d * D + e)] = v; Ad[2 * (e * D + d)] = v; }
        else { Ad[2 * (d * D + e) + 1] = -v; Ad[2 * (e * D + d) + 1] = v; }
      }
      __syncwarp();
    };
    auto build = [&]() { build_scaled(scale); };
    // Trace-normalise to tr = D (keeps all classes on a comparable scale): the factor D / tr(S) is applied
    // while the matrix is built (the 1 / sum(gamma) scale cancels), the diagonal slots are read directly.
    // covariance_norm=False keeps the reference's absolute scale (it survives into the returned
    // eigenvalues).
    double tr, tn;
    if (a.covariance_norm == PBB_NORM_NONE) {
      build();
      tr = 0.0;
      for (int d = lane; d < D; d += 32) tr += A[d * D + d].x;
      tr = warp_sum(tr);
      tn = 1.0;
    } else {
      double trs = 0.0;
#pragma unroll
      for (int d = 0; d < D; ++d) trs += Sk[(d >> 1) * (NS / (D / 2)) + (d & 1)];  // |z_d|^2 slots (common.cuh)
      tr = trs * scale;
      tn = (double)D / fmax(tr, kTiny);
      build_scaled(scale * tn);
    }
    PBB_PHU(8);   // build + trace + scale
    bool ok;
    const double det = warp_hpd_inverse<D>(A, lane, &ok);
    PBB_PHU(9);   // Gauss-Jordan
    double ldk = log(det);
    double tinv = 0.0;
    bool diag_pos = true;
#pragma unroll
    for (int d = 0; d < D; ++d) {  // every lane reads the diagonal (broadcast loads)
      tinv += A[d * D + d].x;
      diag_pos = diag_pos && A[d * D + d].x > 0.0;
    }
    // lambda_min / lambda_max >= 1 / (tr(A) tr(A^-1)) holds for a positive definite A only.  Positive pivots do not
    // prove that in floating point: a singular scatter matrix (rank-deficient observations) can pass Gauss-Jordan
    // with noise-level positive pivots and come out with a negative diagonal in its "inverse", which made the bound
    // negative and skipped the floor.  Every diagonal entry of the inverse of a positive definite matrix is positive.
    // A bin with an all-zero frame must keep the reference's own normalisation: such a frame has
    // q = `tiny` for every class whatever the scale of B (cacg.py:198), so its posterior depends
    // on det B in the reference's lambda_max = 1 scale -- take the eigendecomposition path there.
    const bool no_floor = ok && diag_pos && isfinite(tinv) && (tr * tn * tinv * a.eigenvalue_floor < 0.5) &&
                          dead_bin == 0;
    double* __restrict__ co = coef_out != nullptr ? coef_out : a.coef + ((size_t)bin * K + k) * NS;
    PBB_PHU(10);  // log det, trace of the inverse, floor test
    if (__any_sync(0xffffffffu, bad)) {
      if (lane == 0) atomicMax(a.status, bin + 1);
    }
    if (no_floor) {
      for (int s = lane; s < NS; s += 32) {
        const int pk = tab[s];
        const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
        const double2 u = A[d * D + e], v = A[e * D + d];
        co[s] = kind == 0 ? u.x : (kind == 1 ? (u.x + v.x) : -(u.y - v.y));
      }
    } else {
      // reference semantics: eigendecomposition, normalise, floor (cacg.py:95-126)
      build();
      if (a.covariance_norm == PBB_NORM_TRACE) {
        for (int i = lane; i < NS; i += 32) { A[i].x *= tn / D; A[i].y *= tn / D; }
        __syncwarp();
      }
      warp_jacobi_small<D>(A, V, lane);
      double lmax = -INFINITY;
      for (int d = lane; d < D; d += 32) lmax = fmax(lmax, A[d * D + d].x);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lmax = fmax(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
      for (int d = lane; d < D; d += 32) {
        double l = A[d * D + d].x;
        if (a.covariance_norm == PBB_NORM_EIGENVALUE) l = fmax(l / fmax(lmax, kTiny), a.eigenvalue_floor);
        else l = fmax(l, lmax * a.eigenvalue_floor);
        if (!isfinite(l)) atomicMax(a.status, bin + 1);
        lamk[d] = l;
      }
      __syncwarp();
      ldk = model_from_eig_warp(V, lamk, tab, D, lane, co);
    }
    if (lane == 0) {
      *ld_out = ldk;
      if (!FULL) {
        a.ld[(size_t)bin * 4 + k] = ldk;
        a.ew[(size_t)bin * 4 + k] = Sk[NS];
      }
    }
    PBB_PHU(11);  // coefficient stores
}

// E-step weight of class k of the lean model from its published form (cacg_update_class: a.ew holds sum gamma_k and
// a.ld log det_k, stride 4): ew_k = w_k exp(ld_min - ld_k), w_k = 1 / K or sum gamma_k / T.  ld[0 .. K) are the
// classes' log dets (ldk = ld[k]); fmin is exact, so the minimum does not depend on the class it starts from.
template <int K>
__device__ __forceinline__ double lean_ew(double sgam, double ldk, const double* ld, int weight_mode, int T) {
  double ldmin = ld[0];
#pragma unroll
  for (int j = 1; j < K; ++j) ldmin = fmin(ldmin, ld[j]);
  const double wk = weight_mode == PBB_WEIGHT_CONST ? 1.0 / K : sgam / (double)T;
  return wk * exp(ldmin - ldk);
}

// Posterior of a padded frame (z = 0) under the staged model: the lean sweeps count the zs - T padded frames of the
// last ring stage like observations, and the caller subtracts this from the lanes that counted them.
template <int D, int K, int MODEL, typename SMT>
__device__ __forceinline__ void padded_gamma(const SMT& sm, int cb, double eps, double (&gp)[K]) {
  double q[K], cw[K];
#pragma unroll
  for (int k = 0; k < K; ++k) q[k] = 0.0;
  if constexpr (MODEL == 1) softmax_watson<K>(q, sm.ew[cb], sm.ld, sm.w, gp, cw);
  else softmax_product<D, K>(q, sm.ew[cb], eps, gp, cw);
}

// End of a sweep, after warp_reduce_halving of acc (the 32 frames of warp g reduced): the lanes store the group's
// slots [g NSG, (g + 1) NSG) into the scatter-sum rows S[k].  The callers then add up the warp's sum of gamma, each
// into its own destination.
template <int D, int K>
__device__ __forceinline__ void store_group_sums(const double (&acc)[K * GroupDims<D>::NSG], int g, int lane,
                                                 double (*S)[D * D + 1]) {
  constexpr int NSG = GroupDims<D>::NSG;
  int lo, hi;
  reduce_range<K * NSG>(lane, lo, hi);
#pragma unroll
  for (int j = 0; j < HalvingSizes<K * NSG>::n5; ++j) {
    const int idx = lo + j;
    if (idx < hi) {
      const int k = idx / NSG, i = idx - k * NSG;
      S[k][g * NSG + i] = acc[j];
    }
  }
}

// Frame split (PersistArgs::tsplit = S > 1): every part of (bin, it) leaves its scatter sums in a.tpart[bin][part] and
// counts itself here (one thread); true for the part that arrives last, which then adds the S parts.
__device__ __forceinline__ bool split_last_part(const PersistArgs& a, int bin, int it, int S) {
  const int old = atomicAdd(a.tcount + bin, 1);
  __threadfence();
  return old + 1 == (it + 1) * S;
}
// Element i of the bin's scatter sums (row of K (NS + 1)): the parts added in the order p = 0 .. S-1, so that the
// result does not depend on which CTA delivers the last part.
template <int D, int K>
__device__ __forceinline__ double split_sum(const PersistArgs& a, int bin, int S, int i) {
  constexpr int kRow = K * (D * D + 1);
  const double* __restrict__ tb = a.tpart + (size_t)bin * S * kRow;
  double v = __ldcg(tb + i);
  for (int q = 1; q < S; ++q) v += __ldcg(tb + (size_t)q * kRow + i);
  return v;
}

// Threads of a CTA: the D / 2 slot-group warps and, when there are more classes than those, one "update only" warp
// per class beyond them (D = 6, K = 4: the fourth class had to wait for a whole class update of warp 0, a quarter of
// the complex Watson chain).  The extra warps follow the control flow, take every CTA-wide barrier, skip the E / M
// arithmetic (the slot-group warps then exchange on named barrier 1) and update class g in the update phase.
__host__ __device__ constexpr int persist_extra_warps(int D, int K) { return K > D / 2 ? K - D / 2 : 0; }
__host__ __device__ constexpr int persist_threads(int D, int K) { return 32 * (D / 2 + persist_extra_warps(D, K)); }
// CTAs per SM of em_persistent_kernel (full variant: one frame per lane; lean: two), which the host's frame split
// plans with; em_ws_kernel runs the lean D = 8 figure as well
__host__ __device__ constexpr int persist_ctas_per_sm(int D, bool full) {
  return full ? (D == 8 ? 3 : (D == 6 ? 4 : 6)) : (D == 4 ? 4 : 2);
}

template <int D, int K, typename CT, bool FULL, int MODEL = 0>
__global__ void __launch_bounds__(persist_threads(D, K), persist_ctas_per_sm(D, FULL))
em_persistent_kernel(const PersistArgs a) {
  using SM = PersistSmem<D, K, CT>;
  using G = GroupDims<D>;
  constexpr int NS = D * D, M = D / 2, NSG = G::NSG;
  constexpr int XW = persist_extra_warps(D, K);
  constexpr bool NAMED = XW > 0;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SM& sm = *reinterpret_cast<SM*>(smem_raw);
  const int tid = threadIdx.x, g = tid >> 5, lane = tid & 31;
  const int F = a.F, T = a.T, zs = a.zs;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  // Frame split (see em_ws.cuh): S consecutive tickets per (bin, iteration), part p sweeps the ring stages
  // [p * nchunks / S, (p + 1) * nchunks / S); the part that arrives last adds the partial sums and updates the model.
  const int S = a.tsplit > 1 ? a.tsplit : 1;
  const int total = a.iterations * F * S;
  const CT* __restrict__ zbase = reinterpret_cast<const CT*>(a.z);

  for (int s = tid; s < NS; s += blockDim.x) sm.tab[s] = slot_pack(D, s);
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(&sm.full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    sm.tick[0] = atomicAdd(a.ticket, 1);
  }
  __syncthreads();
  int cur = sm.tick[0];
  int bin = 0, it = 0, part = 0;
  if (cur < total) decode_task(a, cur, S, order_entry(a, cur, S), bin, it, part);
  unsigned chunk_cnt = 0;  // chunks consumed so far by this CTA (ring position)

  // 1-D TMA bulk copies per ring stage (stage_g2s), issued by a single elected lane.
  auto issue_chunk = [&](int bin, int c, unsigned n) {  // warp 0
    if (lane == 0) {
      const int st = n & 1u;
      stage_g2s<D>(sm.zbuf[st], zbase, bin, nchunks, c, &sm.full[st]);
    }
  };
  // streamed upload: a bin's observation may not have arrived yet; its first task issues its own
  // first chunk after the arrival flag instead of having it prefetched
  if (g == 0 && cur < total && !(a.wait_load && it == 0)) issue_chunk(bin, part * nchunks / S, 0);

#ifdef PBB_PHASE_TIMING
  long long _tp = clock64();
#endif
  // lean variant: the model of a task can be prefetched (cp.async, L2 -> smem) during the previous
  // task's last chunk; cb = buffer holding the current task's model, pf = it is already there
  int cb = 0;
  bool pf = false;
  while (cur < total) {
    const bool mstep_only = a.first_is_m && it == 0;
    const bool last_it = it == a.iterations - 1;
    const int c0 = part * nchunks / S, c1 = (part + 1) * nchunks / S, ncp = c1 - c0;  // this task's ring stages
    int tnext = 0, nbin = 0, nit = 0, npart = 0;  // the task after this one (thread 0; decoded a chunk later)
    int oraw = 0;                      // its entry of the explicit order table, in flight
    if (tid == 0) tnext = atomicAdd(a.ticket, 1);
    if (a.wait_load && it == 0) {
      if (tid == 0) {
        while (ld_acquire_gpu(a.flags + bin) < 0) __nanosleep(200);
      }
      __syncthreads();
      if (g == 0) {
        // the staged rows were written with ordinary stores by another CTA: order them before
        // this CTA's async-proxy (TMA) read
        asm volatile("fence.proxy.async;" ::: "memory");
        issue_chunk(bin, c0, chunk_cnt);
      }
    }
    if (!mstep_only && !pf) {
      if (tid == 0) {
        while (ld_acquire_gpu(a.flags + bin) < it) __nanosleep(40);
      }
      __syncthreads();
      PBB_PH(0);  // flag wait
      const double* __restrict__ cf = a.coef + (size_t)bin * K * NS;
      for (int i = tid; i < K * NS; i += blockDim.x) (&sm.coef[cb][0][0])[i] = __ldcg(cf + i);
      if (FULL) {
        if (tid < K) {
          sm.ew[cb][tid] = __ldcg(a.ew + (size_t)bin * K + tid);
          sm.ld[tid] = __ldcg(a.ld + (size_t)bin * K + tid);
          sm.w[tid] = __ldcg(a.w + (size_t)bin * K + tid);
        }
      } else if (MODEL == 1) {
        if (tid < K) {
          sm.ew[cb][tid] = __ldcg(a.ew + (size_t)bin * 4 + tid);  // kappa
          sm.ld[tid] = __ldcg(a.ld + (size_t)bin * 4 + tid);      // log norm
          sm.w[tid] = __ldcg(a.w + (size_t)bin * K + tid);
        }
      } else if (tid < 8) {
        sm.raw[cb][tid] = __ldcg((tid < 4 ? a.ew : a.ld) + (size_t)bin * 4 + (tid & 3));
      }
    } else if (pf) {
      asm volatile("cp.async.wait_all;" ::: "memory");
    }
    if (!FULL && MODEL == 0 && !mstep_only && tid < 32) {
      // weights and ew from the published raw scalars (sum of gamma, log det): all of it lives in warp 0
      __syncwarp();
      if (tid < K) sm.ew[cb][tid] = lean_ew<K>(sm.raw[cb][tid], sm.raw[cb][4 + tid], &sm.raw[cb][4], a.weight_mode, T);
    }
    const bool fast = FULL ? (a.softmax_fast && !(a.user_model && it == 0)) : true;
    const bool lean = !FULL && !mstep_only;

    double acc[K * NSG];
#pragma unroll
    for (int i = 0; i < K * NSG; ++i) acc[i] = 0.0;
    double sg[K];
#pragma unroll
    for (int k = 0; k < K; ++k) sg[k] = 0.0;
    int buf = 0;
    bool pf_next = false;
    int probe = -1;

    __syncthreads();  // model staged
    PBB_PH(7);  // task start -> model staged
#pragma unroll 1
    for (int c = c0; c < c1; ++c) {
      // The stage refilled below was last read in the previous chunk.  In the E+M loops every
      // observation load of a step precedes that step's exchange barrier, so once warp 0 is
      // here all warps are done with it; only the M-step-only loop (no exchange) needs a barrier.
      if (!lean) __syncthreads();
      const bool last_chunk = c + 1 == c1;
      // Thread 0 walks the next ticket through three chunk tops so that neither the ticket atomic
      // nor the flag probe (L2 round trips) is waited for: consume the ticket and issue the probe at
      // chunk n-3, publish both to shared memory at chunk n-2, everybody reads them at chunk n-1.
      if (tid == 0) {
        const int c_probe = ncp >= 3 ? c1 - 3 : -1;
        const int c_pub = ncp >= 2 ? c1 - 2 : c0;
        const int c_first = c_probe >= 0 ? c_probe : c_pub;
        // explicit order: ticket (atomic, task start) -> table entry (issued at c_first) -> decoded at c_pub; no flag
        // probe / model prefetch in this mode
        if (a.order != nullptr) {
          if (c == c_first && tnext < total) oraw = __ldcg(a.order + tnext / S);
          if (c == c_pub) { nbin = oraw & 0xffff; nit = oraw >> 16; npart = tnext % S; }
        } else if (c == c_first && tnext < total) {
          const int tt = tnext / S;
          npart = tnext - tt * S;
          decode_ticket(tt, F, a.iterations, a.wave_c, nbin, nit);
        }
        if (c == c_probe && !FULL && tnext < total && a.order == nullptr) {
          probe = (a.first_is_m && nit == 0) ? -1 : ld_acquire_gpu(a.flags + nbin) - nit;  // >= 0: published
        }
        if (c == c_pub) {
          sm.tick[1] = tnext;
          sm.tick[2] = nbin;
          sm.tick[3] = nit;
          sm.tick[4] = npart;
          // (no model prefetch with update-only warps: they do not take the exchange barriers that order this
          // store before the read at the next chunk top)
          sm.ready = (!FULL && MODEL == 0 && XW == 0 && ncp >= 3 && tnext < total && probe >= 0) ? 1 : 0;
        }
      }
      if (g == 0) {
        if (!last_chunk) {
          issue_chunk(bin, c + 1, chunk_cnt + 1);
        } else {
          const int nx = __shfl_sync(0xffffffffu, tnext, 0);
          const int nxb = __shfl_sync(0xffffffffu, nbin, 0), nxi = __shfl_sync(0xffffffffu, nit, 0);
          const int nxp = __shfl_sync(0xffffffffu, npart, 0);
          if (nx < total && !(a.wait_load && nxi == 0)) issue_chunk(nxb, nxp * nchunks / S, chunk_cnt + 1);
        }
      }
      if (!FULL && XW == 0 && lean && last_chunk && ncp >= 3 && sm.ready) {
        // prefetch the next task's model into the other buffer (16-byte L2 -> smem copies)
        pf_next = true;
        const int nb = sm.tick[2];
        const char* __restrict__ src = reinterpret_cast<const char*>(a.coef + (size_t)nb * K * NS);
        char* dst = reinterpret_cast<char*>(&sm.coef[cb ^ 1][0][0]);
        for (int i = tid; i < K * NS / 2; i += blockDim.x)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst + 16 * i)), "l"(src + 16 * i)
                       : "memory");
        if (tid < 4)  // (sum gamma)[4] from a.ew, (ld)[4] from a.ld, two 16-byte pieces each
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(
                           reinterpret_cast<char*>(&sm.raw[cb ^ 1][0]) + 16 * tid)),
                       "l"(reinterpret_cast<const char*>((tid < 2 ? a.ew : a.ld) + (size_t)nb * 4) + 16 * (tid & 1))
                       : "memory");
      }
      const int st = chunk_cnt & 1u;
      PBB_PH(1);  // staging / chunk top
      if (XW > 0 && g >= M) {  // update-only warp: nothing to do until the sums are complete
        ++chunk_cnt;
        continue;
      }
      mbar_wait(&sm.full[st], (chunk_cnt >> 1) & 1u);
      PBB_PH(2);  // TMA wait
      ++chunk_cnt;
      const int t_chunk = c * kStageFrames;
      const int nsteps = (min(kStageFrames, zs - t_chunk)) >> 5;
      if (lean) {
        lean_chunk2<D, K, CT, MODEL, NAMED>(sm, cb, g, st, nsteps >> 1, lane, buf, a.aff_eps, acc, sg);
        if (nsteps & 1) {  // odd tail step of a short last chunk
          lean_step<D, K, CT, MODEL, NAMED>(sm, cb, g, st, nsteps - 1, lane, buf, a.aff_eps, acc, sg);
        }
      }
      else general_chunk<D, K, CT, FULL, NAMED>(a, sm, g, bin, st, t_chunk, nsteps, lane, buf, mstep_only, fast, acc, sg);
      PBB_PH(3);  // EM steps
    }
    if (lean && zs > T && c1 == nchunks) {
      // the zs - T padded frames of every row behaved like zero observations
      double gp[K];
      padded_gamma<D, K, MODEL>(sm, cb, a.aff_eps, gp);
      const int npad_lane = (lane >= 32 - (zs - T)) ? 1 : 0;  // zs - T < 32: last step's tail lanes
#pragma unroll
      for (int k = 0; k < K; ++k) sg[k] -= npad_lane ? gp[k] : 0.0;
    }

    warp_reduce_halving<K * NSG>(acc, lane);
    if (XW == 0 || g < M) store_group_sums<D, K>(acc, g, lane, sm.S);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double v = warp_sum(sg[k]);
      if (g == 0 && lane == 0) sm.S[k][NS] = v;
    }
    __syncthreads();
    PBB_PH(4);  // reduce

    bool deliver = true;  // this CTA holds the complete sums of the iteration
    if (S > 1) {
      constexpr int kRow = K * (NS + 1);
      double* __restrict__ tp = a.tpart + ((size_t)bin * S + part) * kRow;
      for (int i = tid; i < kRow; i += blockDim.x) __stcg(tp + i, (&sm.S[0][0])[i]);
      __threadfence();
      __syncthreads();
      if (tid == 0) sm.tick[5] = split_last_part(a, bin, it, S);
      __syncthreads();
      deliver = sm.tick[5] != 0;
      if (deliver) {
        for (int i = tid; i < kRow; i += blockDim.x) (&sm.S[0][0])[i] = split_sum<D, K>(a, bin, S, i);
        __syncthreads();
      }
    }

    if (!deliver) {
      // another CTA completes the iteration
    } else if (last_it) {
      // leave the raw sums for cacg_update_kernel (reference-exact eigendecomposition)
      double* __restrict__ po = a.part + (size_t)bin * K * (NS + 1);
      for (int i = tid; i < K * (NS + 1); i += blockDim.x) po[i] = (&sm.S[0][0])[i];
    } else {
      // ---- model update, one warp per class -----------------------------------------
      for (int k = g; k < K; k += M + XW) {
        double2* A = sm.A[k];
        double* Ad = reinterpret_cast<double*>(A);
        if constexpr (MODEL == 1) {
          // complex Watson: covariance = S / sum(gamma) (complex_watson.py:307-312), mode = eigenvector of
          // the largest eigenvalue (pb_bss/utils.py:154-163), concentration from the spline (:314)
          const double wscale = 1.0 / sm.S[k][NS];
          bool wbad = false;
          for (int s = lane; s < NS; s += 32) {
            const int pk = sm.tab[s];
            const int d = pk & 255, e = (pk >> 8) & 255, kind = pk >> 16;
            const double v = sm.S[k][s] * wscale;
            wbad |= !isfinite(v);
            if (kind == 0) { Ad[2 * (d * D + d)] = v; Ad[2 * (d * D + d) + 1] = 0.0; }
            else if (kind == 1) { Ad[2 * (d * D + e)] = v; Ad[2 * (e * D + d)] = v; }
            else { Ad[2 * (d * D + e) + 1] = -v; Ad[2 * (e * D + d) + 1] = v; }
          }
          __syncwarp();
          if (__any_sync(0xffffffffu, wbad) && lane == 0) atomicMax(a.status, bin + 1);
          double2* mloc = reinterpret_cast<double2*>(sm.rot[k]);  // ((D+1)/2)*6 doubles >= 2*D, 16-byte aligned
          double lmax;
          // only the largest eigenpair is needed: repeated squaring, exact Jacobi when the spectrum is too close
          if (!warp_top_eigenpair<D>(A, sm.V[k], sm.W[k], lane, &lmax, mloc)) {
            __syncwarp();
            warp_jacobi_small<D>(A, sm.V[k], lane);
            int best = 0;
            lmax = A[0].x;
#pragma unroll
            for (int d = 1; d < D; ++d) {
              const double l = A[d * D + d].x;
              if (l >= lmax) { lmax = l; best = d; }
            }
            __syncwarp();
            for (int d = lane; d < D; d += 32) mloc[d] = sm.V[k][d * D + best];
          }
          __syncwarp();
          cw_coef_from_mode(mloc, sm.tab, D, lane, a.coef + ((size_t)bin * K + k) * NS);
          if (lane == 0) {
            const double kappa = cw_spline_eval(a.spline, lmax);
            a.ew[(size_t)bin * 4 + k] = kappa;
            a.ld[(size_t)bin * 4 + k] = cw_log_norm(kappa, D);
          }
          continue;
        }
        cacg_update_class<D, FULL>(a, bin, k, K, lane, A, sm.V[k], sm.lam[k], sm.S[k], sm.tab, &sm.ld[k]);
      }
      __syncthreads();
      PBB_PH(5);  // update (Gauss-Jordan)
      // publish with a single cumulative gpu-scope release; the CTA barrier above ordered every
      // warp's model stores before it.  Lean variant: the class warps already stored the raw
      // scalars (sum of gamma, log det) and the consumer derives weights / ew itself.
      if (tid == 0) {
        if (MODEL == 1) {
          double n1 = 0.0;
          for (int j = 0; j < K; ++j) n1 += fabs(sm.S[j][NS]);
          for (int k = 0; k < K; ++k)
            a.w[(size_t)bin * K + k] =
                a.weight_mode == PBB_WEIGHT_CONST ? 1.0 / K : sm.S[k][NS] / (n1 == 0.0 ? 1e-10 : n1);
        } else if (FULL) {
          double ldmin = sm.ld[0];
          for (int j = 1; j < K; ++j) ldmin = fmin(ldmin, sm.ld[j]);
          double n1 = 0.0;
          for (int j = 0; j < K; ++j) n1 += fabs(sm.S[j][NS]);
          for (int k = 0; k < K; ++k) {
            double wk;
            if (a.weight_mode == PBB_WEIGHT_CONST) wk = 1.0 / K;
            else if (a.saliency == nullptr) wk = sm.S[k][NS] / (double)T;
            else wk = sm.S[k][NS] / (n1 == 0.0 ? 1e-10 : n1);
            a.w[(size_t)bin * K + k] = wk;
            a.ld[(size_t)bin * K + k] = sm.ld[k];
            a.ew[(size_t)bin * K + k] = wk * exp(ldmin - sm.ld[k]);
          }
        }
        st_release_gpu(a.flags + bin, it + 1);
      }
      PBB_PH(6);  // weights + publish
    }
    // all threads read the next ticket (published one chunk before the end of the pass)
    cur = sm.tick[1];
    bin = sm.tick[2];
    it = sm.tick[3];
    part = sm.tick[4];
    pf = pf_next;
    if (pf_next) cb ^= 1;
    // no barrier needed here: tick / ld / S are next written behind later barriers of the next task
  }
}


}  // namespace pbb
