// C-ABI entry points for the cACGMM EM path (see include/pbb.h).
#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstring>
#include <map>
#include <mutex>
#include <type_traits>
#include <vector>

#include <cuda.h>

#include "em_backward.cuh"
#include "em_kernels.cuh"
#include "em_persistent.cuh"
#include "em_ws.cuh"
#include "em_sticky.cuh"
#include "bingham.cuh"
#include "prof.cuh"

namespace pbb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  return (int)e;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// out[r] = sum_c in[r * n + c], fixed order
__global__ void sum_rows_kernel(const double* in, double* out, int rows, int n) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s = 0.0;
  for (int c = 0; c < n; ++c) s += in[(size_t)r * n + c];
  out[r] = s;
}

// ---- workspace carving -------------------------------------------------------
// Control block of the persistent fits, cleared by one memset (control_bytes) before the launch: flags (F) and the
// ticket, then, 8-byte aligned, the PBB_PHASE_TIMING cycle sums (kPhaseWords; the kernels write 0..11) and the
// two counters of the streamed upload's stream_load_kernel.
constexpr int kPhaseWords = 16;

struct CacgmmWorkspace {
  void* z;
  int zs;       // padded row stride of z (frames)
  int* flags;   // (F) per-bin model version, persistent kernel
  int* ticket;  // (1)
  unsigned long long* phase;  // (kPhaseWords) debug phase counters
  int* load_started;          // (1) stream_load_kernel CTAs running
  int* load_next_bin;         // (1) next bin a stream_load_kernel CTA takes
  size_t control_bytes;       // flags .. load_next_bin
  int* dead;    // (F) bins with an all-zero observation frame
  double* part;
  double* coef;
  double* ld;
  double* w;
  double* ew;
  double* loglik_part;
  double* aff_stage;  // (F, K, T) device copy of host-resident initial affiliations (streamed upload)
  int* tcount;        // (F) frame split of em_ws_kernel: parts delivered per bin
  size_t bytes;
};

static int max_chunks(int T) { return (T + 31) / 32; }
constexpr int kMaxOrder = 1 << 20;  // tasks (bins x iterations) an explicit task order may have

static CacgmmWorkspace carve(void* base, int F, int T, int D, int K) {
  CacgmmWorkspace ws;
  const size_t NS = (size_t)D * D;
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += align_up(n); return o; };
  const int zs = (T + 31) / 32 * 32;
  const size_t nchunks = ((size_t)zs + kStageFrames - 1) / kStageFrames;
  const size_t z_plain = (size_t)F * D * zs * sizeof(double2);
  const size_t z_staged = (size_t)F * nchunks * D * kStageFrames * sizeof(double2);
  const size_t o_phase = align_up((size_t)(F + 1) * sizeof(int), 8);
  ws.control_bytes = o_phase + kPhaseWords * sizeof(unsigned long long) + 2 * sizeof(int);
  const size_t o_z = take(z_plain > z_staged ? z_plain : z_staged);
  const size_t o_flags = take(ws.control_bytes);
  const size_t o_dead = take((size_t)F * sizeof(int));
  const size_t o_part = take((size_t)F * max_chunks(T) * K * (NS + 1) * sizeof(double));
  const size_t o_coef = take((size_t)F * K * NS * sizeof(double));
  const size_t o_ld = take((size_t)F * (K > 4 ? K : 4) * sizeof(double) + 64);  // lean kernel: stride 4
  const size_t o_w = take((size_t)F * K * sizeof(double));
  const size_t o_ew = take((size_t)F * (K > 4 ? K : 4) * sizeof(double) + 64);  // lean kernel: stride 4
  const size_t o_ll = take((size_t)F * max_chunks(T) * sizeof(double));
  const size_t o_aff = take((size_t)F * K * T * sizeof(double));
  const size_t o_tcount = take((size_t)F * sizeof(int));
  char* b = reinterpret_cast<char*>(base);
  ws.z = b + o_z;
  ws.zs = zs;
  ws.flags = reinterpret_cast<int*>(b + o_flags);
  ws.ticket = ws.flags + F;
  ws.phase = reinterpret_cast<unsigned long long*>(b + o_flags + o_phase);
  ws.load_started = reinterpret_cast<int*>(ws.phase + kPhaseWords);
  ws.load_next_bin = ws.load_started + 1;
  ws.dead = reinterpret_cast<int*>(b + o_dead);
  ws.part = reinterpret_cast<double*>(b + o_part);
  ws.coef = reinterpret_cast<double*>(b + o_coef);
  ws.ld = reinterpret_cast<double*>(b + o_ld);
  ws.w = reinterpret_cast<double*>(b + o_w);
  ws.ew = reinterpret_cast<double*>(b + o_ew);
  ws.loglik_part = reinterpret_cast<double*>(b + o_ll);
  ws.aff_stage = reinterpret_cast<double*>(b + o_aff);
  ws.tcount = reinterpret_cast<int*>(b + o_tcount);
  ws.bytes = off;
  return ws;
}

// Frame split of the persistent kernels (em_ws.cuh, em_persistent.cuh): with fewer bins than CTA slots the fit is
// bound by the per-bin dependency chain (E / M sweep -> update -> publish -> next sweep), so the sweep of one bin is
// spread over S CTAs.  The partial sums live behind the final iteration's block of ws.part (the multi-kernel path
// uses max_chunks(T) blocks there).
// Parts a bin-iteration is split into (pure host logic, unit-tested through pbb_em_dispatch); the result always
// satisfies 1 <= S <= nchunks and S + 1 <= max_chunks(T).
static int choose_frame_split(int F, int T, int D, int K, int ctas_per_sm, int sms) {
  const int zs = (T + 31) / 32 * 32;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  const long long slots = (long long)ctas_per_sm * sms;
  int S = 1;
  // a part must keep enough of the sweep to pay for the extra L2 round trip (partials out, counter, partials in,
  // ~3 us): measured break-even around T D^2 (K + 1) / S ~ 2.4e4 (C1, D = 4, T = 200 loses 10 % with S = 2;
  // D = 8, T = 500 gains 12 % with S = 4)
  const long long sweep = (long long)T * D * D * (K + 1);
  while (S < 4 && 2 * S <= nchunks && (long long)F * 2 * S <= slots && sweep >= 24000LL * 2 * S) S *= 2;
  if (S > nchunks) S = nchunks;
  if (S + 1 > max_chunks(T)) S = 1;
  return S < 1 ? 1 : S;
}
// Cluster size of the sticky-bins kernel (em_sticky.cuh), 0 = not applicable: the largest of 4, 2, 1 whose parts fit
// the ring (ceil(nchunks / S) <= kWsStages), that leaves every part a stage and whose F clusters run at once:
// F <= clusters[i] for S = 1 << i.  Clusters of 4 are placed within a GPC, so on an H100 (132 SMs in GPCs of uneven
// size) fewer of them fit than 2 x SMs / 4; a second wave would double the fit time.
static int choose_sticky(int F, int T, const int clusters[3]) {
  const int zs = (T + 31) / 32 * 32;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  for (int c = 4, i = 2; c >= 1; c /= 2, --i) {
    if (c > nchunks || (nchunks + c - 1) / c > kWsStages) continue;
    if (F > clusters[i]) continue;
    return c;
  }
  return 0;
}

// Persistent kernels of a fit, numbered as pbb_em_dispatch reports them (pbb.h).
enum { kKernelWs = 0, kKernelSticky = 1, kKernelSingle = 2 };

struct FitPlan {
  int kernel;  // kKernel*
  int split;   // sticky: CTAs per cluster; otherwise parts per bin-iteration (1 = no frame split)
};

// Models of the persistent fit: full = saliency / activity mask / log-domain softmax; lean = product-form softmax,
// 2 frames per lane; cw = complex Watson EM (lean structure, MODEL = 1, always the single-role kernel).
enum class Persist { kFull, kLean, kCw };

// The lean D = 8 fit runs em_ws_kernel, or the sticky-bins kernel for device-resident input.
static bool runs_ws(int D, Persist model) { return D == 8 && model == Persist::kLean; }
static bool sticky_eligible(int D, Persist model, bool streamed) { return runs_ws(D, model) && !streamed; }

// Which persistent kernel a fit runs and how it splits a bin-iteration (pure host logic).  sms: SMs of the device;
// clusters: sticky-kernel clusters of 1, 2, 4 CTAs the device runs at once, read only when sticky_eligible.
static FitPlan plan_persistent_fit(int F, int T, int D, int K, Persist model, bool streamed, int sms,
                                   const int* clusters) {
  if (sticky_eligible(D, model, streamed)) {
    const int S = choose_sticky(F, T, clusters);
    if (S > 0) return {kKernelSticky, S};
  }
  return {runs_ws(D, model) ? kKernelWs : kKernelSingle,
          choose_frame_split(F, T, D, K, persist_ctas_per_sm(D, model == Persist::kFull), sms)};
}

static int device_sms(int* sms) {
  int dev = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  PBB_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

static int setup_frame_split(PersistArgs* p, const CacgmmWorkspace& ws, int F, int D, int K, int S, cudaStream_t st) {
  if (S > 1) {
    p->tsplit = S;
    p->tpart = ws.part + (size_t)F * K * ((size_t)D * D + 1);
    p->tcount = ws.tcount;
    PBB_CUDA(cudaMemsetAsync(ws.tcount, 0, (size_t)F * sizeof(int), st));
  }
  return 0;
}

// ---- shape / dtype dispatch ------------------------------------------------------
// fn(k, ct) with k = std::integral_constant<int, K> for the instantiated K in {2, 3, 4}
template <class Fn>
static int with_k_ct(int K, int dtype, Fn&& fn) {
  auto on_k = [&](auto k) { return with_ct(dtype, [&](auto ct) { return fn(k, ct); }); };
  switch (K) {
    case 2: return on_k(std::integral_constant<int, 2>{});
    case 3: return on_k(std::integral_constant<int, 3>{});
    default: return on_k(std::integral_constant<int, 4>{});
  }
}
// fn(d, k, ct) with d for the instantiated D in {4, 6, 8}
template <class Fn>
static int with_d_k_ct(int D, int K, int dtype, Fn&& fn) {
  auto on_d = [&](auto d) { return with_k_ct(K, dtype, [&](auto k, auto ct) { return fn(d, k, ct); }); };
  switch (D) {
    case 4: return on_d(std::integral_constant<int, 4>{});
    case 6: return on_d(std::integral_constant<int, 6>{});
    default: return on_d(std::integral_constant<int, 8>{});
  }
}
// complex Bingham kernels are instantiated for D = 2..6, the reference's domain (complex_bingham_utils.py:342-348)
template <class Fn>
static int with_bingham_d(int D, Fn&& fn) {
  switch (D) {
    case 2: return fn(std::integral_constant<int, 2>{});
    case 3: return fn(std::integral_constant<int, 3>{});
    case 4: return fn(std::integral_constant<int, 4>{});
    case 5: return fn(std::integral_constant<int, 5>{});
    case 6: return fn(std::integral_constant<int, 6>{});
    default: set_error("complex Bingham: D = %d, need 2 <= D <= 6", D); return -5;
  }
}

// The normalisation kernels put the bins on gridDim.y (at most 65535): more bins take one launch per 65535, with
// y, z (and dead) offset to the launch's first bin.
constexpr int kNormMaxGridY = 65535;

template <typename CT>
static int launch_normalize(const CT* y, CT* z, int F, int T, int D, int swap, int zs, cudaStream_t st) {
  const int block = D <= 16 ? 128 : 32;
  for (int f0 = 0; f0 < F; f0 += kNormMaxGridY) {
    const int nf = std::min(F - f0, kNormMaxGridY);
    // per-bin stride of z: D rows of zs frames (swap), or zs = T frames of D channels
    if (int r = launch_kernel("normalize_kernel", normalize_kernel<CT>, dim3((T + block - 1) / block, nf), block,
                              (size_t)block * (D + 1) * sizeof(double2), st, y + (size_t)f0 * T * D,
                              z + (size_t)f0 * D * zs, nf, T, D, swap, zs))
      return r;
  }
  return 0;
}

// y -> ws.z, rows padded to ws.zs frames, or (staged) in the chunk-major layout of the persistent kernels: one TMA
// bulk copy per ring stage, ws.dead cleared and set for bins with an all-zero frame
static int normalize(const void* y, int dtype, const CacgmmWorkspace& ws, int F, int T, int D, bool staged,
                     cudaStream_t st) {
  if (staged) PBB_CUDA(cudaMemsetAsync(ws.dead, 0, (size_t)F * sizeof(int), st));
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    const CT* src = static_cast<const CT*>(y);
    CT* dst = static_cast<CT*>(ws.z);
    if (!staged) return launch_normalize(src, dst, F, T, D, 1, ws.zs, st);
    const int block = 64;  // divides kStageFrames
    const int nchunks = (ws.zs + kStageFrames - 1) / kStageFrames;
    const size_t bin_elems = (size_t)nchunks * D * kStageFrames;  // out[f][c][d][i]
    for (int f0 = 0; f0 < F; f0 += kNormMaxGridY) {
      const int nf = std::min(F - f0, kNormMaxGridY);
      if (int r = launch_kernel("normalize_staged_kernel", normalize_staged_kernel<CT>,
                                dim3(nchunks * (kStageFrames / block), nf), block,
                                (size_t)block * (D + 1) * sizeof(double2), st, src + (size_t)f0 * T * D,
                                dst + (size_t)f0 * bin_elems, nf, T, D, kStageFrames, nchunks, ws.dead + f0))
        return r;
    }
    return 0;
  });
}

static bool fast_shape(int D, int K) { return (D == 4 || D == 6 || D == 8) && K >= 2 && K <= 4; }

// Fills nch / frames_per_block and launches the EM kernel for the shape.  The bins lie on gridDim.y (at most 65535):
// more bins take one launch per 65535, each bin's work unchanged.  A failed launch returns the (positive) CUDA error
// negated: the callers take any positive value for nch.
int launch_em(EmArgs a, int dtype, int frames_per_block, cudaStream_t st) {
  constexpr int kMaxGridY = 65535;
  const int F = a.F;
  if (fast_shape(a.D, a.K)) {
    int fpb = frames_per_block > 0 ? frames_per_block : 128;
    fpb = (fpb + 31) / 32 * 32;
    if (fpb > (a.T + 31) / 32 * 32) fpb = (a.T + 31) / 32 * 32;
    a.frames_per_block = fpb;
    a.nch = (a.T + fpb - 1) / fpb;
    for (a.f0 = 0; a.f0 < F; a.f0 += kMaxGridY) {
      const int r = with_d_k_ct(a.D, a.K, dtype, [&](auto d, auto k, auto ct) {
        return launch_kernel("em_fast_kernel", em_fast_kernel<decltype(d)::value, decltype(k)::value, decltype(ct)>,
                             dim3(a.nch, std::min(F - a.f0, kMaxGridY)), 32 * kEmGroups, 0, st, a);
      });
      if (r) return r > 0 ? -r : r;
    }
    return a.nch;
  }
  a.frames_per_block = kGenFrames;
  a.nch = (a.T + kGenFrames - 1) / kGenFrames;
  a.softmax_fast = 0;
  const size_t smem = (size_t)2 * a.K * kGenFrames * sizeof(double) + (size_t)a.D * a.D * sizeof(int);
  for (a.f0 = 0; a.f0 < F; a.f0 += kMaxGridY) {
    const int r = with_ct(dtype, [&](auto ct) {
      const auto kern = em_generic_kernel<decltype(ct)>;
      PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      return launch_kernel("em_generic_kernel", kern, dim3(a.nch, std::min(F - a.f0, kMaxGridY)), kGenFrames, smem,
                           st, a);
    });
    if (r) return r > 0 ? -r : r;
  }
  return a.nch;
}

// cacg_update_kernel (UpdArgs) or cw_update_kernel (CwUpdArgs): one CTA per bin, up to 16 warps
// Warps per CTA are also capped by the kernel's own limit (its registers): at small D the shared memory would allow
// 16 warps, more than cacg_update_kernel / cw_update_kernel can launch with, and the class loop covers K > warps.
// cap: the kernel's limit in warps, queried on the first launch (0 until then).
static int max_warps(const void* kern, int* cap, int* w) {
  if (*cap == 0) {
    cudaFuncAttributes at;
    PBB_CUDA(cudaFuncGetAttributes(&at, kern));
    *cap = at.maxThreadsPerBlock / 32;
  }
  if (*w > *cap) *w = *cap;
  return 0;
}

template <typename U>
static int launch_update(void (*kern)(U), const char* name, U u, cudaStream_t st) {
  const size_t per = update_smem_per_warp(u.D);
  int w = (int)((size_t)(200 * 1024) / per);
  if (w > u.K) w = u.K;
  if (w > 16) w = 16;
  static int cap = 0;  // one kernel per instantiation (UpdArgs / CwUpdArgs)
  if (int r = max_warps(reinterpret_cast<const void*>(kern), &cap, &w)) return r;
  if (w < 1) w = 1;
  u.warps = w;
  const size_t smem = per * w + (size_t)2 * u.K * sizeof(double) + (size_t)u.D * u.D * sizeof(int);
  PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  const int threads = 32 * w < u.K ? ((u.K + 31) / 32 * 32) : 32 * w;
  return launch_kernel(name, kern, u.F, threads, smem, st, u);
}

// E-step form of a model given by eigenvectors, eigenvalues and weights (null: 1/K) into the workspace
static int launch_from_eig(const CacgmmWorkspace& ws, int F, int D, int K, const void* evec, const double* eval,
                           const double* weight, cudaStream_t st) {
  FromEigArgs u;
  u.F = F; u.D = D; u.K = K;
  u.evec = reinterpret_cast<const double2*>(evec);
  u.eval = eval; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.w = ws.w; u.ew = ws.ew;
  const size_t per = from_eig_smem_per_warp(D);
  int w = (int)((size_t)(200 * 1024) / per);
  if (w > K) w = K;
  if (w > 16) w = 16;
  static int cap = 0;
  if (int r = max_warps(reinterpret_cast<const void*>(cacg_from_eig_kernel), &cap, &w)) return r;
  u.warps = w;
  const size_t smem = per * w + (size_t)K * sizeof(double) + (size_t)D * D * sizeof(int);
  PBB_CUDA(cudaFuncSetAttribute(cacg_from_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  const int threads = 32 * w < K ? ((K + 31) / 32 * 32) : 32 * w;
  return launch_kernel("cacg_from_eig_kernel", cacg_from_eig_kernel, F, threads, smem, st, u);
}

// ---- kernel arguments --------------------------------------------------------------
// the workspace and shape part of the arguments; each entry point adds what is specific to it
static EmArgs em_args(const CacgmmWorkspace& ws, int F, int T, int D, int K) {
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.coef = ws.coef; a.ld = ws.ld; a.w = ws.w; a.ew = ws.ew; a.part = ws.part;
  return a;
}

static UpdArgs upd_args(const CacgmmWorkspace& ws, int F, int T, int D, int K, const pbb_cacgmm_options* opt,
                        bool has_saliency, void* evec, double* eval, double* weight, int* status) {
  UpdArgs u;
  memset(&u, 0, sizeof(u));
  u.F = F; u.T = T; u.D = D; u.K = K;
  u.part = ws.part;
  u.covariance_norm = opt->covariance_norm;
  u.weight_mode = opt->weight_mode;
  u.has_saliency = has_saliency;
  u.eigenvalue_floor = opt->eigenvalue_floor;
  u.evec = reinterpret_cast<double2*>(evec);
  u.eval = eval; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.ew = ws.ew;
  u.status = status;
  return u;
}

static PersistArgs persist_args(const CacgmmWorkspace& ws, int F, int T, int iterations, int* status) {
  PersistArgs p;
  memset(&p, 0, sizeof(p));
  p.z = ws.z; p.zs = ws.zs; p.F = F; p.T = T;
  p.iterations = iterations;
  p.coef = ws.coef; p.ld = ws.ld; p.w = ws.w; p.ew = ws.ew;
  p.part = ws.part; p.flags = ws.flags; p.ticket = ws.ticket; p.status = status; p.phase = ws.phase;
  return p;
}

// ---- persistent kernel launch ---------------------------------------------------
constexpr int kLoadReserve = 4;  // EM CTA slots left free in streamed-upload mode (insurance, see launch_stream_load)
constexpr int kLoadCtas = 16;    // stream_load_kernel grid

// Task order of the streamed upload (em_persistent.cuh).  The bins arrive over PCIe in ascending
// order, `arrive` per time slot; a slot is one task duration and the machine runs `cap` tasks per
// slot.  List scheduling: every slot takes the (at most cap) arrived, unfinished bins that have
// done the FEWEST iterations -- early bins run ahead while the link is the bottleneck, late bins
// catch up afterwards and all bins finish together instead of leaving a thin tail of late bins.
// A task still only depends on a lower ticket ((b, it - 1) sits in an earlier slot).
// The table (4 bytes per task) is built once per (device, F, iterations, arrive, cap) and kept in a
// small library-owned device cache -- the only device memory the library allocates itself.
// host part of streamed_order: order[ticket] = bin | iteration << 16 (also exported for the CPU tests
// as pbb_streamed_task_order)
static void build_streamed_order(int F, int I, int arrive, int cap, std::vector<int>& order) {
  order.clear();
  order.reserve((size_t)F * I);
  std::vector<int> done(F, 0), count(I + 1), pick;
  for (long long slot = 0; order.size() < (size_t)F * I; ++slot) {
    const int arrived = (int)std::min<long long>(F, (long long)arrive * (slot + 1));
    // threshold = the done-count below which everything is taken, plus a partial level
    std::fill(count.begin(), count.end(), 0);
    for (int b = 0; b < arrived; ++b)
      if (done[b] < I) ++count[done[b]];
    int level = 0, left = cap;
    while (level < I && count[level] <= left) left -= count[level++];
    // all unfinished bins with done < level, and `left` bins of done == level (highest bins first)
    pick.clear();
    for (int b = arrived - 1; b >= 0; --b) {
      if (done[b] >= I) continue;
      if (done[b] < level) pick.push_back(b);
      else if (done[b] == level && left > 0) { pick.push_back(b); --left; }
    }
    for (auto p = pick.rbegin(); p != pick.rend(); ++p) {
      order.push_back(*p | (done[*p] << 16));
      ++done[*p];
    }
  }
}

static int streamed_order(int F, int I, int arrive, int cap, const int** out) {
  static std::mutex mu;
  static std::map<std::array<int, 5>, int*> cache;
  std::lock_guard<std::mutex> lk(mu);
  int dev = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  const std::array<int, 5> key{dev, F, I, arrive, cap};
  auto hit = cache.find(key);
  if (hit != cache.end()) { *out = hit->second; return 0; }
  if (cache.size() >= 16) {
    for (auto& kv : cache) cudaFree(kv.second);
    cache.clear();
  }
  std::vector<int> order;
  build_streamed_order(F, I, arrive, cap, order);
  int* d = nullptr;
  PBB_CUDA(cudaMalloc(&d, order.size() * sizeof(int)));
  PBB_CUDA(cudaMemcpy(d, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice));
  cache[key] = d;
  *out = d;
  return 0;
}

// Replaces *p by the address the kernels use: itself for device memory, the mapped device alias of pinned host
// memory (*is_host = true); any other memory is an error.
template <typename P>
static int device_alias(P** p, bool* is_host, const char* what) {
  cudaPointerAttributes at;
  PBB_CUDA(cudaPointerGetAttributes(&at, *p));
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) {
    *is_host = false;
    return 0;
  }
  if (at.type == cudaMemoryTypeHost && at.devicePointer != nullptr) {
    *is_host = true;
    *p = static_cast<P*>(at.devicePointer);
    return 0;
  }
  set_error("%s must be device memory or pinned (page-locked, mapped) host memory", what);
  return -1;
}

// side stream + events for the upload that overlaps the EM kernel (one set per process)
typedef CUresult (*StreamWaitValue32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
struct LoadStream {
  std::mutex mu;  // one streamed fit per device enqueues at a time (the side stream and its events are shared)
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  StreamWaitValue32Fn wait_value = nullptr;  // cuStreamWaitValue32, resolved through the runtime
  int device = -1;
};
static int get_load_stream(LoadStream** out) {
  static LoadStream ls[16];
  static std::mutex init_mu;
  std::lock_guard<std::mutex> init_lk(init_mu);
  int dev = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 16) { set_error("device index %d out of range", dev); return 1; }
  LoadStream& l = ls[dev];
  if (l.stream == nullptr) {
    PBB_CUDA(cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking));
    PBB_CUDA(cudaEventCreateWithFlags(&l.fork, cudaEventDisableTiming));
    PBB_CUDA(cudaEventCreateWithFlags(&l.join, cudaEventDisableTiming));
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      l.wait_value = reinterpret_cast<StreamWaitValue32Fn>(fn);
    (void)cudaGetLastError();
    l.device = dev;
  }
  *out = &l;
  return 0;
}

static int launch_stream_load(const void* y, int dtype, const CacgmmWorkspace& ws, const double* aff_src,
                              double* aff_dst, int F, int T, int D, int K, int ctas, cudaStream_t st) {
  const int nchunks = (ws.zs + kStageFrames - 1) / kStageFrames;
  const size_t smem = (size_t)kStageFrames * (D + 1) * sizeof(double2);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("stream_load_kernel", stream_load_kernel<CT>, ctas, kLoadThreads, smem, st,
                         static_cast<const CT*>(y), static_cast<CT*>(ws.z), aff_src, aff_dst, F, T, D, K,
                         kStageFrames, nchunks, ws.dead, ws.flags, ws.load_next_bin, ws.load_started);
  });
}

template <typename Kern>
static int launch_persistent_generic(Kern kern, int threads, size_t smem, int* cache, const PersistArgs& a,
                                     const char* name, cudaStream_t st) {
  // streamed upload: leave kLoadReserve CTA slots free so that stream_load_kernel's CTAs are
  // resident whatever order the two launches start in (the EM kernel waits on their flags)
  const int reserve = a.wait_load ? kLoadReserve : 0;
  if (*cache == 0) {
    PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int n = 0;
    PBB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, threads, smem));
    if (n < 1) { set_error("%s does not fit on this device", name); return 1; }
    *cache = n;
  }
  int sms = 0;
  if (int r = device_sms(&sms)) return r;
  long long grid = (long long)(*cache) * sms - reserve;
  if (grid < 1) grid = 1;
  const long long tasks = (long long)a.iterations * a.F * (a.tsplit > 1 ? a.tsplit : 1);
  if (grid > tasks) grid = tasks;
  return launch_kernel(name, kern, (unsigned)grid, threads, smem, st, a);
}

// The task kernel of a model: em_ws_kernel for the lean D = 8 model (the warp-specialised kernel), otherwise
// em_persistent_kernel.
static int launch_persist(const PersistArgs& a, int D, int K, int dtype, Persist v, cudaStream_t st) {
  return with_d_k_ct(D, K, dtype, [&](auto d, auto k, auto ct) {
    constexpr int Dc = decltype(d)::value, Kc = decltype(k)::value;
    using CT = decltype(ct);
    static int cache[3] = {0, 0, 0};  // occupancy per Persist, queried on the first launch
    const int threads = persist_threads(Dc, Kc);
    const size_t smem = sizeof(PersistSmem<Dc, Kc, CT>);
    int* c = &cache[(int)v];
    // the full variant's launches carry their own name, so that profiles and tests can tell it from the lean one
    if (v == Persist::kFull)
      return launch_persistent_generic(em_persistent_kernel<Dc, Kc, CT, true>, threads, smem, c, a,
                                       "em_persistent_kernel_full", st);
    if (v == Persist::kCw)
      return launch_persistent_generic(em_persistent_kernel<Dc, Kc, CT, false, 1>, threads, smem, c, a,
                                       "em_persistent_kernel_cw", st);
    if constexpr (Dc == 8)
      return launch_persistent_generic(em_ws_kernel<Kc, CT>, 256, sizeof(WsSmem<Dc, Kc, CT>), c, a, "em_ws_kernel", st);
    else
      return launch_persistent_generic(em_persistent_kernel<Dc, Kc, CT, false>, threads, smem, c, a,
                                       "em_persistent_kernel", st);
  });
}

// "Sticky bins" (em_sticky.cuh): when the device runs F clusters of S CTAs at once, a cluster keeps one bin for the
// whole fit (choose_sticky).
// Clusters of 1, 2, 4 CTAs of em_sticky_kernel the device runs at once (queried once per instantiation).
static int sticky_clusters(int K, int dtype, int clusters[3], cudaStream_t st) {
  return with_k_ct(K, dtype, [&](auto k, auto ct) {
    static int cache[3] = {-1, -1, -1};
    if (cache[0] < 0) {
      const auto kern = em_sticky_kernel<decltype(k)::value, decltype(ct)>;
      const size_t smem = sizeof(WsSmem<8, decltype(k)::value, decltype(ct)>);
      PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      for (int i = 0; i < 3; ++i) {
        const ClusterLaunch cl(1u << i, 256, smem, 1u << i, st);
        int n = 0;
        PBB_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cl.cfg));
        cache[i] = n;
      }
    }
    for (int i = 0; i < 3; ++i) clusters[i] = cache[i];
    return 0;
  });
}

// one cluster of S CTAs per bin; sticky_clusters has set the kernel's shared-memory limit
static int launch_sticky(const PersistArgs& a, int K, int dtype, int S, cudaStream_t st) {
  return with_k_ct(K, dtype, [&](auto k, auto ct) {
    const ClusterLaunch cl((unsigned)(a.F * S), 256, sizeof(WsSmem<8, decltype(k)::value, decltype(ct)>),
                           (unsigned)S, st);
    return launch_ex("em_sticky_kernel", cl.cfg, em_sticky_kernel<decltype(k)::value, decltype(ct)>, a);
  });
}

// The plan of the last persistent fit this host thread launched (pbb_em_last_plan): kernel, split, variant.
struct LastPlan { int kernel, split, variant; };
static thread_local LastPlan g_last_plan = {-1, 0, -1};

// Plan and launch of a persistent fit whose control block is clear: the sticky-bins kernel when the plan picks it,
// otherwise the frame split and the task kernel.
static int launch_planned(PersistArgs p, const CacgmmWorkspace& ws, int D, int K, int dtype, Persist model,
                          bool streamed, cudaStream_t st) {
  int clusters[3] = {0, 0, 0}, sms = 0, r;
  if (sticky_eligible(D, model, streamed) && (r = sticky_clusters(K, dtype, clusters, st))) return r;
  if ((r = device_sms(&sms))) return r;
  const FitPlan plan = plan_persistent_fit(p.F, p.T, D, K, model, streamed, sms, clusters);
  g_last_plan = {plan.kernel, plan.split,
                 model == Persist::kCw ? 3 : (model == Persist::kLean ? 0 : (p.softmax_fast ? 1 : 2))};
  if (plan.kernel == kKernelSticky) return launch_sticky(p, K, dtype, plan.split, st);  // few bins: one cluster per bin
  if ((r = setup_frame_split(&p, ws, p.F, D, K, plan.split, st))) return r;
  return launch_persist(p, D, K, dtype, model, st);
}

#ifdef PBB_PHASE_TIMING
// cycles per task of the persistent kernel's phases (PBB_PH / PBB_PHU in em_persistent.cuh and em_ws.cuh)
static void print_phases(const CacgmmWorkspace& ws, long long tasks, bool cw, cudaStream_t st) {
  unsigned long long ph[12];
  cudaStreamSynchronize(st);
  cudaMemcpy(ph, ws.phase, sizeof(ph), cudaMemcpyDeviceToHost);
  if (!cw)
    fprintf(stderr, "[phase] update of class 0, cycles per task: build %.0f  gauss-jordan %.0f  logdet/tinv %.0f  stores %.0f\n",
            ph[8] / (double)tasks, ph[9] / (double)tasks, ph[10] / (double)tasks, ph[11] / (double)tasks);
  unsigned long long tot = 0;
  for (int i = 0; i < 8; ++i) tot += ph[i];
  static const char* nm[8] = {"ticket+flag / model wait", "chunk-top / updater busy", "tma-wait", "em-steps", "reduce", "update / S wait", "publish / hand-over", "task-start / updater idle"};
  static const char* nm_cw[8] = {"flag wait", "chunk top / staging", "tma-wait", "em-steps", "reduce", "update (jacobi)", "publish", "task-start"};
  for (int i = 0; i < 8; ++i)
    fprintf(stderr, "[phase%s] %-20s %6.2f%%  %8.0f cycles per task\n", cw ? " cw" : "", cw ? nm_cw[i] : nm[i],
            100.0 * ph[i] / (double)tot, ph[i] / (double)tasks);
}
#endif

// ---- entry-point steps ------------------------------------------------------------
static bool softmax_fast_ok(int D, const pbb_cacgmm_options* o) {
  if (o->covariance_norm != PBB_NORM_EIGENVALUE) return false;
  if (!(o->eigenvalue_floor > 0.0) || o->eigenvalue_floor > 1.0) return false;
  return 2.0 * D * log10(1.0 / o->eigenvalue_floor) < 280.0;
}

static int check_shape(int F, int T, int D, int K, int dtype) {
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(F > 0, 3, "F must be positive");
  PBB_CHECK_ARG(T > 0, 4, "T must be positive");
  PBB_CHECK_ARG(D > 1 && D < 35, 5, "need 1 < D < 35 (cacgmm.py:197,250)");
  PBB_CHECK_ARG(K > 0 && K < kMaxK, 6, "need 0 < K < 20 (cacgmm.py:249)");
  return 0;
}

static int check_cbmm_shape(int F, int T, int D, int K, int dtype) {
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(D >= 2 && D <= 6, 5, "complex Bingham: need 2 <= D <= 6 (complex_bingham_utils.py:342-348)");
  PBB_CHECK_ARG((long long)F * K <= kCbMaxIndex, 6, "F * K too large for the status word");
  return 0;
}

enum class Layout { kNone, kPlain, kStaged };

// Opening of the EM entry points, after their other argument checks: the workspace (argument ws_arg) and status
// (ws_arg + 2) checks, the workspace carve, the status reset and, unless layout is kNone, normalize.
static int begin_call(const void* y, int dtype, int F, int T, int D, int K, void* workspace, size_t workspace_bytes,
                      int ws_arg, const char* ws_msg, int* status, Layout layout, cudaStream_t st,
                      CacgmmWorkspace* ws) {
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= carve(nullptr, F, T, D, K).bytes, ws_arg, ws_msg);
  PBB_CHECK_ARG(status != nullptr, ws_arg + 2, "status is null");
  *ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  return layout == Layout::kNone ? 0 : normalize(y, dtype, *ws, F, T, D, layout == Layout::kStaged, st);
}

// One pbb_cacgmm_fit call after its argument checks.
struct FitCall {
  const void* y;
  int dtype, F, T, D, K;
  const double *init_aff, *saliency;
  const uint8_t* activity;
  const pbb_cacgmm_options* opt;
  void* evec;
  double *eval, *weight;
  int* status;
  cudaStream_t st;
  CacgmmWorkspace ws;
  bool y_host, aff_host;  // y / the initial affiliations are pinned host memory
};

// y (and the initial affiliations) may be pinned host memory: the kernels then read them in place over PCIe.  The
// model may be written straight into pinned host memory as well (write-only on this path).
static int resolve_host_aliases(FitCall& c) {
  int r;
  bool h = false;
  if ((r = device_alias(&c.y, &c.y_host, "y"))) return r;
  if (c.init_aff != nullptr && (r = device_alias(&c.init_aff, &c.aff_host, "initial affiliations"))) return r;
  if ((r = device_alias(&c.evec, &h, "eigenvectors"))) return r;
  if ((r = device_alias(&c.eval, &h, "eigenvalues"))) return r;
  return device_alias(&c.weight, &h, "weight");
}

// Streamed upload: on the persistent path with a host-resident y and an affiliation initialisation, a separate
// small kernel on a side stream reads them over PCIe into the staged layout while the EM kernel runs.  Clears the
// control block (flags[bin] = -1 until the bin has arrived) and fills the upload fields of p.
static int start_streamed_upload(FitCall& c, LoadStream& l, PersistArgs* p) {
  const CacgmmWorkspace& ws = c.ws;
  const int F = c.F, T = c.T, D = c.D, K = c.K, iterations = c.opt->iterations;
  PBB_CUDA(cudaMemsetAsync(ws.flags, 0, ws.control_bytes, c.st));
  PBB_CUDA(cudaMemsetAsync(ws.flags, 0xFF, (size_t)F * sizeof(int), c.st));
  PBB_CUDA(cudaMemsetAsync(ws.dead, 0, (size_t)F * sizeof(int), c.st));
  PBB_CUDA(cudaEventRecord(l.fork, c.st));
  PBB_CUDA(cudaStreamWaitEvent(l.stream, l.fork, 0));
  const int ctas = std::min(kLoadCtas, F);
  if (int r = launch_stream_load(c.y, c.dtype, ws, c.init_aff, c.aff_host ? ws.aff_stage : nullptr, F, T, D, K, ctas,
                                 l.stream))
    return r;
  PBB_CUDA(cudaEventRecord(l.join, l.stream));
  // Hold the EM kernel back until every loader CTA runs: launched at the same moment, the EM grid
  // could take the whole machine first and leave the loader only the reserved slots (it would still
  // finish -- bins are handed out by a counter -- but at a fraction of the link rate).
  if (l.wait_value != nullptr) {
    if (l.wait_value(reinterpret_cast<CUstream>(c.st), reinterpret_cast<CUdeviceptr>(ws.load_started),
                     (cuuint32_t)ctas, CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
      l.wait_value = nullptr;  // not supported here: rely on the reserved slots
  }
  if (c.aff_host) c.init_aff = ws.aff_stage;
  // bins joining per slot ~ slot duration / arrival time of one bin at ~50 GB/s of PCIe reads
  const double bin_bytes = (double)T * D * (c.dtype == PBB_C128 ? 16.0 : 8.0) + (c.aff_host ? 8.0 * K * T : 0.0);
  // one slot of the order table = one link of a bin's dependency chain (task + update + staging
  // of the next model, ~23 us at D = 8, K = 3, T = 500), during which the machine runs ~1.6 tasks per CTA
  const double round_us = 23.0 * (T / 500.0) * (D * D / 64.0) * (K / 3.0);
  int wave = (int)(round_us / (bin_bytes / 50e3) + 0.5);
  wave = wave < 1 ? 1 : (wave > F ? F : wave);
  p->wave_c = wave;
  p->wait_load = 1;
  // the explicit task order where the table stays small; beyond that decode_ticket's rounds of wave_c bins
  if ((long long)F * iterations <= kMaxOrder && F <= 4096 && iterations < 32768) {
    int sms = 0;
    if (int r = device_sms(&sms)) return r;
    const int cap = (int)(1.6 * (2 * sms - kLoadReserve));
    if (int r = streamed_order(F, iterations, wave, cap < 1 ? 1 : cap, &p->order)) return r;
  }
  return 0;
}

// Persistent fit: every EM iteration in one launch (em_persistent.cuh), then the last iteration's raw scatter sums
// through cacg_update_kernel for the reference-exact model.  p carries the streamed-upload fields; load is the side
// stream of a streamed upload (which has cleared the control block), else null.
static int run_persistent_fit(const FitCall& c, PersistArgs p, bool full, bool fast_sm, const LoadStream* load) {
  const CacgmmWorkspace& ws = c.ws;
  const pbb_cacgmm_options* opt = c.opt;
  int r;
  if (load == nullptr) PBB_CUDA(cudaMemsetAsync(ws.flags, 0, ws.control_bytes, c.st));
  if (c.init_aff == nullptr && (r = launch_from_eig(ws, c.F, c.D, c.K, c.evec, c.eval, c.weight, c.st))) return r;
  p.first_is_m = c.init_aff != nullptr;
  p.user_model = c.init_aff == nullptr;
  p.softmax_fast = fast_sm;
  p.aff_in = c.init_aff; p.saliency = c.saliency; p.activity = c.activity;
  p.aff_eps = opt->affiliation_eps; p.eigenvalue_floor = opt->eigenvalue_floor;
  p.covariance_norm = opt->covariance_norm; p.weight_mode = opt->weight_mode;
  p.dead = ws.dead;
  if ((r = launch_planned(p, ws, c.D, c.K, c.dtype, full ? Persist::kFull : Persist::kLean, load != nullptr, c.st)))
    return r;
  if (load != nullptr) PBB_CUDA(cudaStreamWaitEvent(c.st, load->join, 0));
#ifdef PBB_PHASE_TIMING
  print_phases(ws, (long long)c.F * opt->iterations, false, c.st);
#endif
  UpdArgs u = upd_args(ws, c.F, c.T, c.D, c.K, opt, c.saliency != nullptr, c.evec, c.eval, c.weight, c.status);
  u.nch = 1;         // the last iteration's raw scatter sums -> reference-exact model
  u.coef = nullptr;  // nobody reads the E-step form of the final model
  return launch_update(cacg_update_kernel, "cacg_update_kernel", u, c.st);
}

// Per-iteration fit: one EM launch and one update launch per iteration.
static int run_iterative_fit(const FitCall& c, bool fast_sm) {
  const CacgmmWorkspace& ws = c.ws;
  EmArgs a = em_args(ws, c.F, c.T, c.D, c.K);
  a.activity = c.activity; a.aff_eps = c.opt->affiliation_eps; a.saliency = c.saliency;
  UpdArgs u = upd_args(ws, c.F, c.T, c.D, c.K, c.opt, c.saliency != nullptr, c.evec, c.eval, c.weight, c.status);
  int it = 0, r;
  if (c.init_aff != nullptr) {
    // iteration 0: M-step from the initial affiliations, q = 1 (cacgmm.py:206-228,269)
    a.mode = kModeM; a.aff_in = c.init_aff; a.q_in = nullptr;
    int nch = launch_em(a, c.dtype, c.opt->frames_per_block, c.st);
    if (nch <= 0) return nch ? nch : 1;
    u.nch = nch;
    if ((r = launch_update(cacg_update_kernel, "cacg_update_kernel", u, c.st))) return r;
    it = 1;
  } else {
    // warm start: the model in the output arrays drives the first E-step (cacgmm.py:229-234)
    if ((r = launch_from_eig(ws, c.F, c.D, c.K, c.evec, c.eval, c.weight, c.st))) return r;
  }
  // the update kernel writes the E-step weights into `weight`; the E-step reads them from there
  a.w = c.weight;
  for (; it < c.opt->iterations; ++it) {
    a.mode = kModeEM;
    // a user-supplied model gives no bound on q / log det: keep the log-domain softmax for its E-step
    a.softmax_fast = (fast_sm && !(c.init_aff == nullptr && it == 0)) ? 1 : 0;
    if (c.init_aff == nullptr && it == 0) a.w = ws.w;
    int nch = launch_em(a, c.dtype, c.opt->frames_per_block, c.st);
    if (nch <= 0) return nch ? nch : 1;
    a.w = c.weight;
    u.nch = nch;
    if ((r = launch_update(cacg_update_kernel, "cacg_update_kernel", u, c.st))) return r;
  }
  return 0;
}

// ---- backward passes (em_backward.cuh) ------------------------------------------------
// The forward's workspace (carve), then the backward's own arrays.
struct CacgmmBwdWorkspace {
  CacgmmWorkspace em;
  double* qcoef;   // (F, K, T) coefficients of the E-step adjoint's scatter
  double* wpart;   // (F, nchb, 2K) chunk sums of the weight and log det gradients
  double2* gpsi;   // (F, K, D, D) Psibar of the M-step adjoint
  double* gS;      // (F, K) Sbar
  size_t bytes;
};

static int bwd_chunks(int T) { return (T + kBwdFrames - 1) / kBwdFrames; }

static CacgmmBwdWorkspace carve_bwd(void* base, int F, int T, int D, int K) {
  CacgmmBwdWorkspace b;
  b.em = carve(base, F, T, D, K);
  char* p = reinterpret_cast<char*>(base);
  size_t off = align_up(b.em.bytes);
  auto take = [&](size_t n) { char* q = p + off; off += align_up(n); return q; };
  b.qcoef = reinterpret_cast<double*>(take((size_t)F * K * T * sizeof(double)));
  b.wpart = reinterpret_cast<double*>(take((size_t)F * bwd_chunks(T) * 2 * K * sizeof(double)));
  b.gpsi = reinterpret_cast<double2*>(take((size_t)F * K * D * D * sizeof(double2)));
  b.gS = reinterpret_cast<double*>(take((size_t)F * K * sizeof(double)));
  b.bytes = off;
  return b;
}

// one CTA per (bin, frame chunk) (per_frame) or per (bin, class)
template <typename Kern, typename Args>
static int launch_bwd(const char* name, Kern kern, dim3 grid, int threads, size_t smem, const Args& a,
                      cudaStream_t st) {
  PBB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel(name, kern, grid, threads, smem, st, a);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

const char* pbb_last_error(void) { return g_err; }
int pbb_version(void) { return 109; }

int pbb_normalize_observation(const void* y, void* z, int F, int T, int D, int dtype, int swap, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(z != nullptr, 2, "z is null");
  PBB_CHECK_ARG(F > 0 && T > 0, 3, "empty shape");
  PBB_CHECK_ARG(D > 0 && D < 256, 5, "bad D");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 6, "bad dtype");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_normalize(static_cast<const CT*>(y), static_cast<CT*>(z), F, T, D, swap, T, st);
  });
}

int pbb_em_dispatch(int F, int T, int D, int K, int lean, int streamed, int sms, int* kernel, int* split) {
  PBB_CHECK_ARG(F > 0, 1, "F must be positive");
  PBB_CHECK_ARG(T > 0, 2, "T must be positive");
  PBB_CHECK_ARG(D == 4 || D == 6 || D == 8, 3, "persistent kernels: D in {4, 6, 8}");
  PBB_CHECK_ARG(K >= 2 && K <= 4, 4, "persistent kernels: K in {2, 3, 4}");
  PBB_CHECK_ARG(sms > 0, 7, "sms must be positive");
  PBB_CHECK_ARG(kernel != nullptr && split != nullptr, 8, "output is null");
  const int clusters[3] = {2 * sms, sms, sms / 2};  // machine model: two CTAs per SM, clusters placed anywhere
  const FitPlan plan =
      plan_persistent_fit(F, T, D, K, lean ? Persist::kLean : Persist::kFull, streamed != 0, sms, clusters);
  *kernel = plan.kernel;
  *split = plan.split;
  return 0;
}

int pbb_em_last_plan(int* kernel, int* split, int* variant) {
  PBB_CHECK_ARG(kernel != nullptr && split != nullptr && variant != nullptr, 1, "output is null");
  *kernel = g_last_plan.kernel;
  *split = g_last_plan.split;
  *variant = g_last_plan.variant;
  return 0;
}

int pbb_streamed_task_order(int F, int iterations, int arrive, int cap, int* order) {
  PBB_CHECK_ARG(F > 0 && F <= 65535, 1, "need 0 < F < 65536");
  PBB_CHECK_ARG(iterations > 0 && iterations < 32768, 2, "need 0 < iterations < 32768");
  PBB_CHECK_ARG(arrive > 0, 3, "arrive must be positive");
  PBB_CHECK_ARG(cap > 0, 4, "cap must be positive");
  PBB_CHECK_ARG(order != nullptr, 5, "order is null");
  std::vector<int> o;
  build_streamed_order(F, iterations, arrive, cap, o);
  memcpy(order, o.data(), o.size() * sizeof(int));
  return 0;
}

size_t pbb_cacgmm_workspace_bytes(int F, int T, int D, int K) {
  if (F <= 0 || T <= 0 || D <= 0 || K <= 0) return 0;
  return carve(nullptr, F, T, D, K).bytes;
}

int pbb_cacgmm_fit(const void* y, int dtype, int F, int T, int D, int K, const double* init_aff,
                   const double* saliency, const uint8_t* activity, const pbb_cacgmm_options* opt,
                   void* eigenvectors, double* eigenvalues, double* weight, void* workspace,
                   size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(opt != nullptr, 10, "options are null");
  PBB_CHECK_ARG(opt->iterations > 0, 10, "iterations must be positive (cacgmm.py:200)");
  PBB_CHECK_ARG(opt->covariance_norm >= 0 && opt->covariance_norm <= 2, 10, "bad covariance_norm");
  PBB_CHECK_ARG(opt->weight_mode == PBB_WEIGHT_TIME || opt->weight_mode == PBB_WEIGHT_CONST, 10, "bad weight_mode");
  PBB_CHECK_ARG((opt->reserved & ~1) == 0, 10, "reserved: only bit 0 (multi-kernel path) is defined");
  PBB_CHECK_ARG(eigenvectors && eigenvalues && weight, 11, "model output is null");
  FitCall c{y, dtype, F, T, D, K, init_aff, saliency, activity, opt, eigenvectors, eigenvalues, weight, status,
            reinterpret_cast<cudaStream_t>(stream)};
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 14,
                      "workspace too small (pbb_cacgmm_workspace_bytes)", status, Layout::kNone, c.st, &c.ws)))
    return r;
  if ((r = resolve_host_aliases(c))) return r;
  const bool persistent = fast_shape(D, K) && !(opt->reserved & 1);
  const bool fast_sm = softmax_fast_ok(D, opt);
  if (!persistent) {
    if ((r = normalize(c.y, dtype, c.ws, F, T, D, false, c.st))) return r;
    return run_iterative_fit(c, fast_sm);
  }
  const bool streamed = c.y_host && c.init_aff != nullptr;
  // lean variant: product-form softmax, needs (K-1) D log10(1/floor) < 290 (em_persistent.cuh).  The extra decade
  // per factor below is a margin kept as is: without it some fits (e.g. K = 4, D = 8 with floors between about 1e-12
  // and 1e-11) would move from the full variant to the lean one.
  const bool lean_ok = fast_sm && (K - 1) * D * (log10(1.0 / opt->eigenvalue_floor) + 1.0) < 290.0;
  const bool full = saliency != nullptr || activity != nullptr || !lean_ok || c.init_aff == nullptr;
  PersistArgs p = persist_args(c.ws, F, T, opt->iterations, status);
  if (!streamed) {
    if ((r = normalize(c.y, dtype, c.ws, F, T, D, true, c.st))) return r;
    return run_persistent_fit(c, p, full, fast_sm, nullptr);
  }
  // Thread safety: the side stream and the fork / join events of the streamed upload exist once per device, so two
  // host threads enqueueing streamed fits on the same device are serialised from here to the end of the call
  // (the enqueue only; the GPU work of the two fits still overlaps as far as their streams allow).
  LoadStream* load = nullptr;
  if ((r = get_load_stream(&load))) return r;
  std::lock_guard<std::mutex> stream_lock(load->mu);
  if ((r = start_streamed_upload(c, *load, &p))) return r;
  return run_persistent_fit(c, p, full, fast_sm, load);
}

int pbb_cacgmm_predict(const void* y, int dtype, int F, int T, int D, int K, const void* eigenvectors,
                       const double* eigenvalues, const double* weight, int weight_mode,
                       const uint8_t* activity, double affiliation_eps, double* affiliation, double* quadratic,
                       double* loglik, void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(eigenvectors && eigenvalues, 7, "model is null");
  PBB_CHECK_ARG(weight != nullptr || weight_mode == PBB_WEIGHT_CONST, 9, "weight is null");
  PBB_CHECK_ARG(weight_mode >= 0 && weight_mode <= PBB_WEIGHT_TIED, 10, "bad weight_mode");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws;
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 16,
                      "workspace too small (pbb_cacgmm_workspace_bytes)", status, Layout::kPlain, st, &ws)))
    return r;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  const double* w = (weight_mode == PBB_WEIGHT_CONST || tied) ? nullptr : weight;
  if ((r = launch_from_eig(ws, F, D, K, eigenvectors, eigenvalues, w, st))) return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.mode = kModeE;
  if (tied) { a.w_time = weight; a.w_time_st = weight_mode == PBB_WEIGHT_TIED_TIME ? 1 : 0; }
  a.activity = activity; a.aff_eps = affiliation_eps;
  a.aff_out = affiliation; a.q_out = quadratic;
  a.loglik_part = loglik ? ws.loglik_part : nullptr;
  int nch = launch_em(a, dtype, 0, st);
  if (nch <= 0) return nch ? nch : 1;
  if (!loglik) return 0;
  // per-bin sum of the chunk partials, fixed order
  return launch_kernel("sum_rows_kernel", sum_rows_kernel, (F + 127) / 128, 128, 0, st, ws.loglik_part, loglik, F, nch);
}

int pbb_cacgmm_mstep(const void* y, int dtype, int F, int T, int D, int K, const double* affiliation,
                     const double* quadratic, const double* saliency, const pbb_cacgmm_options* opt,
                     void* eigenvectors, double* eigenvalues, double* weight, void* workspace,
                     size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(affiliation != nullptr, 7, "affiliation is null");
  PBB_CHECK_ARG(opt != nullptr, 10, "options are null");
  PBB_CHECK_ARG(eigenvectors && eigenvalues && weight, 11, "model output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws;
  if (int r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 14,
                         "workspace too small (pbb_cacgmm_workspace_bytes)", status, Layout::kPlain, st, &ws))
    return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.mode = kModeM; a.aff_in = affiliation; a.q_in = quadratic;
  a.saliency = saliency;
  int nch = launch_em(a, dtype, opt->frames_per_block, st);
  if (nch <= 0) return nch ? nch : 1;
  UpdArgs u = upd_args(ws, F, T, D, K, opt, saliency != nullptr, eigenvectors, eigenvalues, weight, status);
  u.nch = nch;
  return launch_update(cacg_update_kernel, "cacg_update_kernel", u, st);
}

size_t pbb_cacgmm_predict_backward_workspace_bytes(int F, int T, int D, int K) {
  if (F <= 0 || T <= 0 || D <= 0 || K <= 0) return 0;
  return carve_bwd(nullptr, F, T, D, K).bytes;
}

size_t pbb_cacgmm_mstep_backward_workspace_bytes(int F, int T, int D, int K) {
  return pbb_cacgmm_predict_backward_workspace_bytes(F, T, D, K);
}

int pbb_cacgmm_predict_backward(const void* y, int dtype, int F, int T, int D, int K, const void* eigenvectors,
                                const double* eigenvalues, const double* weight, const uint8_t* activity,
                                double affiliation_eps, const double* affiliation, const double* quadratic,
                                const double* grad_affiliation, const double* grad_quadratic,
                                const double* grad_loglik, void* grad_y, void* grad_eigenvectors,
                                double* grad_eigenvalues, double* grad_weight, void* workspace,
                                size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(eigenvectors && eigenvalues && weight, 7, "model is null");
  PBB_CHECK_ARG(affiliation && quadratic, 12, "the forward's affiliation / quadratic form is null");
  PBB_CHECK_ARG(grad_y && grad_eigenvectors && grad_eigenvalues && grad_weight, 17, "gradient output is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= carve_bwd(nullptr, F, T, D, K).bytes, 21,
                "workspace too small (pbb_cacgmm_predict_backward_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CacgmmBwdWorkspace ws = carve_bwd(workspace, F, T, D, K);
  int r;
  if ((r = normalize(y, dtype, ws.em, F, T, D, false, st))) return r;
  if ((r = launch_from_eig(ws.em, F, D, K, eigenvectors, eigenvalues, weight, st))) return r;
  const int nchb = bwd_chunks(T);
  EstepBwdArgs e;
  e.y = y; e.F = F; e.T = T; e.D = D; e.K = K; e.nch = nchb;
  e.coef = ws.em.coef; e.ld = ws.em.ld; e.w = ws.em.w; e.activity = activity; e.eps = affiliation_eps;
  e.aff = affiliation; e.q = quadratic; e.gaff = grad_affiliation; e.gq = grad_quadratic; e.gll = grad_loglik;
  e.qcoef = ws.qcoef; e.part = ws.wpart; e.ybar = static_cast<double2*>(grad_y);
  if ((r = with_ct(dtype, [&](auto ct) {
         return launch_bwd("cacgmm_estep_bwd_kernel", cacgmm_estep_bwd_kernel<decltype(ct)>, dim3(F, nchb),
                           kBwdFrames, bwd_frame_smem(D, 3 * K), e, st);
       })))
    return r;
  // Bbar^-1 = sum_t qbar_raw z z^H: the forward's scatter kernel with the coefficients as affiliations
  EmArgs a = em_args(ws.em, F, T, D, K);
  a.mode = kModeM; a.aff_in = ws.qcoef; a.q_in = nullptr;
  const int nch = launch_em(a, dtype, 0, st);
  if (nch <= 0) return nch ? nch : 1;
  PredictSpecBwdArgs p;
  p.F = F; p.D = D; p.K = K; p.nch = nch; p.nchb = nchb; p.part = ws.em.part; p.wpart = ws.wpart;
  p.V = static_cast<const double2*>(eigenvectors); p.lam = eigenvalues;
  p.gV = static_cast<double2*>(grad_eigenvectors); p.glam = grad_eigenvalues; p.gw = grad_weight;
  const size_t smem = (size_t)2 * D * D * sizeof(double2) + (size_t)D * D * sizeof(double);
  return launch_bwd("cacgmm_predict_spec_bwd_kernel", cacgmm_predict_spec_bwd_kernel, dim3(F, K), 32, smem, p, st);
}

int pbb_cacgmm_mstep_backward(const void* y, int dtype, int F, int T, int D, int K, const double* affiliation,
                              const double* quadratic, const double* saliency, const pbb_cacgmm_options* opt,
                              const void* eigenvectors, const double* eigenvalues, const void* grad_eigenvectors,
                              const double* grad_eigenvalues, const double* grad_weight, void* grad_y,
                              double* grad_affiliation, double* grad_quadratic, double* grad_saliency,
                              void* workspace, size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(affiliation != nullptr, 7, "affiliation is null");
  PBB_CHECK_ARG(opt != nullptr, 10, "options are null");
  PBB_CHECK_ARG(opt->covariance_norm >= 0 && opt->covariance_norm <= 2, 10, "bad covariance_norm");
  PBB_CHECK_ARG(opt->weight_mode == PBB_WEIGHT_TIME || opt->weight_mode == PBB_WEIGHT_CONST, 10,
                "weight_mode: PBB_WEIGHT_TIME or PBB_WEIGHT_CONST");
  PBB_CHECK_ARG(eigenvectors && eigenvalues, 11, "the forward's model is null");
  PBB_CHECK_ARG(grad_y && grad_affiliation, 16, "gradient output is null");
  PBB_CHECK_ARG((grad_quadratic != nullptr) == (quadratic != nullptr), 18, "grad_quadratic iff quadratic");
  PBB_CHECK_ARG((grad_saliency != nullptr) == (saliency != nullptr), 19, "grad_saliency iff saliency");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= carve_bwd(nullptr, F, T, D, K).bytes, 20,
                "workspace too small (pbb_cacgmm_mstep_backward_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const CacgmmBwdWorkspace ws = carve_bwd(workspace, F, T, D, K);
  int r;
  if ((r = normalize(y, dtype, ws.em, F, T, D, false, st))) return r;
  // the forward's scatter sums, recomputed by the forward's launch
  EmArgs a = em_args(ws.em, F, T, D, K);
  a.mode = kModeM; a.aff_in = affiliation; a.q_in = quadratic; a.saliency = saliency;
  const int nch = launch_em(a, dtype, opt->frames_per_block, st);
  if (nch <= 0) return nch ? nch : 1;
  MstepSpecBwdArgs m;
  m.F = F; m.T = T; m.D = D; m.K = K; m.nch = nch; m.part = ws.em.part;
  m.covariance_norm = opt->covariance_norm; m.weight_mode = opt->weight_mode; m.has_saliency = saliency != nullptr;
  m.eigenvalue_floor = opt->eigenvalue_floor;
  m.V = static_cast<const double2*>(eigenvectors); m.lam = eigenvalues;
  m.gV = static_cast<const double2*>(grad_eigenvectors); m.glam = grad_eigenvalues; m.gw = grad_weight;
  m.gpsi = ws.gpsi; m.gS = ws.gS;
  if ((r = launch_bwd("cacgmm_mstep_spec_bwd_kernel", cacgmm_mstep_spec_bwd_kernel, dim3(F, K), 32,
                      mstep_spec_bwd_smem(D), m, st)))
    return r;
  MstepBwdArgs b;
  b.y = y; b.F = F; b.T = T; b.D = D; b.K = K; b.nch = bwd_chunks(T);
  b.aff = affiliation; b.q = quadratic; b.saliency = saliency; b.gpsi = ws.gpsi; b.gS = ws.gS;
  b.gaff = grad_affiliation; b.gq = grad_quadratic; b.gsal = grad_saliency; b.ybar = static_cast<double2*>(grad_y);
  return with_ct(dtype, [&](auto ct) {
    return launch_bwd("cacgmm_mstep_bwd_kernel", cacgmm_mstep_bwd_kernel<decltype(ct)>, dim3(F, b.nch), kBwdFrames,
                      bwd_frame_smem(D, 0), b, st);
  });
}

size_t pbb_cwmm_workspace_bytes(int F, int T, int D, int K) { return pbb_cacgmm_workspace_bytes(F, T, D, K); }

int pbb_cwmm_fit(const void* y, int dtype, int F, int T, int D, int K, const double* init_aff,
                 const double* saliency, int iterations, int weight_mode, const double* spline_t,
                 const double* spline_c, int spline_n, double max_concentration, void* mode,
                 double* concentration, double* weight, void* workspace, size_t workspace_bytes, int* status,
                 void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(init_aff != nullptr, 7, "initial affiliations are null (cwmm.py:121-127)");
  PBB_CHECK_ARG(iterations > 0, 9, "iterations must be positive");
  PBB_CHECK_ARG(weight_mode == PBB_WEIGHT_TIME || weight_mode == PBB_WEIGHT_CONST, 10, "bad weight_mode");
  PBB_CHECK_ARG(spline_t && spline_c && spline_n >= 3, 11, "spline table is missing");
  PBB_CHECK_ARG(mode && concentration && weight, 15, "model output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool persistent = fast_shape(D, K) && saliency == nullptr;
  CacgmmWorkspace ws;
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 18,
                      "workspace too small (pbb_cwmm_workspace_bytes)", status,
                      persistent ? Layout::kStaged : Layout::kPlain, st, &ws)))
    return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.model_kind = 1;
  a.w = weight;
  a.saliency = saliency;
  CwUpdArgs u;
  memset(&u, 0, sizeof(u));
  u.F = F; u.T = T; u.D = D; u.K = K;
  u.part = ws.part; u.weight_mode = weight_mode;
  u.spline.t = spline_t; u.spline.c = spline_c; u.spline.n = spline_n;
  u.spline.max_concentration = max_concentration;
  // (the domain of the interpolant -- first and last knot -- is read from the table on the device)
  u.mode = reinterpret_cast<double2*>(mode); u.concentration = concentration; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.ew = ws.ew; u.status = status;
  if (persistent) {
    // every EM iteration in one launch (em_persistent.cuh, MODEL = 1); the last iteration's raw
    // scatter sums go through cw_update_kernel for the reference-exact mode / concentration / weight
    PBB_CUDA(cudaMemsetAsync(ws.flags, 0, ws.control_bytes, st));
    PersistArgs p = persist_args(ws, F, T, iterations, status);
    p.first_is_m = 1;
    p.aff_in = init_aff; p.weight_mode = weight_mode;
    p.spline = u.spline;
    if ((r = launch_planned(p, ws, D, K, dtype, Persist::kCw, false, st))) return r;
#ifdef PBB_PHASE_TIMING
    print_phases(ws, (long long)F * iterations, true, st);
#endif
    u.nch = 1;
    return launch_update(cw_update_kernel, "cw_update_kernel", u, st);
  }
  for (int it = 0; it < iterations; ++it) {
    if (it == 0) { a.mode = kModeM; a.aff_in = init_aff; a.q_in = nullptr; }
    else { a.mode = kModeEM; a.aff_in = nullptr; }
    int nch = launch_em(a, dtype, 0, st);
    if (nch <= 0) return nch ? nch : 1;
    u.nch = nch;
    if ((r = launch_update(cw_update_kernel, "cw_update_kernel", u, st))) return r;
  }
  return 0;
}

int pbb_cwmm_predict(const void* y, int dtype, int F, int T, int D, int K, const void* mode,
                     const double* concentration, const double* weight, int weight_mode, double* affiliation,
                     void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(mode && concentration, 7, "model is null");
  PBB_CHECK_ARG(weight_mode >= 0 && weight_mode <= PBB_WEIGHT_TIED, 10, "bad weight_mode");
  PBB_CHECK_ARG(weight != nullptr || weight_mode == PBB_WEIGHT_CONST, 9, "weight is null");
  PBB_CHECK_ARG(affiliation != nullptr, 11, "affiliation output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws;
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 12,
                      "workspace too small (pbb_cwmm_workspace_bytes)", status, Layout::kPlain, st, &ws)))
    return r;
  CwFromModelArgs fm;
  fm.F = F; fm.D = D; fm.K = K;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  fm.mode = reinterpret_cast<const double2*>(mode); fm.concentration = concentration;
  fm.weight = (tied || weight_mode == PBB_WEIGHT_CONST) ? nullptr : weight;
  fm.coef = ws.coef; fm.ld = ws.ld; fm.ew = ws.ew; fm.w = ws.w;
  if ((r = launch_kernel("cw_from_model_kernel", cw_from_model_kernel, F, 128, (size_t)D * D * sizeof(int), st, fm)))
    return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.mode = kModeE; a.model_kind = 1;
  if (tied) { a.w_time = weight; a.w_time_st = weight_mode == PBB_WEIGHT_TIED_TIME ? 1 : 0; }
  a.aff_out = affiliation;
  int nch = launch_em(a, dtype, 0, st);
  return nch > 0 ? 0 : (nch ? nch : 1);
}

size_t pbb_cbmm_workspace_bytes(int F, int T, int D, int K) { return pbb_cacgmm_workspace_bytes(F, T, D, K); }

int pbb_cbmm_fit(const void* y, int dtype, int F, int T, int D, int K, const double* init_aff,
                 const double* saliency, int iterations, int weight_mode, double affiliation_eps,
                 double eigenvalue_eps, double max_concentration, void* eigenvectors, double* eigenvalues,
                 double* weight, void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_cbmm_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(init_aff != nullptr, 7, "initial affiliations are null (cbmm.py:120-126)");
  PBB_CHECK_ARG(iterations > 0, 9, "iterations must be positive");
  PBB_CHECK_ARG(weight_mode == PBB_WEIGHT_TIME || weight_mode == PBB_WEIGHT_CONST, 10, "bad weight_mode");
  PBB_CHECK_ARG(affiliation_eps >= 0.0 && affiliation_eps < 0.5, 11, "need 0 <= affiliation_eps < 0.5");
  PBB_CHECK_ARG(max_concentration > 0.0, 13, "max_concentration must be positive (complex_bingham.py:221)");
  PBB_CHECK_ARG(eigenvectors && eigenvalues && weight, 14, "model output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws;
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 17,
                      "workspace too small (pbb_cbmm_workspace_bytes)", status, Layout::kPlain, st, &ws)))
    return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.model_kind = 1;  // lp = ew q - ld with ew = -1, q = y^H (-B) y
  a.w = weight;
  a.saliency = saliency; a.aff_eps = affiliation_eps;
  CbUpdArgs u;
  memset(&u, 0, sizeof(u));
  u.F = F; u.T = T; u.K = K;
  u.part = ws.part; u.weight_mode = weight_mode;
  u.eigenvalue_eps = eigenvalue_eps; u.max_concentration = max_concentration;
  u.evec = reinterpret_cast<double2*>(eigenvectors); u.eval = eigenvalues; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.ew = ws.ew; u.status = status;
  for (int it = 0; it < iterations; ++it) {
    // iteration 0: M-step from the initial affiliations; then E-step (predict) + M-step (cbmm.py:186-203)
    if (it == 0) { a.mode = kModeM; a.aff_in = init_aff; a.q_in = nullptr; }
    else { a.mode = kModeEM; a.aff_in = nullptr; }
    const int nch = launch_em(a, dtype, 0, st);
    if (nch <= 0) return nch ? nch : 1;
    u.nch = nch;
    u.coef = it + 1 < iterations ? ws.coef : nullptr;  // nobody reads the E-step form of the final model
    if ((r = with_bingham_d(D, [&](auto d) {
           return launch_kernel("cb_update_kernel", cb_update_kernel<decltype(d)::value>, u.F, 32 * kCbWarps, 0, st,
                                u);
         })))
      return r;
  }
  return 0;
}

int pbb_cbmm_predict(const void* y, int dtype, int F, int T, int D, int K, const void* eigenvectors,
                     const double* eigenvalues, const double* weight, int weight_mode, double affiliation_eps,
                     double* affiliation, void* workspace, size_t workspace_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  if (int r = check_cbmm_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(eigenvectors && eigenvalues, 7, "model is null");
  PBB_CHECK_ARG(weight != nullptr || weight_mode == PBB_WEIGHT_CONST, 9, "weight is null");
  PBB_CHECK_ARG(weight_mode >= 0 && weight_mode <= PBB_WEIGHT_TIED, 10, "bad weight_mode");
  PBB_CHECK_ARG(affiliation_eps >= 0.0 && affiliation_eps < 0.5, 11, "need 0 <= affiliation_eps < 0.5");
  PBB_CHECK_ARG(affiliation != nullptr, 12, "affiliation output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws;
  int r;
  if ((r = begin_call(y, dtype, F, T, D, K, workspace, workspace_bytes, 13,
                      "workspace too small (pbb_cbmm_workspace_bytes)", status, Layout::kPlain, st, &ws)))
    return r;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  CbFromModelArgs fm;
  fm.F = F; fm.K = K;
  fm.evec = reinterpret_cast<const double2*>(eigenvectors); fm.eval = eigenvalues;
  fm.weight = (tied || weight_mode == PBB_WEIGHT_CONST) ? nullptr : weight;
  fm.coef = ws.coef; fm.ld = ws.ld; fm.ew = ws.ew; fm.w = ws.w;
  if ((r = with_bingham_d(D, [&](auto d) {
         return launch_kernel("cb_from_model_kernel", cb_from_model_kernel<decltype(d)::value>, F, 32 * kCbWarps, 0,
                              st, fm);
       })))
    return r;
  EmArgs a = em_args(ws, F, T, D, K);
  a.mode = kModeE; a.model_kind = 1;
  if (tied) { a.w_time = weight; a.w_time_st = weight_mode == PBB_WEIGHT_TIED_TIME ? 1 : 0; }
  a.aff_eps = affiliation_eps;
  a.aff_out = affiliation;
  const int nch = launch_em(a, dtype, 0, st);
  return nch > 0 ? 0 : (nch ? nch : 1);
}

int pbb_bingham_parameters(const double* scatter_eigenvalues, int n, int D, double eps, double max_concentration,
                           double* eigenvalues, int* status, void* stream) {
  PBB_CHECK_ARG(scatter_eigenvalues != nullptr, 1, "scatter eigenvalues are null");
  PBB_CHECK_ARG(n > 0 && n <= kCbMaxIndex, 2, "need 0 < n < 2^29");
  PBB_CHECK_ARG(D >= 2 && D <= 6, 3, "complex Bingham: need 2 <= D <= 6 (complex_bingham_utils.py:342-348)");
  PBB_CHECK_ARG(max_concentration > 0.0, 5, "max_concentration must be positive (complex_bingham.py:221)");
  PBB_CHECK_ARG(eigenvalues != nullptr, 6, "output is null");
  PBB_CHECK_ARG(status != nullptr, 7, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  return with_bingham_d(D, [&](auto d) {
    return launch_kernel("bingham_parameters_kernel", bingham_parameters_kernel<decltype(d)::value>, (n + 3) / 4, 128,
                         0, st, scatter_eigenvalues, n, eps, max_concentration, eigenvalues, status);
  });
}

int pbb_bingham_log_norm(const double* eigenvalues, int n, int D, double eps, double* log_norm, void* stream) {
  PBB_CHECK_ARG(eigenvalues != nullptr, 1, "eigenvalues are null");
  PBB_CHECK_ARG(n > 0, 2, "n must be positive");
  PBB_CHECK_ARG(D >= 2 && D <= 6, 3, "complex Bingham: need 2 <= D <= 6 (complex_bingham_utils.py:342-348)");
  PBB_CHECK_ARG(log_norm != nullptr, 5, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_bingham_d(D, [&](auto d) {
    return launch_kernel("bingham_log_norm_kernel", bingham_log_norm_kernel<decltype(d)::value>, (n + 127) / 128, 128,
                         0, st, eigenvalues, n, eps, log_norm);
  });
}

int pbb_bingham_log_pdf(const void* y, int dtype, int M, int T, int D, const void* eigenvectors,
                        const double* eigenvalues, const double* log_norm, double* log_pdf, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(M > 0 && T > 0, 3, "empty shape");
  PBB_CHECK_ARG(D >= 1 && D < 256, 5, "bad D");
  PBB_CHECK_ARG(eigenvectors != nullptr && eigenvalues != nullptr && log_norm != nullptr, 6, "model is null");
  PBB_CHECK_ARG(log_pdf != nullptr, 9, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long n = (long long)M * T;
  const unsigned blocks = (unsigned)((n + 127) / 128);
  const double2* V = static_cast<const double2*>(eigenvectors);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("bingham_log_pdf_kernel", bingham_log_pdf_kernel<CT>, blocks, 128, 0, st,
                         static_cast<const CT*>(y), V, eigenvalues, log_norm, M, T, D, log_pdf);
  });
}

}  // extern "C"
