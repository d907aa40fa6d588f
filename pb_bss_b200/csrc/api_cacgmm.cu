// C-ABI entry points for the cACGMM EM path (see include/pbb.h).
#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include <cuda.h>

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

// out[k][t] = mean over f of aff[f][k][t]   (estimate_mixture_weight, axis -3)
__global__ void mean_over_bins_kernel(const double* __restrict__ aff, int F, int K, int T, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= K * T) return;
  double s = 0.0;
  for (int f = 0; f < F; ++f) s += aff[(size_t)f * K * T + i];
  out[i] = s / (double)F;
}
// out[k] = mean over t of in[k][t]
__global__ void mean_over_time_kernel(const double* __restrict__ in, int K, int T, double* __restrict__ out) {
  const int k = blockIdx.x;
  __shared__ double red[32];
  double s = 0.0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) s += in[(size_t)k * T + t];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
    out[k] = tot / (double)T;
  }
}

// w[k][t] /= sum_k |w[k][t]|  (a zero norm counts as 1e-10)
__global__ void unit_norm_over_classes_kernel(double* __restrict__ w, int K, int T) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double n = 0.0;
  for (int k = 0; k < K; ++k) n += fabs(w[(size_t)k * T + t]);
  if (n == 0.0) n = 1e-10;
  for (int k = 0; k < K; ++k) w[(size_t)k * T + t] /= n;
}

// ---- workspace carving -------------------------------------------------------
struct CacgmmWorkspace {
  void* z;
  int zs;       // padded row stride of z (frames)
  int* flags;   // (F) per-bin model version, persistent kernel
  int* ticket;  // (1)
  unsigned long long* phase;  // (16) debug phase counters
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
  const size_t z_staged = (size_t)F * nchunks * stage_rows(D % 2 == 0 ? D : D + 1) * kStageFrames * sizeof(double2);
  const size_t o_z = take(z_plain > z_staged ? z_plain : z_staged);
  const size_t o_flags = take((size_t)(F + 1) * sizeof(int) + 16 * sizeof(unsigned long long) + 8);
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
  ws.dead = reinterpret_cast<int*>(b + o_dead);
  ws.phase = reinterpret_cast<unsigned long long*>(b + o_flags + (((size_t)(F + 1) * sizeof(int) + 7) / 8) * 8);
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
// Parts a bin-iteration is split into (pure host logic, unit-tested through pbb_em_dispatch).  force > 0 overrides
// the choice (PBB_TSPLIT); the result always satisfies 1 <= S <= nchunks and S + 1 <= max_chunks(T).
static int choose_frame_split(int F, int T, int D, int K, int ctas_per_sm, int sms, int force) {
  const int zs = (T + 31) / 32 * 32;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  const long long slots = (long long)ctas_per_sm * sms;
  int S = 1;
  // a part must keep enough of the sweep to pay for the extra L2 round trip (partials out, counter, partials in,
  // ~3 us): measured break-even around T D^2 (K + 1) / S ~ 2.4e4 (C1, D = 4, T = 200 loses 10 % with S = 2;
  // D = 8, T = 500 gains 12 % with S = 4)
  const long long sweep = (long long)T * D * D * (K + 1);
  while (S < 4 && 2 * S <= nchunks && (long long)F * 2 * S <= slots && sweep >= 24000LL * 2 * S) S *= 2;
  if (force > 0) S = force;
  if (S > nchunks) S = nchunks;
  if (S + 1 > max_chunks(T)) S = 1;
  return S < 1 ? 1 : S;
}
// Cluster size of the sticky-bins kernel (em_sticky.cuh), 0 = not applicable: the largest of 4, 2, 1 whose parts fit
// the ring (ceil(nchunks / S) <= kWsStages), that leaves every part a stage and whose F clusters run at once:
// F <= clusters[i] for S = 1 << i.  Clusters of 4 are placed within a GPC, so on an H100 (132 SMs in GPCs of uneven
// size) fewer of them fit than 2 x SMs / 4; a second wave would double the fit time.  force: -1 automatic, S > 0
// only that size (PBB_STICKY).
static int choose_sticky(int F, int T, const int clusters[3], int force) {
  const int zs = (T + 31) / 32 * 32;
  const int nchunks = (zs + kStageFrames - 1) / kStageFrames;
  for (int c = 4, i = 2; c >= 1; c /= 2, --i) {
    if (force > 0 && c != force) continue;
    if (c > nchunks || (nchunks + c - 1) / c > kWsStages) continue;
    if (F > clusters[i]) continue;
    return c;
  }
  return 0;
}

// Persistent kernels of a fit, numbered as pbb_em_dispatch reports them (pbb.h).
enum { kKernelWs = 0, kKernelSticky = 1, kKernelSingle = 2 };

// Tuning overrides of the kernel choice (environment of pbb_cacgmm_fit).
struct PlanOverrides {
  int tsplit = 0;       // > 0: frame split into that many parts (PBB_TSPLIT)
  int sticky = -1;      // sticky-bins cluster size: -1 automatic, 0 off, S > 0 only S (PBB_STICKY)
  bool single = false;  // single-role kernel only (PBB_EM_KERNEL=single; the complex Watson fit has no other)
};

struct FitPlan {
  int kernel;  // kKernel*
  int split;   // sticky: CTAs per cluster; otherwise parts per bin-iteration (1 = no frame split)
};

static PlanOverrides env_overrides() {
  static const bool single = [] {
    const char* e = getenv("PBB_EM_KERNEL");
    return e != nullptr && !strcmp(e, "single");
  }();
  PlanOverrides o;
  o.single = single;
  if (const char* e = getenv("PBB_TSPLIT")) o.tsplit = atoi(e);
  if (const char* e = getenv("PBB_STICKY")) o.sticky = atoi(e);
  return o;
}

// The sticky-bins kernel exists for the lean D = 8 fit of device-resident input.
static bool sticky_eligible(int D, bool lean, bool streamed, const PlanOverrides& o) {
  return D == 8 && lean && !streamed && !o.single && o.sticky != 0;
}

// Which persistent kernel a fit runs and how it splits a bin-iteration (pure host logic).  sms: SMs of the device;
// clusters: sticky-kernel clusters of 1, 2, 4 CTAs the device runs at once, read only when sticky_eligible.
static FitPlan plan_persistent_fit(int F, int T, int D, int K, bool lean, bool streamed, int sms,
                                   const int* clusters, const PlanOverrides& o) {
  if (sticky_eligible(D, lean, streamed, o)) {
    const int S = choose_sticky(F, T, clusters, o.sticky);
    if (S > 0) return {kKernelSticky, S};
  }
  const int kernel = D == 8 && lean && !o.single ? kKernelWs : kKernelSingle;
  return {kernel, choose_frame_split(F, T, D, K, persist_ctas_per_sm(D, !lean), sms, o.tsplit)};
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

// ---- launches ------------------------------------------------------------------
template <typename CT>
static int launch_normalize(const void* y, void* z, int F, int T, int D, int swap, int zs, cudaStream_t st) {
  const int block = D <= 16 ? 128 : 32;
  dim3 grid((T + block - 1) / block, F);
  const size_t smem = (size_t)block * (D + 1) * sizeof(double2);
  LaunchScope ls("normalize_kernel", st);
  normalize_kernel<CT><<<grid, block, smem, st>>>(reinterpret_cast<const CT*>(y), reinterpret_cast<CT*>(z), F, T,
                                                    D, swap, zs);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

template <typename CT>
static int launch_normalize_staged(const void* y, void* z, int F, int T, int D, int* dead, cudaStream_t st) {
  if (dead != nullptr) PBB_CUDA(cudaMemsetAsync(dead, 0, (size_t)F * sizeof(int), st));
  const int block = 64;  // divides kStageFrames
  const int nchunks = (((T + 31) / 32 * 32) + kStageFrames - 1) / kStageFrames;
  dim3 grid(nchunks * (kStageFrames / block), F);
  const size_t smem = (size_t)block * (D + 1) * sizeof(double2);
  LaunchScope ls("normalize_staged_kernel", st);
  normalize_staged_kernel<CT><<<grid, block, smem, st>>>(reinterpret_cast<const CT*>(y), reinterpret_cast<CT*>(z), F, T, D,
                                                          stage_rows(D), kStageFrames, nchunks, dead);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

static bool fast_shape(int D, int K) { return (D == 4 || D == 6 || D == 8) && K >= 2 && K <= 4; }

template <int D, int K>
static cudaError_t launch_fast_dk(const EmArgs& a, int dtype, cudaStream_t st) {
  dim3 grid(a.nch, a.F);
  LaunchScope ls("em_fast_kernel", st);
  if (dtype == PBB_C128) em_fast_kernel<D, K, double2><<<grid, 32 * kEmGroups, 0, st>>>(a);
  else em_fast_kernel<D, K, float2><<<grid, 32 * kEmGroups, 0, st>>>(a);
  return cudaGetLastError();
}

template <int D>
static cudaError_t launch_fast_d(const EmArgs& a, int dtype, cudaStream_t st) {
  switch (a.K) {
    case 2: return launch_fast_dk<D, 2>(a, dtype, st);
    case 3: return launch_fast_dk<D, 3>(a, dtype, st);
    default: return launch_fast_dk<D, 4>(a, dtype, st);
  }
}

// Fills nch / frames_per_block and launches the EM kernel for the shape.
int launch_em(EmArgs a, int dtype, int frames_per_block, cudaStream_t st) {
  if (fast_shape(a.D, a.K)) {
    int fpb = frames_per_block > 0 ? frames_per_block : 128;
    fpb = (fpb + 31) / 32 * 32;
    if (fpb > (a.T + 31) / 32 * 32) fpb = (a.T + 31) / 32 * 32;
    a.frames_per_block = fpb;
    a.nch = (a.T + fpb - 1) / fpb;
    cudaError_t e;
    switch (a.D) {
      case 4: e = launch_fast_d<4>(a, dtype, st); break;
      case 6: e = launch_fast_d<6>(a, dtype, st); break;
      default: e = launch_fast_d<8>(a, dtype, st); break;
    }
    PBB_CUDA(e);
    return a.nch;
  }
  a.frames_per_block = kGenFrames;
  a.nch = (a.T + kGenFrames - 1) / kGenFrames;
  a.softmax_fast = 0;
  dim3 grid(a.nch, a.F);
  const size_t smem = (size_t)2 * a.K * kGenFrames * sizeof(double) + (size_t)a.D * a.D * sizeof(int);
  LaunchScope ls("em_generic_kernel", st);
  if (dtype == PBB_C128) {
    PBB_CUDA(cudaFuncSetAttribute(em_generic_kernel<double2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    em_generic_kernel<double2><<<grid, kGenFrames, smem, st>>>(a);
  } else {
    PBB_CUDA(cudaFuncSetAttribute(em_generic_kernel<float2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    em_generic_kernel<float2><<<grid, kGenFrames, smem, st>>>(a);
  }
  PBB_CUDA(cudaGetLastError());
  return a.nch;
}

static int update_warps(int D, int K) {
  const size_t per = update_smem_per_warp(D);
  int w = (int)((size_t)(200 * 1024) / per);
  if (w > K) w = K;
  if (w > 16) w = 16;
  if (w < 1) w = 1;
  return w;
}

static int launch_update(UpdArgs u, cudaStream_t st) {
  u.warps = update_warps(u.D, u.K);
  const size_t smem = update_smem_per_warp(u.D) * u.warps + (size_t)2 * u.K * sizeof(double) +
                      (size_t)u.D * u.D * sizeof(int);
  PBB_CUDA(cudaFuncSetAttribute(cacg_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  const int threads = 32 * u.warps < u.K ? ((u.K + 31) / 32 * 32) : 32 * u.warps;
  LaunchScope ls("cacg_update_kernel", st);
  cacg_update_kernel<<<u.F, threads, smem, st>>>(u);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

static int launch_from_eig(FromEigArgs u, cudaStream_t st) {
  const size_t per = from_eig_smem_per_warp(u.D);
  int w = (int)((size_t)(200 * 1024) / per);
  if (w > u.K) w = u.K;
  if (w > 16) w = 16;
  u.warps = w;
  const size_t smem = per * w + (size_t)u.K * sizeof(double) + (size_t)u.D * u.D * sizeof(int);
  PBB_CUDA(cudaFuncSetAttribute(cacg_from_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  const int threads = 32 * w < u.K ? ((u.K + 31) / 32 * 32) : 32 * w;
  LaunchScope ls("cacg_from_eig_kernel", st);
  cacg_from_eig_kernel<<<u.F, threads, smem, st>>>(u);
  PBB_CUDA(cudaGetLastError());
  return 0;
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

// device-usable address of a pinned host allocation, nullptr for device memory, error otherwise
static int classify_pointer(const void* p, const void** dev_alias, bool* is_host, const char* what) {
  cudaPointerAttributes at;
  PBB_CUDA(cudaPointerGetAttributes(&at, p));
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) {
    *is_host = false;
    *dev_alias = p;
    return 0;
  }
  if (at.type == cudaMemoryTypeHost && at.devicePointer != nullptr) {
    *is_host = true;
    *dev_alias = at.devicePointer;
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

template <typename CT>
static int launch_stream_load(const void* y, void* z, const double* aff_src, double* aff_dst, int F, int T, int D, int K,
                              int* dead, int* flags, int* next_bin, int* started, int* ctas_out, cudaStream_t st) {
  const int nchunks = (((T + 31) / 32 * 32) + kStageFrames - 1) / kStageFrames;
  const size_t smem = (size_t)kStageFrames * (D + 1) * sizeof(double2);
  LaunchScope ls("stream_load_kernel", st);
  int ctas = kLoadCtas;
  if (const char* e = getenv("PBB_LOAD_CTAS")) ctas = atoi(e) > 0 ? atoi(e) : ctas;  // tuning override
  ctas = ctas < F ? ctas : F;
  *ctas_out = ctas;
  stream_load_kernel<CT><<<ctas, kLoadThreads, smem, st>>>(
      reinterpret_cast<const CT*>(y), reinterpret_cast<CT*>(z), aff_src, aff_dst, F, T, D, K,
      stage_rows(D), kStageFrames, nchunks, dead, flags, next_bin, started);
  PBB_CUDA(cudaGetLastError());
  return 0;
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
  int dev = 0, sms = 0;
  PBB_CUDA(cudaGetDevice(&dev));
  PBB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  long long grid = (long long)(*cache) * sms - reserve;
  if (grid < 1) grid = 1;
  const long long tasks = (long long)a.iterations * a.F * (a.tsplit > 1 ? a.tsplit : 1);
  if (grid > tasks) grid = tasks;
  LaunchScope ls(name, st);
  kern<<<(unsigned)grid, threads, smem, st>>>(a);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

// full = saliency / activity mask / log-domain softmax; lean = product-form softmax, 2 frames per lane;
// ws = the warp-specialised em_ws_kernel (D = 8, lean) instead of the single-role kernel
template <int D, int K, typename CT>
static int launch_persist_t(const PersistArgs& a, bool full, bool ws, cudaStream_t st) {
  static int cache_full = 0, cache_lean = 0;
  if (full)
    return launch_persistent_generic(em_persistent_kernel<D, K, CT, true, 1>, persist_threads(D, K),
                                     sizeof(PersistSmem<D, K, CT>), &cache_full, a, "em_persistent_kernel", st);
  if constexpr (D == 8) {
    static int cache_ws = 0;
    if (ws)
      return launch_persistent_generic(em_ws_kernel<K, CT>, 256, sizeof(WsSmem<D, K, CT>), &cache_ws, a,
                                       "em_ws_kernel", st);
  }
  return launch_persistent_generic(em_persistent_kernel<D, K, CT, false, 2>, persist_threads(D, K),
                                   sizeof(PersistSmem<D, K, CT>), &cache_lean, a, "em_persistent_kernel", st);
}

// complex Watson EM on the persistent kernel (lean structure, MODEL = 1)
template <int D, int K, typename CT>
static int launch_persist_cw_t(const PersistArgs& a, cudaStream_t st) {
  static int cache = 0;
  return launch_persistent_generic(em_persistent_kernel<D, K, CT, false, 2, 1>, persist_threads(D, K),
                                   sizeof(PersistSmem<D, K, CT>), &cache, a, "em_persistent_kernel_cw", st);
}
template <int D>
static int launch_persist_cw_d(const PersistArgs& a, int K, int dtype, cudaStream_t st) {
  const bool c128 = dtype == PBB_C128;
  switch (K) {
    case 2: return c128 ? launch_persist_cw_t<D, 2, double2>(a, st) : launch_persist_cw_t<D, 2, float2>(a, st);
    case 3: return c128 ? launch_persist_cw_t<D, 3, double2>(a, st) : launch_persist_cw_t<D, 3, float2>(a, st);
    default: return c128 ? launch_persist_cw_t<D, 4, double2>(a, st) : launch_persist_cw_t<D, 4, float2>(a, st);
  }
}
static int launch_persist_cw(const PersistArgs& a, int D, int K, int dtype, cudaStream_t st) {
  switch (D) {
    case 4: return launch_persist_cw_d<4>(a, K, dtype, st);
    case 6: return launch_persist_cw_d<6>(a, K, dtype, st);
    default: return launch_persist_cw_d<8>(a, K, dtype, st);
  }
}

template <int D, int K>
static int launch_persist_dk(const PersistArgs& a, int dtype, bool full, bool ws, cudaStream_t st) {
  if (dtype == PBB_C128) return launch_persist_t<D, K, double2>(a, full, ws, st);
  return launch_persist_t<D, K, float2>(a, full, ws, st);
}

template <int D>
static int launch_persist_d(const PersistArgs& a, int K, int dtype, bool full, bool ws, cudaStream_t st) {
  switch (K) {
    case 2: return launch_persist_dk<D, 2>(a, dtype, full, ws, st);
    case 3: return launch_persist_dk<D, 3>(a, dtype, full, ws, st);
    default: return launch_persist_dk<D, 4>(a, dtype, full, ws, st);
  }
}

// "Sticky bins" (em_sticky.cuh): when the device runs F clusters of S CTAs at once, a cluster keeps one bin for the
// whole fit (choose_sticky).  PBB_STICKY=0 disables it, PBB_STICKY=S forces a cluster size (A/B).
static void sticky_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, unsigned ctas, int S, size_t smem,
                          cudaStream_t st) {
  memset(cfg, 0, sizeof(*cfg));
  cfg->gridDim = dim3(ctas);
  cfg->blockDim = dim3(256);
  cfg->dynamicSmemBytes = smem;
  cfg->stream = st;
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = (unsigned)S;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  cfg->attrs = attr;
  cfg->numAttrs = 1;
}
// clusters of 1, 2, 4 CTAs of em_sticky_kernel the device runs at once (queried once per instantiation)
template <int K, typename CT>
static int sticky_clusters_t(int clusters[3], cudaStream_t st) {
  static int cache[3] = {-1, -1, -1};
  if (cache[0] < 0) {
    const size_t smem = sizeof(WsSmem<8, K, CT>);
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    PBB_CUDA(cudaFuncSetAttribute(em_sticky_kernel<K, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int i = 0; i < 3; ++i) {
      sticky_config(&cfg, attr, 1u << i, 1 << i, smem, st);
      int n = 0;
      PBB_CUDA(cudaOccupancyMaxActiveClusters(&n, em_sticky_kernel<K, CT>, &cfg));
      cache[i] = n;
    }
  }
  for (int i = 0; i < 3; ++i) clusters[i] = cache[i];
  return 0;
}
static int sticky_clusters(int K, int dtype, int clusters[3], cudaStream_t st) {
  const bool c128 = dtype == PBB_C128;
  switch (K) {
    case 2: return c128 ? sticky_clusters_t<2, double2>(clusters, st) : sticky_clusters_t<2, float2>(clusters, st);
    case 3: return c128 ? sticky_clusters_t<3, double2>(clusters, st) : sticky_clusters_t<3, float2>(clusters, st);
    default: return c128 ? sticky_clusters_t<4, double2>(clusters, st) : sticky_clusters_t<4, float2>(clusters, st);
  }
}

// one cluster of S CTAs per bin; sticky_clusters has set the kernel's shared-memory limit
template <int K, typename CT>
static int launch_sticky_t(const PersistArgs& a, int S, cudaStream_t st) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  sticky_config(&cfg, attr, (unsigned)(a.F * S), S, sizeof(WsSmem<8, K, CT>), st);
  LaunchScope ls("em_sticky_kernel", st);
  PBB_CUDA(cudaLaunchKernelEx(&cfg, em_sticky_kernel<K, CT>, a));
  return 0;
}
static int launch_sticky(const PersistArgs& a, int K, int dtype, int S, cudaStream_t st) {
  const bool c128 = dtype == PBB_C128;
  switch (K) {
    case 2: return c128 ? launch_sticky_t<2, double2>(a, S, st) : launch_sticky_t<2, float2>(a, S, st);
    case 3: return c128 ? launch_sticky_t<3, double2>(a, S, st) : launch_sticky_t<3, float2>(a, S, st);
    default: return c128 ? launch_sticky_t<4, double2>(a, S, st) : launch_sticky_t<4, float2>(a, S, st);
  }
}

static int launch_persist(const PersistArgs& a, int D, int K, int dtype, bool full, bool ws, cudaStream_t st) {
  switch (D) {
    case 4: return launch_persist_d<4>(a, K, dtype, full, ws, st);
    case 6: return launch_persist_d<6>(a, K, dtype, full, ws, st);
    default: return launch_persist_d<8>(a, K, dtype, full, ws, st);
  }
}

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

static int launch_cw_update(CwUpdArgs u, cudaStream_t st) {
  u.warps = update_warps(u.D, u.K);
  const size_t smem = update_smem_per_warp(u.D) * u.warps + (size_t)2 * u.K * sizeof(double) +
                      (size_t)u.D * u.D * sizeof(int);
  PBB_CUDA(cudaFuncSetAttribute(cw_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  const int threads = 32 * u.warps < u.K ? ((u.K + 31) / 32 * 32) : 32 * u.warps;
  LaunchScope ls("cw_update_kernel", st);
  cw_update_kernel<<<u.F, threads, smem, st>>>(u);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

// complex Bingham kernels are instantiated for D = 2..6, the reference's domain (complex_bingham_utils.py:342-348)
template <template <int> class Launch, typename... Args>
static int bingham_dispatch(int D, Args... args) {
  switch (D) {
    case 2: return Launch<2>::run(args...);
    case 3: return Launch<3>::run(args...);
    case 4: return Launch<4>::run(args...);
    case 5: return Launch<5>::run(args...);
    case 6: return Launch<6>::run(args...);
    default: set_error("complex Bingham: D = %d, need 2 <= D <= 6", D); return -5;
  }
}
template <int D> struct CbUpdateLaunch {
  static int run(CbUpdArgs u, cudaStream_t st) {
    LaunchScope ls("cb_update_kernel", st);
    cb_update_kernel<D><<<u.F, 32 * kCbWarps, 0, st>>>(u);
    PBB_CUDA(cudaGetLastError());
    return 0;
  }
};
template <int D> struct CbFromModelLaunch {
  static int run(CbFromModelArgs u, cudaStream_t st) {
    LaunchScope ls("cb_from_model_kernel", st);
    cb_from_model_kernel<D><<<u.F, 32 * kCbWarps, 0, st>>>(u);
    PBB_CUDA(cudaGetLastError());
    return 0;
  }
};
template <int D> struct BinghamParametersLaunch {
  static int run(const double* s, int n, double eps, double mc, double* lam, int* status, cudaStream_t st) {
    LaunchScope ls("bingham_parameters_kernel", st);
    bingham_parameters_kernel<D><<<(n + 3) / 4, 128, 0, st>>>(s, n, eps, mc, lam, status);
    PBB_CUDA(cudaGetLastError());
    return 0;
  }
};
template <int D> struct BinghamLogNormLaunch {
  static int run(const double* lam, int n, double eps, double* out, cudaStream_t st) {
    LaunchScope ls("bingham_log_norm_kernel", st);
    bingham_log_norm_kernel<D><<<(n + 127) / 128, 128, 0, st>>>(lam, n, eps, out);
    PBB_CUDA(cudaGetLastError());
    return 0;
  }
};

static int check_cbmm_shape(int F, int T, int D, int K, int dtype) {
  if (int r = check_shape(F, T, D, K, dtype)) return r;
  PBB_CHECK_ARG(D >= 2 && D <= 6, 5, "complex Bingham: need 2 <= D <= 6 (complex_bingham_utils.py:342-348)");
  PBB_CHECK_ARG((long long)F * K <= kCbMaxIndex, 6, "F * K too large for the status word");
  return 0;
}

}  // namespace pbb

using namespace pbb;

extern "C" {

const char* pbb_last_error(void) { return g_err; }
int pbb_version(void) { return 100; }

int pbb_normalize_observation(const void* y, void* z, int F, int T, int D, int dtype, int swap, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(z != nullptr, 2, "z is null");
  PBB_CHECK_ARG(F > 0 && T > 0, 3, "empty shape");
  PBB_CHECK_ARG(D > 0 && D < 256, 5, "bad D");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 6, "bad dtype");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return dtype == PBB_C128 ? launch_normalize<double2>(y, z, F, T, D, swap, T, st)
                           : launch_normalize<float2>(y, z, F, T, D, swap, T, st);
}

int pbb_em_dispatch(int F, int T, int D, int K, int lean, int streamed, int sms, int* kernel, int* split) {
  PBB_CHECK_ARG(F > 0, 1, "F must be positive");
  PBB_CHECK_ARG(T > 0, 2, "T must be positive");
  PBB_CHECK_ARG(D == 4 || D == 6 || D == 8, 3, "persistent kernels: D in {4, 6, 8}");
  PBB_CHECK_ARG(K >= 2 && K <= 4, 4, "persistent kernels: K in {2, 3, 4}");
  PBB_CHECK_ARG(sms > 0, 7, "sms must be positive");
  PBB_CHECK_ARG(kernel != nullptr && split != nullptr, 8, "output is null");
  const int clusters[3] = {2 * sms, sms, sms / 2};  // machine model: two CTAs per SM, clusters placed anywhere
  const FitPlan plan = plan_persistent_fit(F, T, D, K, lean != 0, streamed != 0, sms, clusters, PlanOverrides{});
  *kernel = plan.kernel;
  *split = plan.split;
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
  PBB_CHECK_ARG(eigenvectors && eigenvalues && weight, 11, "model output is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 14,
                "workspace too small (pbb_cacgmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 16, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  const bool persistent = fast_shape(D, K) && !(opt->reserved & 1);
  int r;
  // y (and the initial affiliations) may be pinned host memory: the kernels then read them in
  // place over PCIe.  On the persistent path with an affiliation initialisation that read is a
  // separate small kernel on a side stream that overlaps the EM kernel ("streamed upload").
  bool y_host = false, aff_host = false;
  if ((r = classify_pointer(y, &y, &y_host, "y"))) return r;
  if (init_aff != nullptr) {
    const void* alias = nullptr;
    if ((r = classify_pointer(init_aff, &alias, &aff_host, "initial affiliations"))) return r;
    init_aff = static_cast<const double*>(alias);
  }
  // the model may be written straight into pinned host memory as well (write-only on this path)
  {
    bool h = false;
    const void* alias = nullptr;
    if ((r = classify_pointer(eigenvectors, &alias, &h, "eigenvectors"))) return r;
    eigenvectors = const_cast<void*>(alias);
    if ((r = classify_pointer(eigenvalues, &alias, &h, "eigenvalues"))) return r;
    eigenvalues = static_cast<double*>(const_cast<void*>(alias));
    if ((r = classify_pointer(weight, &alias, &h, "weight"))) return r;
    weight = static_cast<double*>(const_cast<void*>(alias));
  }
  const bool streamed = persistent && y_host && init_aff != nullptr && !(opt->reserved & 2) &&
                        ws.aff_stage != nullptr;
  const bool fast_sm = softmax_fast_ok(D, opt);
  // lean variant: product-form softmax, needs (K-1) D log10(1/floor) < 290 (em_persistent.cuh).  The extra decade
  // per factor below is a margin kept as is: without it some fits (e.g. K = 4, D = 8 with floors between about 1e-12
  // and 1e-11) would move from the full variant to the lean one.
  const bool lean_ok = fast_sm && (K - 1) * D * (log10(1.0 / opt->eigenvalue_floor) + 1.0) < 290.0;
  const bool full = saliency != nullptr || activity != nullptr || !lean_ok || init_aff == nullptr;
  // Thread safety: the side stream and the fork / join events of the streamed upload exist once per device, so two
  // host threads enqueueing streamed fits on the same device are serialised from here to the end of the call
  // (the enqueue only; the GPU work of the two fits still overlaps as far as their streams allow).
  std::unique_lock<std::mutex> stream_lock;
  if (streamed) {
    LoadStream* lsm = nullptr;
    if ((r = get_load_stream(&lsm))) return r;
    stream_lock = std::unique_lock<std::mutex>(lsm->mu);
  }
  if (streamed) {
    // flags[bin] = -1 until the bin has arrived
    PBB_CUDA(cudaMemsetAsync(ws.flags, 0, (size_t)(F + 1) * sizeof(int) + 16 * sizeof(unsigned long long) + 8, st));
    PBB_CUDA(cudaMemsetAsync(ws.flags, 0xFF, (size_t)F * sizeof(int), st));
    PBB_CUDA(cudaMemsetAsync(ws.dead, 0, (size_t)F * sizeof(int), st));
    LoadStream* l = nullptr;
    if ((r = get_load_stream(&l))) return r;
    PBB_CUDA(cudaEventRecord(l->fork, st));
    PBB_CUDA(cudaStreamWaitEvent(l->stream, l->fork, 0));
    double* aff_dst = aff_host ? ws.aff_stage : nullptr;
    int* next_bin = reinterpret_cast<int*>(ws.phase + 15);
    int* started = reinterpret_cast<int*>(ws.phase + 14);
    int ctas = 0;
    r = dtype == PBB_C128
            ? launch_stream_load<double2>(y, ws.z, init_aff, aff_dst, F, T, D, K, ws.dead, ws.flags, next_bin, started, &ctas, l->stream)
            : launch_stream_load<float2>(y, ws.z, init_aff, aff_dst, F, T, D, K, ws.dead, ws.flags, next_bin, started, &ctas, l->stream);
    if (r) return r;
    PBB_CUDA(cudaEventRecord(l->join, l->stream));
    // Hold the EM kernel back until every loader CTA runs: launched at the same moment, the EM grid
    // could take the whole machine first and leave the loader only the reserved slots (it would still
    // finish -- bins are handed out by a counter -- but at a fraction of the link rate).
    if (l->wait_value != nullptr) {
      if (l->wait_value(reinterpret_cast<CUstream>(st), reinterpret_cast<CUdeviceptr>(started), (cuuint32_t)ctas,
                        CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
        l->wait_value = nullptr;  // not supported here: rely on the reserved slots
    }
    if (aff_host) init_aff = ws.aff_stage;
  } else if (persistent)  // chunk-major staged layout: one TMA bulk copy per ring stage
    r = dtype == PBB_C128 ? launch_normalize_staged<double2>(y, ws.z, F, T, D, ws.dead, st)
                          : launch_normalize_staged<float2>(y, ws.z, F, T, D, ws.dead, st);
  else
    r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                          : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;

  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.coef = ws.coef; a.ld = ws.ld; a.w = ws.w; a.ew = ws.ew;
  a.activity = activity; a.aff_eps = opt->affiliation_eps;
  a.saliency = saliency; a.part = ws.part;

  UpdArgs u;
  memset(&u, 0, sizeof(u));
  u.F = F; u.T = T; u.D = D; u.K = K;
  u.part = ws.part;
  u.covariance_norm = opt->covariance_norm;
  u.weight_mode = opt->weight_mode;
  u.has_saliency = saliency != nullptr;
  u.eigenvalue_floor = opt->eigenvalue_floor;
  u.evec = reinterpret_cast<double2*>(eigenvectors);
  u.eval = eigenvalues; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.ew = ws.ew;
  u.status = status;

  if (persistent) {
    // ---- persistent path: every EM iteration in one launch (em_persistent.cuh) ----
    if (!streamed)
      PBB_CUDA(cudaMemsetAsync(ws.flags, 0, (size_t)(F + 1) * sizeof(int) + 16 * sizeof(unsigned long long) + 8, st));
    if (init_aff == nullptr) {
      FromEigArgs fe;
      fe.F = F; fe.D = D; fe.K = K;
      fe.evec = reinterpret_cast<const double2*>(eigenvectors);
      fe.eval = eigenvalues; fe.weight = weight;
      fe.coef = ws.coef; fe.ld = ws.ld; fe.w = ws.w; fe.ew = ws.ew;
      if ((r = launch_from_eig(fe, st))) return r;
    }
    PersistArgs p;
    memset(&p, 0, sizeof(p));
    p.z = ws.z; p.zs = ws.zs; p.F = F; p.T = T;
    p.iterations = opt->iterations;
    p.first_is_m = init_aff != nullptr;
    p.user_model = init_aff == nullptr;
    p.softmax_fast = fast_sm;
    p.aff_in = init_aff; p.saliency = saliency; p.activity = activity;
    p.aff_eps = opt->affiliation_eps; p.eigenvalue_floor = opt->eigenvalue_floor;
    p.covariance_norm = opt->covariance_norm; p.weight_mode = opt->weight_mode;
    p.coef = ws.coef; p.ld = ws.ld; p.w = ws.w; p.ew = ws.ew;
    p.part = ws.part; p.flags = ws.flags; p.ticket = ws.ticket; p.status = status;
    p.phase = ws.phase; p.dead = ws.dead;
    if (streamed) {
      // bins joining per slot ~ slot duration / arrival time of one bin at ~50 GB/s of PCIe reads
      const double bin_bytes = (double)T * D * (dtype == PBB_C128 ? 16.0 : 8.0) + (aff_host ? 8.0 * K * T : 0.0);
      // one slot of the order table = one link of a bin's dependency chain (task + update + staging
      // of the next model, ~23 us at D = 8, K = 3, T = 500), during which the machine runs ~1.6 tasks per CTA
      const double round_us = 23.0 * (T / 500.0) * (D * D / 64.0) * (K / 3.0);
      int c = (int)(round_us / (bin_bytes / 50e3) + 0.5);
      if (const char* e = getenv("PBB_WAVE_C")) c = atoi(e);  // tuning override
      c = c < 1 ? 1 : (c > F ? F : c);
      p.wave_c = c;
      p.wait_load = 1;
      const long long tasks = (long long)F * opt->iterations;
      if (tasks <= kMaxOrder && F <= 4096 && opt->iterations < 32768 && !getenv("PBB_NO_ORDER")) {
        int dev = 0, sms = 0;
        PBB_CUDA(cudaGetDevice(&dev));
        PBB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        int cap = (int)(1.6 * (2 * sms - kLoadReserve));
        if (const char* e = getenv("PBB_ORDER_CAP")) cap = atoi(e);  // tuning override
        if ((r = streamed_order(F, opt->iterations, c, cap < 1 ? 1 : cap, &p.order))) return r;
      }
    }
    const PlanOverrides ov = env_overrides();
    int clusters[3] = {0, 0, 0}, sms = 0;
    if (sticky_eligible(D, !full, streamed, ov) && (r = sticky_clusters(K, dtype, clusters, st))) return r;
    if ((r = device_sms(&sms))) return r;
    const FitPlan plan = plan_persistent_fit(F, T, D, K, !full, streamed, sms, clusters, ov);
    if (plan.kernel == kKernelSticky) {
      if ((r = launch_sticky(p, K, dtype, plan.split, st))) return r;  // few bins: one cluster per bin (em_sticky.cuh)
    } else {
      if ((r = setup_frame_split(&p, ws, F, D, K, plan.split, st))) return r;
      if ((r = launch_persist(p, D, K, dtype, full, plan.kernel == kKernelWs, st))) return r;
    }
    if (streamed) {
      LoadStream* l = nullptr;
      if ((r = get_load_stream(&l))) return r;
      PBB_CUDA(cudaStreamWaitEvent(st, l->join, 0));
    }
#ifdef PBB_PHASE_TIMING
    {
      unsigned long long ph[16];
      cudaStreamSynchronize(st);
      cudaMemcpy(ph, ws.phase, sizeof(ph), cudaMemcpyDeviceToHost);
      fprintf(stderr, "[phase] update of class 0, cycles per task: build %.0f  gauss-jordan %.0f  logdet/tinv %.0f  stores %.0f\n",
              ph[8] / (double)((size_t)F * opt->iterations), ph[9] / (double)((size_t)F * opt->iterations),
              ph[10] / (double)((size_t)F * opt->iterations), ph[11] / (double)((size_t)F * opt->iterations));
      fprintf(stderr, "[phase] producer, cycles per task: ticket->dependency %.0f  model buffer wait %.0f  model issue %.0f  ring refill %.0f\n",
              ph[12] / (double)((size_t)F * opt->iterations), ph[13] / (double)((size_t)F * opt->iterations),
              ph[14] / (double)((size_t)F * opt->iterations), ph[15] / (double)((size_t)F * opt->iterations));
      unsigned long long tot = 0;
      for (int i = 0; i < 8; ++i) tot += ph[i];
      static const char* nm[8] = {"ticket+flag / model wait", "chunk-top / updater busy", "tma-wait", "em-steps", "reduce", "update / S wait", "publish / hand-over", "task-start / updater idle"};
      for (int i = 0; i < 8; ++i) fprintf(stderr, "[phase] %-20s %6.2f%%  %8.0f cycles per task\n", nm[i], 100.0 * ph[i] / (double)tot, ph[i] / (double)((size_t)F * opt->iterations));
    }
#endif
    u.nch = 1;  // the last iteration's raw scatter sums -> reference-exact model
    u.coef = nullptr;  // nobody reads the E-step form of the final model
    return launch_update(u, st);
  }
  int it = 0;
  if (init_aff != nullptr) {
    // iteration 0: M-step from the initial affiliations, q = 1 (cacgmm.py:206-228,269)
    a.mode = kModeM; a.aff_in = init_aff; a.q_in = nullptr;
    int nch = launch_em(a, dtype, opt->frames_per_block, st);
    if (nch <= 0) return nch ? nch : 1;
    u.nch = nch;
    if ((r = launch_update(u, st))) return r;
    it = 1;
  } else {
    // warm start: the model in the output arrays drives the first E-step (cacgmm.py:229-234)
    FromEigArgs fe;
    fe.F = F; fe.D = D; fe.K = K;
    fe.evec = reinterpret_cast<const double2*>(eigenvectors);
    fe.eval = eigenvalues; fe.weight = weight;
    fe.coef = ws.coef; fe.ld = ws.ld; fe.w = ws.w; fe.ew = ws.ew;
    if ((r = launch_from_eig(fe, st))) return r;
  }
  // the update kernel writes the E-step weights into `weight`; the E-step reads them from there
  a.w = weight;
  for (; it < opt->iterations; ++it) {
    a.mode = kModeEM;
    // a user-supplied model gives no bound on q / log det: keep the log-domain softmax for its E-step
    a.softmax_fast = (fast_sm && !(init_aff == nullptr && it == 0)) ? 1 : 0;
    if (init_aff == nullptr && it == 0) a.w = ws.w;
    int nch = launch_em(a, dtype, opt->frames_per_block, st);
    if (nch <= 0) return nch ? nch : 1;
    a.w = weight;
    u.nch = nch;
    if ((r = launch_update(u, st))) return r;
  }
  return 0;
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 16,
                "workspace too small (pbb_cacgmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 18, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  int r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                            : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  FromEigArgs fe;
  fe.F = F; fe.D = D; fe.K = K;
  fe.evec = reinterpret_cast<const double2*>(eigenvectors);
  fe.eval = eigenvalues;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  fe.weight = (weight_mode == PBB_WEIGHT_CONST || tied) ? nullptr : weight;
  fe.coef = ws.coef; fe.ld = ws.ld; fe.w = ws.w; fe.ew = ws.ew;
  if ((r = launch_from_eig(fe, st))) return r;
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.mode = kModeE; a.softmax_fast = 0;
  if (tied) { a.w_time = weight; a.w_time_st = weight_mode == PBB_WEIGHT_TIED_TIME ? 1 : 0; }
  a.coef = ws.coef; a.ld = ws.ld; a.w = ws.w; a.ew = ws.ew;
  a.activity = activity; a.aff_eps = affiliation_eps;
  a.aff_out = affiliation; a.q_out = quadratic;
  a.loglik_part = loglik ? ws.loglik_part : nullptr;
  int nch = launch_em(a, dtype, 0, st);
  if (nch <= 0) return nch ? nch : 1;
  if (loglik) {
    // per-bin sum of the chunk partials, fixed order
    sum_rows_kernel<<<(F + 127) / 128, 128, 0, st>>>(ws.loglik_part, loglik, F, nch);
    PBB_CUDA(cudaGetLastError());
  }
  return 0;
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 14,
                "workspace too small (pbb_cacgmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 16, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  int r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                            : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.mode = kModeM; a.aff_in = affiliation; a.q_in = quadratic;
  a.saliency = saliency; a.part = ws.part;
  int nch = launch_em(a, dtype, opt->frames_per_block, st);
  if (nch <= 0) return nch ? nch : 1;
  UpdArgs u;
  memset(&u, 0, sizeof(u));
  u.F = F; u.T = T; u.D = D; u.K = K; u.nch = nch;
  u.part = ws.part;
  u.covariance_norm = opt->covariance_norm;
  u.weight_mode = opt->weight_mode;
  u.has_saliency = saliency != nullptr;
  u.eigenvalue_floor = opt->eigenvalue_floor;
  u.evec = reinterpret_cast<double2*>(eigenvectors);
  u.eval = eigenvalues; u.weight = weight;
  u.coef = ws.coef; u.ld = ws.ld; u.ew = ws.ew;
  u.status = status;
  return launch_update(u, st);
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 18,
                "workspace too small (pbb_cwmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 20, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  const bool persistent = fast_shape(D, K) && saliency == nullptr;
  int r;
  if (persistent)
    r = dtype == PBB_C128 ? launch_normalize_staged<double2>(y, ws.z, F, T, D, ws.dead, st)
                          : launch_normalize_staged<float2>(y, ws.z, F, T, D, ws.dead, st);
  else
    r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                          : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.model_kind = 1;
  a.coef = ws.coef; a.ld = ws.ld; a.w = weight; a.ew = ws.ew;
  a.saliency = saliency; a.part = ws.part;
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
    PBB_CUDA(cudaMemsetAsync(ws.flags, 0, (size_t)(F + 1) * sizeof(int) + 16 * sizeof(unsigned long long) + 8, st));
    PersistArgs p;
    memset(&p, 0, sizeof(p));
    p.z = ws.z; p.zs = ws.zs; p.F = F; p.T = T;
    p.iterations = iterations; p.first_is_m = 1; p.user_model = 0; p.softmax_fast = 0;
    p.aff_in = init_aff; p.aff_eps = 0.0; p.weight_mode = weight_mode;
    p.coef = ws.coef; p.ld = ws.ld; p.w = ws.w; p.ew = ws.ew;
    p.part = ws.part; p.flags = ws.flags; p.ticket = ws.ticket; p.status = status; p.phase = ws.phase;
    p.spline = u.spline;
    PlanOverrides ov = env_overrides();
    ov.single = true;
    int sms = 0;
    if ((r = device_sms(&sms))) return r;
    const FitPlan plan = plan_persistent_fit(F, T, D, K, true, false, sms, nullptr, ov);
    if ((r = setup_frame_split(&p, ws, F, D, K, plan.split, st))) return r;
    if ((r = launch_persist_cw(p, D, K, dtype, st))) return r;
#ifdef PBB_PHASE_TIMING
    {
      unsigned long long ph[16];
      cudaStreamSynchronize(st);
      cudaMemcpy(ph, ws.phase, sizeof(ph), cudaMemcpyDeviceToHost);
      unsigned long long tot = 0;
      for (int i = 0; i < 8; ++i) tot += ph[i];
      static const char* nm[8] = {"flag wait", "chunk top / staging", "tma-wait", "em-steps", "reduce", "update (jacobi)", "publish", "task-start"};
      for (int i = 0; i < 8; ++i) fprintf(stderr, "[phase cw] %-20s %6.2f%%  %8.0f cycles per task\n", nm[i], 100.0 * ph[i] / (double)tot, ph[i] / (double)((size_t)F * iterations));
    }
#endif
    u.nch = 1;
    return launch_cw_update(u, st);
  }
  for (int it = 0; it < iterations; ++it) {
    if (it == 0) { a.mode = kModeM; a.aff_in = init_aff; a.q_in = nullptr; }
    else { a.mode = kModeEM; a.aff_in = nullptr; }
    int nch = launch_em(a, dtype, 0, st);
    if (nch <= 0) return nch ? nch : 1;
    u.nch = nch;
    if ((r = launch_cw_update(u, st))) return r;
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 12,
                "workspace too small (pbb_cwmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 14, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  int r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                            : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  CwFromModelArgs fm;
  fm.F = F; fm.D = D; fm.K = K;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  fm.mode = reinterpret_cast<const double2*>(mode); fm.concentration = concentration;
  fm.weight = (tied || weight_mode == PBB_WEIGHT_CONST) ? nullptr : weight;
  fm.coef = ws.coef; fm.ld = ws.ld; fm.ew = ws.ew; fm.w = ws.w;
  {
    LaunchScope ls("cw_from_model_kernel", st);
    cw_from_model_kernel<<<F, 128, (size_t)D * D * sizeof(int), st>>>(fm);
    PBB_CUDA(cudaGetLastError());
  }
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.mode = kModeE; a.model_kind = 1;
  a.coef = ws.coef; a.ld = ws.ld; a.w = ws.w; a.ew = ws.ew;
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 17,
                "workspace too small (pbb_cbmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 19, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  int r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                            : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.model_kind = 1;  // lp = ew q - ld with ew = -1, q = y^H (-B) y
  a.coef = ws.coef; a.ld = ws.ld; a.w = weight; a.ew = ws.ew;
  a.saliency = saliency; a.part = ws.part; a.aff_eps = affiliation_eps;
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
    if ((r = bingham_dispatch<CbUpdateLaunch>(D, u, st))) return r;
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
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_cacgmm_workspace_bytes(F, T, D, K), 13,
                "workspace too small (pbb_cbmm_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 15, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CacgmmWorkspace ws = carve(workspace, F, T, D, K);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  int r = dtype == PBB_C128 ? launch_normalize<double2>(y, ws.z, F, T, D, 1, ws.zs, st)
                            : launch_normalize<float2>(y, ws.z, F, T, D, 1, ws.zs, st);
  if (r) return r;
  const bool tied = weight_mode == PBB_WEIGHT_TIED_TIME || weight_mode == PBB_WEIGHT_TIED;
  CbFromModelArgs fm;
  fm.F = F; fm.K = K;
  fm.evec = reinterpret_cast<const double2*>(eigenvectors); fm.eval = eigenvalues;
  fm.weight = (tied || weight_mode == PBB_WEIGHT_CONST) ? nullptr : weight;
  fm.coef = ws.coef; fm.ld = ws.ld; fm.ew = ws.ew; fm.w = ws.w;
  if ((r = bingham_dispatch<CbFromModelLaunch>(D, fm, st))) return r;
  EmArgs a;
  memset(&a, 0, sizeof(a));
  a.z = ws.z; a.zs = ws.zs; a.F = F; a.T = T; a.D = D; a.K = K;
  a.mode = kModeE; a.model_kind = 1;
  a.coef = ws.coef; a.ld = ws.ld; a.w = ws.w; a.ew = ws.ew;
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
  return bingham_dispatch<BinghamParametersLaunch>(D, scatter_eigenvalues, n, eps, max_concentration, eigenvalues,
                                                   status, st);
}

int pbb_bingham_log_norm(const double* eigenvalues, int n, int D, double eps, double* log_norm, void* stream) {
  PBB_CHECK_ARG(eigenvalues != nullptr, 1, "eigenvalues are null");
  PBB_CHECK_ARG(n > 0, 2, "n must be positive");
  PBB_CHECK_ARG(D >= 2 && D <= 6, 3, "complex Bingham: need 2 <= D <= 6 (complex_bingham_utils.py:342-348)");
  PBB_CHECK_ARG(log_norm != nullptr, 5, "output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return bingham_dispatch<BinghamLogNormLaunch>(D, eigenvalues, n, eps, log_norm, st);
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
  LaunchScope ls("bingham_log_pdf_kernel", st);
  if (dtype == PBB_C128)
    bingham_log_pdf_kernel<double2><<<blocks, 128, 0, st>>>(static_cast<const double2*>(y), V, eigenvalues, log_norm,
                                                            M, T, D, log_pdf);
  else
    bingham_log_pdf_kernel<float2><<<blocks, 128, 0, st>>>(static_cast<const float2*>(y), V, eigenvalues, log_norm,
                                                           M, T, D, log_pdf);
  PBB_CUDA(cudaGetLastError());
  return 0;
}

int pbb_mixture_weight_over_bins(const double* affiliation, int F, int K, int T, int flags, double* weight_kt,
                                 double* weight_k, void* stream) {
  const int also_over_time = flags & 1, unit_norm = flags & 2;
  PBB_CHECK_ARG(affiliation != nullptr, 1, "affiliation is null");
  PBB_CHECK_ARG(F > 0 && K > 0 && K < kMaxK && T > 0, 2, "bad shape");
  PBB_CHECK_ARG(weight_kt != nullptr, 6, "weight (K, T) output is null");
  PBB_CHECK_ARG(!also_over_time || weight_k != nullptr, 7, "weight (K) output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  LaunchScope ls("mean_over_bins_kernel", st);
  mean_over_bins_kernel<<<(K * T + 255) / 256, 256, 0, st>>>(affiliation, F, K, T, weight_kt);
  if (also_over_time) mean_over_time_kernel<<<K, 256, 0, st>>>(weight_kt, K, T, weight_k);
  if (unit_norm) {
    // the saliency form of estimate_mixture_weight (mixture_model_utils.py:192-203, used by CWMMTrainer):
    // sums instead of means, then _unit_norm(ord=1, axis=-2, eps=1e-10, 'where') -- the 1/F (1/T) cancels
    if (also_over_time) unit_norm_over_classes_kernel<<<1, 32, 0, st>>>(weight_k, K, 1);
    else unit_norm_over_classes_kernel<<<(T + 127) / 128, 128, 0, st>>>(weight_kt, K, T);
  }
  PBB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
