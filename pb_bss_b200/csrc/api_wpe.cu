// C-ABI entry points for WPE dereverberation, nara_wpe.wpe -- see include/pbb.h, csrc/wpe.cuh and
// csrc/wpe_online.cuh.
#include "common.cuh"
#include "prof.cuh"
#include "wpe.cuh"
#include "wpe_online.cuh"

namespace pbb {

static size_t wpe_align(size_t b) { return (b + 255) & ~(size_t)255; }

static WpeShape wpe_shape(int D, long long T, int taps, int delay, int valid, long long psd_context) {
  WpeShape s{};
  s.T = T;
  s.D = D;
  s.taps = taps;
  s.delay = delay;
  s.n = taps * D;
  s.N2 = s.n + D;
  s.T8 = (2 * s.N2 + 7) / 8;
  s.ntiles = s.T8 * (s.T8 + 1) / 2;
  s.tb = valid ? (long long)delay + taps - 1 : 0;
  const long long tv = T - s.tb;
  if (tv <= 0) {
    s.parts = 1;
    s.span = kWpeChunk;
  } else {
    long long parts = (tv + kWpePartFrames - 1) / kWpePartFrames;
    parts = parts > kWpeMaxParts ? kWpeMaxParts : parts;
    long long span = (tv + parts - 1) / parts;
    s.span = (span + kWpeChunk - 1) / kWpeChunk * kWpeChunk;
    s.parts = (int)((tv + s.span - 1) / s.span);
  }
  s.psd_context = psd_context;
  return s;
}

struct WpeLayout {
  size_t w, lam, part, G, lstsq, total;  // byte offsets
};

static WpeLayout wpe_layout(long long group, const WpeShape& s) {
  WpeLayout l;
  l.w = 0;
  l.lam = wpe_align(l.w + (size_t)group * s.T * sizeof(double));
  l.part = wpe_align(l.lam + (size_t)group * s.T * sizeof(double));
  l.G = wpe_align(l.part + (size_t)group * s.parts * s.ntiles * 64 * sizeof(double));
  l.lstsq = wpe_align(l.G + (size_t)group * s.n * s.D * sizeof(double2));
  l.total = l.lstsq + (size_t)group * sizeof(int);
  return l;
}

template <class TIn>
static int wpe_filter_launch(const TIn* y, WpeStrides ys, const WpeShape& s, long long bins, const double2* G,
                             TIn* out, WpeStrides os, int power, double* lam, double* pw, int* status,
                             cudaStream_t st) {
  const size_t smem = wpe_filter_smem_bytes(s.D, s.taps);
  PBB_CUDA(cudaFuncSetAttribute(wpe_filter_kernel<TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel("wpe_filter_kernel", wpe_filter_kernel<TIn>, (unsigned)bins, 256, smem, st, y, ys, s, G, out, os,
                       power, lam, pw, status);
}

template <int TPW, class TIn>
static int wpe_corr_launch(const TIn* y, WpeStrides ys, const WpeShape& s, long long bins, const double* w,
                           double* part, cudaStream_t st) {
  const size_t smem = wpe_corr_smem_doubles(s.D, s.taps) * sizeof(double);
  const unsigned passes = (unsigned)((s.ntiles + kWpeCorrWarps * TPW - 1) / (kWpeCorrWarps * TPW));
  PBB_CUDA(cudaFuncSetAttribute(wpe_corr_kernel<TPW, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel("wpe_corr_kernel", wpe_corr_kernel<TPW, TIn>, dim3((unsigned)s.parts, (unsigned)bins, passes),
                       32 * kWpeCorrWarps, smem, st, y, ys, s, w, part);
}

// tiles per warp: the smallest instantiated slot count that covers every lower-triangle tile in one pass; more than
// 16 x 22 tiles (n + D > 104) run in several passes of 22 slots
template <class TIn>
static int wpe_corr(const TIn* y, WpeStrides ys, const WpeShape& s, long long bins, const double* w, double* part,
                    cudaStream_t st) {
  const int tpw = (s.ntiles + kWpeCorrWarps - 1) / kWpeCorrWarps;
  if (tpw <= 2) return wpe_corr_launch<2>(y, ys, s, bins, w, part, st);
  if (tpw <= 6) return wpe_corr_launch<6>(y, ys, s, bins, w, part, st);
  if (tpw <= 12) return wpe_corr_launch<12>(y, ys, s, bins, w, part, st);
  if (tpw <= 16) return wpe_corr_launch<16>(y, ys, s, bins, w, part, st);
  return wpe_corr_launch<22>(y, ys, s, bins, w, part, st);
}

// R, P from the weights w of a group, G = stable_solve(R, P): wpe_corr, wpe_solve_kernel and wpe_lstsq_kernel
template <class TIn>
static int wpe_solve_group(const TIn* yg, WpeStrides ys, const WpeShape& s, long long g, const double* w, double* part,
                           double2* G, int* lstsq, int* status, cudaStream_t st) {
  int rc = wpe_corr<TIn>(yg, ys, s, g, w, part, st);
  if (rc) return rc;
  PBB_TRY(launch_kernel("wpe_solve_kernel", wpe_solve_kernel, (unsigned)g, 256, wpe_solve_smem_bytes(s.n, s.D), st,
                        part, s, G, lstsq, status));
  return launch_kernel("wpe_lstsq_kernel", wpe_lstsq_kernel, (unsigned)g, 32, wpe_lstsq_smem_bytes(s.n, s.D), st, part,
                       s, lstsq, G);
}

template <class TIn>
static int wpe_run(const TIn* y, WpeStrides ys, long long bins, TIn* out, WpeStrides os, const WpeShape& s,
                   int iterations, long long group, char* ws, int* status, cudaStream_t st, double2* G_save,
                   double* w_save) {
  const WpeLayout l = wpe_layout(group, s);
  double* w = reinterpret_cast<double*>(ws + l.w);
  double* lam = reinterpret_cast<double*>(ws + l.lam);
  double* part = reinterpret_cast<double*>(ws + l.part);
  double2* G = reinterpret_cast<double2*>(ws + l.G);
  int* lstsq = reinterpret_cast<int*>(ws + l.lstsq);
  const size_t solve_smem = wpe_solve_smem_bytes(s.n, s.D), lstsq_smem = wpe_lstsq_smem_bytes(s.n, s.D);
  PBB_CUDA(cudaFuncSetAttribute(wpe_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
  PBB_CUDA(cudaFuncSetAttribute(wpe_lstsq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lstsq_smem));
  for (long long b0 = 0; b0 < bins; b0 += group) {
    const long long g = bins - b0 < group ? bins - b0 : group;
    const TIn* yg = y + b0 * ys.b;
    TIn* og = out + b0 * os.b;
    int rc = wpe_filter_launch<TIn>(yg, ys, s, g, nullptr, iterations == 0 ? og : nullptr, os,
                                    iterations == 0 ? kWpePowerNone : kWpePowerInverse, lam, w, status, st);
    if (rc) return rc;
    for (int it = 0; it < iterations; ++it) {
      const bool last = it == iterations - 1;
      if (w_save != nullptr)
        PBB_CUDA(cudaMemcpyAsync(w_save + (it * bins + b0) * s.T, w, (size_t)g * s.T * sizeof(double),
                                 cudaMemcpyDeviceToDevice, st));
      rc = wpe_solve_group<TIn>(yg, ys, s, g, w, part, G, lstsq, status, st);
      if (rc) return rc;
      if (G_save != nullptr)
        PBB_CUDA(cudaMemcpyAsync(G_save + (it * bins + b0) * s.n * s.D, G, (size_t)g * s.n * s.D * sizeof(double2),
                                 cudaMemcpyDeviceToDevice, st));
      rc = wpe_filter_launch<TIn>(yg, ys, s, g, G, last ? og : nullptr, os, last ? kWpePowerNone : kWpePowerInverse,
                                  lam, w, status, st);
      if (rc) return rc;
    }
  }
  return 0;
}

// one WPE step with the caller's weights wsrc (element (b, t) at b wsb + t wst), copied into the workspace's w:
// pbb_wpe's launches with the copy in place of the power kernel; G_save (null: not kept) receives the filters
template <class TIn>
static int wpe_step_run(const TIn* y, WpeStrides ys, long long bins, const double* wsrc, long long wsb,
                        long long wst, TIn* out, WpeStrides os, const WpeShape& s, long long group, char* ws,
                        int* status, double2* G_save, cudaStream_t st) {
  const WpeLayout l = wpe_layout(group, s);
  double* w = reinterpret_cast<double*>(ws + l.w);
  double* part = reinterpret_cast<double*>(ws + l.part);
  double2* G = reinterpret_cast<double2*>(ws + l.G);
  int* lstsq = reinterpret_cast<int*>(ws + l.lstsq);
  const size_t solve_smem = wpe_solve_smem_bytes(s.n, s.D), lstsq_smem = wpe_lstsq_smem_bytes(s.n, s.D);
  PBB_CUDA(cudaFuncSetAttribute(wpe_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
  PBB_CUDA(cudaFuncSetAttribute(wpe_lstsq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lstsq_smem));
  for (long long b0 = 0; b0 < bins; b0 += group) {
    const long long g = bins - b0 < group ? bins - b0 : group;
    const long long total = g * s.T;
    PBB_TRY(launch_kernel("wpe_weight_copy_kernel", wpe_weight_copy_kernel,
                          (unsigned)(total / 256 + 1 < 65536 ? total / 256 + 1 : 65536), 256, 0, st, wsrc + b0 * wsb,
                          wsb, wst, g, s.T, w));
    int rc = wpe_solve_group<TIn>(y + b0 * ys.b, ys, s, g, w, part, G, lstsq, status, st);
    if (rc) return rc;
    if (G_save != nullptr)
      PBB_CUDA(cudaMemcpyAsync(G_save + b0 * s.n * s.D, G, (size_t)g * s.n * s.D * sizeof(double2),
                               cudaMemcpyDeviceToDevice, st));
    rc = wpe_filter_launch<TIn>(y + b0 * ys.b, ys, s, g, G, out + b0 * os.b, os, kWpePowerNone, nullptr, nullptr,
                                status, st);
    if (rc) return rc;
  }
  return 0;
}

struct WpeBackLayout {
  size_t part, Pbar, ub, total;  // byte offsets
};

static WpeBackLayout wpe_back_layout(long long group, const WpeShape& s) {
  WpeBackLayout l;
  l.part = 0;
  l.Pbar = wpe_align(l.part + (size_t)group * s.parts * s.ntiles * 64 * sizeof(double));
  l.ub = wpe_align(l.Pbar + (size_t)group * s.n * s.D * sizeof(double2));
  l.total = l.ub + (size_t)group * 2 * s.D * s.T * sizeof(double2);
  return l;
}

// one stage of the step backward: the forward's R again (wpe_corr with the same weights, bit for bit), Gbar, Pbar =
// R^-1 Gbar, then the per-frame pass.  An empty S (valid, T <= delay + taps - 1) has G = 0 for every input: Pbar = 0.
template <class TIn>
static int wpe_backward_run(const TIn* y, WpeStrides ys, long long bins, const WpeShape& s, const double* w,
                            const double2* G, const double2* xbar, double2* ybar, double* wbar, long long group,
                            char* ws, cudaStream_t st) {
  const WpeBackLayout l = wpe_back_layout(group, s);
  double* part = reinterpret_cast<double*>(ws + l.part);
  double2* Pbar = reinterpret_cast<double2*>(ws + l.Pbar);
  double2* ub = reinterpret_cast<double2*>(ws + l.ub);
  const size_t gbar_smem = wpe_gbar_smem_bytes(s.D, s.taps), solve_smem = wpe_solve_smem_bytes(s.n, s.D);
  const size_t back_smem = wpe_step_backward_smem_bytes(s.D, s.taps);
  PBB_CUDA(cudaFuncSetAttribute(wpe_gbar_kernel<TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gbar_smem));
  PBB_CUDA(cudaFuncSetAttribute(wpe_solve_rhs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
  PBB_CUDA(cudaFuncSetAttribute(wpe_step_backward_kernel<TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)back_smem));
  const long long per = (long long)s.D * s.T;
  for (long long b0 = 0; b0 < bins; b0 += group) {
    const long long g = bins - b0 < group ? bins - b0 : group;
    const TIn* yg = y + b0 * ys.b;
    if (s.tb < s.T) {
      int rc = wpe_corr<TIn>(yg, ys, s, g, w + b0 * s.T, part, st);
      if (rc) return rc;
      PBB_TRY(launch_kernel("wpe_gbar_kernel", wpe_gbar_kernel<TIn>, (unsigned)g, 256, gbar_smem, st, yg, ys, s,
                            xbar + b0 * per, Pbar));
      PBB_TRY(launch_kernel("wpe_solve_rhs_kernel", wpe_solve_rhs_kernel, (unsigned)g, 256, solve_smem, st, part, s,
                            Pbar));
    } else {
      PBB_CUDA(cudaMemsetAsync(Pbar, 0, (size_t)g * s.n * s.D * sizeof(double2), st));
    }
    PBB_TRY(launch_kernel("wpe_step_backward_kernel", wpe_step_backward_kernel<TIn>, (unsigned)g, 256, back_smem, st,
                          yg, ys, s, G + b0 * s.n * s.D, Pbar, w + b0 * s.T, xbar + b0 * per, ub, ybar + b0 * per,
                          wbar + b0 * s.T));
  }
  return 0;
}

// the power chain's backward over all bins; workspace: lambda, lambda_c and a gradient scratch, bins T doubles each
template <class TIn>
static int wpe_power_backward_run(const TIn* y, WpeStrides ys, long long bins, const WpeShape& s, const double2* G,
                                  int mode, const double* gin, double2* xbar, double* ws, cudaStream_t st) {
  double* lam = ws;
  double* lamc = ws + bins * s.T;
  double* pbar = lamc + bins * s.T;
  if (mode != kWpeGradPlain) {
    // lambda_c exactly as the forward computed it: the forward's own kernel and arguments
    int rc = wpe_filter_launch<TIn>(y, ys, s, bins, G, nullptr, ys, kWpePowerPlain, lam, lamc, nullptr, st);
    if (rc) return rc;
  }
  if (mode == kWpeGradInverseAll) {
    PBB_TRY(launch_kernel("wpe_power_inverse_backward_kernel", wpe_power_inverse_backward_kernel, 1, 1024, 0, st, lamc,
                          gin, lam, bins * s.T));
    gin = lam;
    mode = kWpeGradPlain;
  }
  const size_t smem = wpe_power_backward_smem_bytes(s.D, s.taps, G != nullptr);
  PBB_CUDA(cudaFuncSetAttribute(wpe_power_backward_kernel<TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem));
  return launch_kernel("wpe_power_backward_kernel", wpe_power_backward_kernel<TIn>, (unsigned)bins, 256, smem, st, y,
                       ys, s, G, lamc, gin, mode, pbar, xbar);
}

template <int R, class TIn>
static int wpe_online_launch(const TIn* y, WpeStrides ys, const TIn* hist, WpeStrides hs, const double* power,
                             const double2* Qin, const double2* Gin, TIn* z, WpeStrides zs, double2* Qout,
                             double2* Gout, long long bins, const WpeOnlineShape& s, cudaStream_t st) {
  const size_t smem = wpe_online_smem_bytes(s.D, s.taps, s.delay);
  PBB_CUDA(cudaFuncSetAttribute(wpe_online_kernel<R, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel("wpe_online_kernel", wpe_online_kernel<R, TIn>, (unsigned)bins, kWpeOnlineThreads, smem, st, y,
                       ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, s);
}

// R = ceil(n / 16): each of the 16 x 16 threads holds R x R entries of Q
template <class TIn>
static int wpe_online_run(const TIn* y, WpeStrides ys, const TIn* hist, WpeStrides hs, const double* power,
                          const double2* Qin, const double2* Gin, TIn* z, WpeStrides zs, double2* Qout,
                          double2* Gout, long long bins, const WpeOnlineShape& s, cudaStream_t st) {
  switch ((s.n + 15) / 16) {
    case 1: return wpe_online_launch<1>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
    case 2: return wpe_online_launch<2>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
    case 3: return wpe_online_launch<3>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
    case 4: return wpe_online_launch<4>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
    case 5: return wpe_online_launch<5>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
    default: return wpe_online_launch<6>(y, ys, hist, hs, power, Qin, Gin, z, zs, Qout, Gout, bins, s, st);
  }
}

static bool wpe_valid_shape(int D, long long T, int taps, int delay) {
  return D >= 1 && D <= PBB_WPE_MAX_D && T >= 1 && taps >= 1 && delay >= 0 && (long long)taps * D <= kWpeMaxN;
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_wpe_workspace_bytes(long long group, int D, long long T, int taps, int delay, int valid) {
  if (group <= 0 || group > PBB_WPE_MAX_GROUP || !wpe_valid_shape(D, T, taps, delay)) return 0;
  return wpe_layout(group, wpe_shape(D, T, taps, delay, valid, 0)).total;
}

int pbb_wpe(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd, long long yst,
            void* out, long long osb, long long osd, long long ost, int taps, int delay, int iterations,
            long long psd_context, int valid, long long group, void* workspace, size_t workspace_bytes, int* status,
            void* stream) {
  return pbb_wpe_forward(y, dtype, bins, D, T, ysb, ysd, yst, out, osb, osd, ost, taps, delay, iterations,
                         psd_context, valid, group, workspace, workspace_bytes, status, nullptr, nullptr, stream);
}

int pbb_wpe_forward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                    long long yst, void* out, long long osb, long long osd, long long ost, int taps, int delay,
                    int iterations, long long psd_context, int valid, long long group, void* workspace,
                    size_t workspace_bytes, int* status, void* G_save, double* w_save, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0, 3, "bins must be positive");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(out != nullptr, 9, "out is null");
  PBB_CHECK_ARG(taps >= 1, 13, "taps must be positive");
  PBB_CHECK_ARG(delay >= 0, 14, "delay must be >= 0");
  PBB_CHECK_ARG((long long)taps * D <= kWpeMaxN, 13, "taps * D must be <= PBB_WPE_MAX_N (96)");
  PBB_CHECK_ARG(iterations >= 0, 15, "iterations must be >= 0");
  PBB_CHECK_ARG(group > 0 && group <= PBB_WPE_MAX_GROUP, 18, "group must be in [1, PBB_WPE_MAX_GROUP]");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid),
                19, "workspace too small (pbb_wpe_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 21, "status is null");
  PBB_CHECK_ARG((G_save == nullptr) == (w_save == nullptr), 22, "G_save and w_save must both be given or both null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeShape s = wpe_shape(D, T, taps, delay, valid, psd_context);
  const WpeStrides ys{ysb, ysd, yst}, os{osb, osd, ost};
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  char* ws = static_cast<char*>(workspace);
  double2* Gs = static_cast<double2*>(G_save);
  if (dtype == PBB_C64)
    return wpe_run<float2>(static_cast<const float2*>(y), ys, bins, static_cast<float2*>(out), os, s, iterations,
                           group, ws, status, st, Gs, w_save);
  return wpe_run<double2>(static_cast<const double2*>(y), ys, bins, static_cast<double2*>(out), os, s, iterations,
                          group, ws, status, st, Gs, w_save);
}

int pbb_wpe_step(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                 long long yst, const double* weight, long long wsb, long long wst, void* out, long long osb,
                 long long osd, long long ost, int taps, int delay, int valid, long long group, void* workspace,
                 size_t workspace_bytes, int* status, void* G_out, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0, 3, "bins must be positive");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(weight != nullptr, 9, "weight is null");
  PBB_CHECK_ARG(out != nullptr, 12, "out is null");
  PBB_CHECK_ARG(taps >= 1, 16, "taps must be positive");
  PBB_CHECK_ARG(delay >= 0, 17, "delay must be >= 0");
  PBB_CHECK_ARG((long long)taps * D <= kWpeMaxN, 16, "taps * D must be <= PBB_WPE_MAX_N (96)");
  PBB_CHECK_ARG(group > 0 && group <= PBB_WPE_MAX_GROUP, 19, "group must be in [1, PBB_WPE_MAX_GROUP]");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid),
                20, "workspace too small (pbb_wpe_workspace_bytes)");
  PBB_CHECK_ARG(status != nullptr, 22, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeShape s = wpe_shape(D, T, taps, delay, valid, 0);
  const WpeStrides ys{ysb, ysd, yst}, os{osb, osd, ost};
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  char* ws = static_cast<char*>(workspace);
  double2* Go = static_cast<double2*>(G_out);
  if (dtype == PBB_C64)
    return wpe_step_run<float2>(static_cast<const float2*>(y), ys, bins, weight, wsb, wst, static_cast<float2*>(out),
                                os, s, group, ws, status, Go, st);
  return wpe_step_run<double2>(static_cast<const double2*>(y), ys, bins, weight, wsb, wst, static_cast<double2*>(out),
                               os, s, group, ws, status, Go, st);
}

size_t pbb_wpe_backward_workspace_bytes(long long group, int D, long long T, int taps, int delay, int valid) {
  if (group <= 0 || group > PBB_WPE_MAX_GROUP || !wpe_valid_shape(D, T, taps, delay)) return 0;
  return wpe_back_layout(group, wpe_shape(D, T, taps, delay, valid, 0)).total;
}

int pbb_wpe_backward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                     long long yst, const double* weight, const void* G, const void* xbar, int taps, int delay,
                     int valid, void* ybar, double* wbar, long long group, void* workspace, size_t workspace_bytes,
                     void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0, 3, "bins must be positive");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(weight != nullptr, 9, "weight is null");
  PBB_CHECK_ARG(G != nullptr, 10, "G is null");
  PBB_CHECK_ARG(xbar != nullptr, 11, "xbar is null");
  PBB_CHECK_ARG(taps >= 1, 12, "taps must be positive");
  PBB_CHECK_ARG(delay >= 0, 13, "delay must be >= 0");
  PBB_CHECK_ARG((long long)taps * D <= kWpeMaxN, 12, "taps * D must be <= PBB_WPE_MAX_N (96)");
  PBB_CHECK_ARG(ybar != nullptr, 15, "ybar is null");
  PBB_CHECK_ARG(wbar != nullptr, 16, "wbar is null");
  PBB_CHECK_ARG(group > 0 && group <= PBB_WPE_MAX_GROUP, 17, "group must be in [1, PBB_WPE_MAX_GROUP]");
  PBB_CHECK_ARG(workspace != nullptr &&
                    workspace_bytes >= pbb_wpe_backward_workspace_bytes(group, D, T, taps, delay, valid),
                18, "workspace too small (pbb_wpe_backward_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeShape s = wpe_shape(D, T, taps, delay, valid, 0);
  const WpeStrides ys{ysb, ysd, yst};
  char* ws = static_cast<char*>(workspace);
  const double2* g = static_cast<const double2*>(G);
  const double2* xb = static_cast<const double2*>(xbar);
  double2* yb = static_cast<double2*>(ybar);
  if (dtype == PBB_C64)
    return wpe_backward_run<float2>(static_cast<const float2*>(y), ys, bins, s, weight, g, xb, yb, wbar, group, ws,
                                    st);
  return wpe_backward_run<double2>(static_cast<const double2*>(y), ys, bins, s, weight, g, xb, yb, wbar, group, ws,
                                   st);
}

size_t pbb_wpe_power_backward_workspace_bytes(long long bins, long long T) {
  if (bins <= 0 || T <= 0) return 0;
  return 3 * (size_t)bins * T * sizeof(double);
}

int pbb_wpe_power_backward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                           long long yst, const void* G, int taps, int delay, long long psd_context, int mode,
                           const double* gin, void* xbar, void* workspace, size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0 && bins <= 0x7fffffffLL, 3, "bins must be in [1, 2^31 - 1]");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(taps >= 1, 10, "taps must be positive");
  PBB_CHECK_ARG(delay >= 0, 11, "delay must be >= 0");
  PBB_CHECK_ARG(G == nullptr || (long long)taps * D <= kWpeMaxN, 10, "taps * D must be <= PBB_WPE_MAX_N (96)");
  PBB_CHECK_ARG(mode >= PBB_WPE_GRAD_INVERSE && mode <= PBB_WPE_GRAD_INVERSE_ALL, 13, "mode must be a PBB_WPE_GRAD_*");
  PBB_CHECK_ARG(gin != nullptr, 14, "gin is null");
  PBB_CHECK_ARG(xbar != nullptr, 15, "xbar is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_wpe_power_backward_workspace_bytes(bins, T), 16,
                "workspace too small (pbb_wpe_power_backward_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeShape s = wpe_shape(D, T, G == nullptr ? 1 : taps, G == nullptr ? 0 : delay, 0, psd_context);
  const WpeStrides ys{ysb, ysd, yst};
  const double2* g = static_cast<const double2*>(G);
  double2* xb = static_cast<double2*>(xbar);
  double* ws = static_cast<double*>(workspace);
  if (dtype == PBB_C64)
    return wpe_power_backward_run<float2>(static_cast<const float2*>(y), ys, bins, s, g, mode, gin, xb, ws, st);
  return wpe_power_backward_run<double2>(static_cast<const double2*>(y), ys, bins, s, g, mode, gin, xb, ws, st);
}

size_t pbb_wpe_power_workspace_bytes(long long bins, long long T) {
  if (bins <= 0 || T <= 0) return 0;
  return (size_t)bins * T * sizeof(double);
}

int pbb_wpe_power(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                  long long yst, long long psd_context, int inverse, double* out, void* workspace,
                  size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0 && bins <= 0x7fffffffLL, 3, "bins must be in [1, 2^31 - 1]");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(out != nullptr, 11, "out is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_wpe_power_workspace_bytes(bins, T), 12,
                "workspace too small (pbb_wpe_power_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeShape s = wpe_shape(D, T, 1, 0, 0, psd_context);
  const WpeStrides ys{ysb, ysd, yst};
  double* lam = static_cast<double*>(workspace);
  int rc = dtype == PBB_C64
               ? wpe_filter_launch<float2>(static_cast<const float2*>(y), ys, s, bins, nullptr, nullptr, ys,
                                           kWpePowerPlain, lam, out, nullptr, st)
               : wpe_filter_launch<double2>(static_cast<const double2*>(y), ys, s, bins, nullptr, nullptr, ys,
                                            kWpePowerPlain, lam, out, nullptr, st);
  if (rc || !inverse) return rc;
  return launch_kernel("wpe_power_inverse_kernel", wpe_power_inverse_kernel, 1, 1024, 0, st, out, bins * T);
}

int pbb_wpe_build_y_tilde(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                          long long yst, int taps, int delay, void* out, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0, 3, "bins must be positive");
  PBB_CHECK_ARG(D >= 1, 4, "D must be positive");
  PBB_CHECK_ARG(T >= 1, 5, "T must be positive");
  PBB_CHECK_ARG(taps >= 1, 9, "taps must be positive");
  PBB_CHECK_ARG(delay >= 0, 10, "delay must be >= 0");
  PBB_CHECK_ARG(out != nullptr, 11, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const WpeStrides ys{ysb, ysd, yst};
  const long long total = bins * taps * D * T;
  const unsigned blocks = (unsigned)(total / 256 + 1 < 65536 ? total / 256 + 1 : 65536);
  return with_ct(dtype, [&](auto ct) {
    using CT = decltype(ct);
    return launch_kernel("wpe_y_tilde_kernel", wpe_y_tilde_kernel<CT>, blocks, 256, 0, st, static_cast<const CT*>(y),
                         ys, bins, D, T, taps, delay, static_cast<CT*>(out));
  });
}

size_t pbb_wpe_online_smem_bytes(int D, int taps, int delay) {
  if (D < 1 || taps < 1 || delay < 0) return 0;
  return wpe_online_smem_bytes(D, taps, delay);
}

int pbb_wpe_online(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                   long long yst, const void* history, long long hsb, long long hsd, long long hst,
                   const double* power, const void* inv_cov, const void* filter_taps, void* z, long long zsb,
                   long long zsd, long long zst, void* inv_cov_out, void* filter_taps_out, int taps, int delay,
                   double alpha, void* stream) {
  PBB_CHECK_ARG(y != nullptr || T == 0, 1, "y is null");
  PBB_CHECK_ARG(dtype == PBB_C64 || dtype == PBB_C128, 2, "dtype must be PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(bins > 0 && bins <= 0x7fffffffLL, 3, "bins must be in [1, 2^31 - 1]");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_WPE_MAX_D, 4, "D must be in [1, PBB_WPE_MAX_D] (30)");
  PBB_CHECK_ARG(T >= 0, 5, "T must be >= 0");
  PBB_CHECK_ARG(power == nullptr || T == 1, 13, "power needs T = 1");
  PBB_CHECK_ARG(z != nullptr || T == 0, 16, "z is null");
  PBB_CHECK_ARG(inv_cov_out != nullptr, 20, "inv_cov_out is null");
  PBB_CHECK_ARG(filter_taps_out != nullptr, 21, "filter_taps_out is null");
  PBB_CHECK_ARG(taps >= 1, 22, "taps must be positive");
  PBB_CHECK_ARG((long long)taps * D <= kWpeMaxN, 22, "taps * D must be <= PBB_WPE_MAX_N (96)");
  PBB_CHECK_ARG(delay >= 0, 23, "delay must be >= 0");
  PBB_CHECK_ARG(alpha > 0.0 && alpha <= 1.0, 24, "alpha must be in (0, 1]");
  PBB_CHECK_ARG(wpe_online_smem_bytes(D, taps, delay) <= (size_t)PBB_WPE_ONLINE_MAX_SMEM, 23,
                "taps + delay + 1 frames of D channels do not fit the shared memory of a CTA "
                "(pbb_wpe_online_smem_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  WpeOnlineShape s{};
  s.T = T;
  s.D = D;
  s.taps = taps;
  s.delay = delay;
  s.n = taps * D;
  s.L = taps + delay + 1;
  s.alpha = alpha;
  s.inv_alpha = 1.0 / alpha;
  const WpeStrides ys{ysb, ysd, yst}, hs{hsb, hsd, hst}, zs{zsb, zsd, zst};
  const double2* Qin = static_cast<const double2*>(inv_cov);
  const double2* Gin = static_cast<const double2*>(filter_taps);
  double2* Qout = static_cast<double2*>(inv_cov_out);
  double2* Gout = static_cast<double2*>(filter_taps_out);
  if (dtype == PBB_C64)
    return wpe_online_run<float2>(static_cast<const float2*>(y), ys, static_cast<const float2*>(history), hs, power,
                                  Qin, Gin, static_cast<float2*>(z), zs, Qout, Gout, bins, s, st);
  return wpe_online_run<double2>(static_cast<const double2*>(y), ys, static_cast<const double2*>(history), hs, power,
                                 Qin, Gin, static_cast<double2*>(z), zs, Qout, Gout, bins, s, st);
}

}  // extern "C"
