// C-ABI entry points for STOI and ESTOI, pb_bss/evaluation/module_stoi.py -- see include/pbb.h and csrc/stoi.cuh.
#include "common.cuh"
#include "prof.cuh"
#include "stoi.cuh"

namespace pbb {

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static long long gcd_ll(long long a, long long b) {
  while (b) {
    const long long t = a % b;
    a = b;
    b = t;
  }
  return a;
}

struct StoiShape {
  long long L;         // length at 10 kHz: ceil(n up / down)
  int F, Mmax, blocks;
  bool resample;
};

static bool stoi_shape(long long n, int up, int down, StoiShape* s) {
  if (n < 1 || n > PBB_STOI_MAX_SAMPLES || up < 1 || down < 1 || gcd_ll(up, down) != 1) return false;
  const long long L = (n * up + down - 1) / down;
  if (L <= kStoiFrame || L > PBB_STOI_MAX_RESAMPLED) return false;
  s->L = L;
  s->F = (int)((L - kStoiFrame + kStoiHop - 1) / kStoiHop);  // 128 f < L - 256
  s->Mmax = s->F - 1;
  s->blocks = s->Mmax >= kStoiSeg ? (s->Mmax - kStoiSeg + 1 + kStoiSegBlock - 1) / kStoiSegBlock : 1;
  s->resample = !(up == 1 && down == 1);
  return true;
}

struct StoiLayout {
  size_t sig, energy, kept, km, tob, partial, total;  // byte offsets
};

static StoiLayout stoi_layout(long long group, const StoiShape& s) {
  StoiLayout l;
  l.sig = 0;
  l.energy = align256(l.sig + (s.resample ? (size_t)group * 2 * s.L * sizeof(double) : 0));
  l.kept = align256(l.energy + (size_t)group * s.F * sizeof(double));
  l.km = align256(l.kept + (size_t)group * s.F * sizeof(int));
  l.tob = align256(l.km + (size_t)group * 2 * sizeof(long long));
  l.partial = align256(l.tob + (size_t)group * 2 * kStoiBands * s.Mmax * sizeof(double));
  l.total = l.partial + (size_t)group * s.blocks * sizeof(double);
  return l;
}

// Grid of a grid-stride kernel over `total` items.
static unsigned stoi_ctas(long long total) {
  return (unsigned)std::max<long long>(1, std::min<long long>((total + kStoiThreads - 1) / kStoiThreads, 1ll << 20));
}

// The resampler (when the rate is not 10 kHz).
template <class T>
static int stoi_resample(const StoiParams& p, const StoiShape& s, cudaStream_t st) {
  if (s.resample) {
    const long long total = p.rows * 2 * p.L;
    const long long ctas = std::min<long long>((total + kStoiThreads - 1) / kStoiThreads, 1ll << 20);
    PBB_TRY(launch_kernel("stoi_resample_kernel", stoi_resample_kernel<T>, (unsigned)ctas, kStoiThreads, 0, st, p));
  }
  return 0;
}

// The stages shared by the forward and the backward past the resampler: the frame energies, the keep mask and the
// kept-frame list, the band energies.  U: double past the resampler, the input's type at 10 kHz.
template <class U>
static int stoi_envelopes(const StoiParams& p, cudaStream_t st) {
  {
    const long long warps = p.rows * p.F;
    PBB_TRY(launch_kernel("stoi_energy_kernel", stoi_energy_kernel<U>,
                          (unsigned)((warps * 32 + kStoiThreads - 1) / kStoiThreads), kStoiThreads, 0, st, p));
  }
  PBB_TRY(launch_kernel("stoi_compact_kernel", stoi_compact_kernel, (unsigned)p.rows, kStoiCompactThreads, 0, st, p));
  if (p.Mmax > 0) {
    const long long ctas = p.rows * 2 * ((p.Mmax + kStoiFpc - 1) / kStoiFpc);
    PBB_TRY(launch_kernel("stoi_bands_kernel", stoi_bands_kernel<U>, (unsigned)ctas, kStoiThreads, 0, st, p));
  }
  return 0;
}

// One group of rows: the shared stages, then the segment kernel of STOI or (extended) ESTOI, then the values.
template <class T>
static int stoi_group(StoiParams p, const StoiShape& s, bool extended, cudaStream_t st) {
  if (int rc = stoi_resample<T>(p, s, st)) return rc;
  // past the resampler every sample is read from p.sig as double, or from the input as T at 10 kHz
  auto run = [&](auto tag) -> int {
    using U = decltype(tag);
    if (int rc = stoi_envelopes<U>(p, st)) return rc;
    if (extended) {
      PBB_CUDA(cudaFuncSetAttribute(estoi_segment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)kEstoiSmemBytes));
      PBB_TRY(launch_kernel("estoi_segment_kernel", estoi_segment_kernel, (unsigned)(p.rows * p.blocks), kStoiThreads,
                            kEstoiSmemBytes, st, p));
    } else {
      PBB_TRY(launch_kernel("stoi_segment_kernel", stoi_segment_kernel, (unsigned)(p.rows * p.blocks), kStoiThreads, 0,
                            st, p));
    }
    return launch_kernel("stoi_value_kernel", stoi_value_kernel, 1, kStoiThreads, 0, st, p);
  };
  if (s.resample) return run(double{});
  return run(T{});
}

// pbb_stoi (extended = false) and pbb_estoi (extended = true): the same checks, workspace and stage outputs.
static int stoi_call(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
                     const double* taps, int taps_per_phase, long long pre_remove, const double* window,
                     const int* bands, const double* twiddle, long long group, void* workspace,
                     size_t workspace_bytes, double* out, long long* frames, double* resampled, double* energies,
                     long long* status, void* stream, bool extended) {
  StoiShape s;
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(y != nullptr, 2, "y is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64, 3, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(rows > 0 && rows <= 0x7fffffffll / 64, 4, "rows out of range");
  PBB_CHECK_ARG(stoi_shape(n, up, down, &s), 5,
                "n must be in [1, PBB_STOI_MAX_SAMPLES], up / down in lowest terms, and ceil(n up / down) in "
                "(PBB_STOI_FRAME, PBB_STOI_MAX_RESAMPLED]");
  PBB_CHECK_ARG(!s.resample || taps != nullptr, 8, "taps is null");
  PBB_CHECK_ARG(!s.resample || taps_per_phase > 0, 9, "taps_per_phase must be positive");
  PBB_CHECK_ARG(pre_remove >= 0, 10, "pre_remove must not be negative");
  PBB_CHECK_ARG(window != nullptr && bands != nullptr && twiddle != nullptr, 11, "a table is null");
  PBB_CHECK_ARG(group > 0 && group <= PBB_STOI_MAX_GROUP, 14, "group must be in [1, PBB_STOI_MAX_GROUP]");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_stoi_workspace_bytes(group, n, up, down), 15,
                "workspace too small (pbb_stoi_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr, 17, "out is null");
  PBB_CHECK_ARG(status != nullptr, 21, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const StoiLayout l = stoi_layout(group, s);
  char* w = static_cast<char*>(workspace);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(long long), st));
  PBB_CUDA(cudaMemsetAsync(status + 1, 0xff, sizeof(long long), st));
  const size_t esz = dtype == PBB_F32 ? sizeof(float) : sizeof(double);
  for (long long g0 = 0; g0 < rows; g0 += group) {
    const long long g = rows - g0 < group ? rows - g0 : group;
    StoiParams p{};
    p.x = static_cast<const char*>(x) + (size_t)g0 * n * esz;
    p.y = static_cast<const char*>(y) + (size_t)g0 * n * esz;
    p.rows = g;
    p.n = n;
    p.L = s.L;
    p.F = s.F;
    p.Mmax = s.Mmax;
    p.blocks = s.blocks;
    p.up = up;
    p.down = down;
    p.tpp = taps_per_phase;
    p.pre_remove = pre_remove;
    p.taps = taps;
    p.window = window;
    p.bands = bands;
    p.tw = reinterpret_cast<const double2*>(twiddle);
    p.sig = !s.resample ? nullptr
            : resampled ? resampled + (size_t)g0 * 2 * s.L
                        : reinterpret_cast<double*>(w + l.sig);
    p.energy = reinterpret_cast<double*>(w + l.energy);
    p.kept = reinterpret_cast<int*>(w + l.kept);
    p.km = frames ? frames + 2 * g0 : reinterpret_cast<long long*>(w + l.km);
    p.tob = energies ? energies + (size_t)g0 * 2 * kStoiBands * s.Mmax : reinterpret_cast<double*>(w + l.tob);
    p.partial = reinterpret_cast<double*>(w + l.partial);
    p.out = out + g0;
    p.status = status;
    p.row0 = g0;
    p.terms = extended ? kStoiSeg : kStoiBands;
    const int rc = dtype == PBB_F32 ? stoi_group<float>(p, s, extended, st) : stoi_group<double>(p, s, extended, st);
    if (rc) return rc;
  }
  return 0;
}

// ---- backward ----------------------------------------------------------------------------------------------------------
struct StoiBackLayout {
  size_t sig, energy, kept, rank, km, tob, tbar, seg, fbar, total;  // byte offsets
};

static int stoi_jmax(const StoiShape& s) { return s.Mmax >= kStoiSeg ? s.Mmax - kStoiSeg + 1 : 1; }

// The forward's stage buffers (sig also holds the gradient of the 10 kHz signals once the spectral adjoint has read
// it), the rank table, the band-energy gradients, the per-segment scalars and the STFT-frame gradients.
static StoiBackLayout stoi_back_layout(long long group, const StoiShape& s, bool extended) {
  StoiBackLayout l;
  const size_t G = (size_t)group;
  l.sig = 0;
  l.energy = align256(l.sig + (s.resample ? G * 2 * s.L * sizeof(double) : 0));
  l.kept = align256(l.energy + G * s.F * sizeof(double));
  l.rank = align256(l.kept + G * s.F * sizeof(int));
  l.km = align256(l.rank + G * s.F * sizeof(int));
  l.tob = align256(l.km + G * 2 * sizeof(long long));
  l.tbar = align256(l.tob + G * 2 * kStoiBands * s.Mmax * sizeof(double));
  l.seg = align256(l.tbar + G * 2 * kStoiBands * s.Mmax * sizeof(double));
  const size_t per_seg = extended ? kEstoiSegDoubles : kStoiFields * kStoiBands;
  l.fbar = align256(l.seg + G * per_seg * stoi_jmax(s) * sizeof(double));
  l.total = l.fbar + G * 2 * s.Mmax * kStoiFrame * sizeof(double);
  return l;
}

// One group: the forward's stages again, then the adjoint steps from the value back to the input.
template <class T>
static int stoi_backward_group(StoiParams p, StoiGrad q, const StoiShape& s, bool extended, cudaStream_t st) {
  if (int rc = stoi_resample<T>(p, s, st)) return rc;
  auto run = [&](auto tag) -> int {
    using U = decltype(tag);
    if (int rc = stoi_envelopes<U>(p, st)) return rc;
    PBB_CUDA(cudaMemsetAsync(q.rank, 0xff, (size_t)p.rows * p.F * sizeof(int), st));
    PBB_TRY(launch_kernel("stoi_rank_kernel", stoi_rank_kernel, stoi_ctas(p.rows * p.F), kStoiThreads, 0, st, p, q));
    if (p.Mmax >= kStoiSeg) {
      if (extended) {
        PBB_CUDA(cudaFuncSetAttribute(estoi_segment_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kEstoiSmemBytes));
        PBB_TRY(launch_kernel("estoi_segment_prep_kernel", estoi_segment_prep_kernel, (unsigned)(p.rows * p.blocks),
                              kStoiThreads, kEstoiSmemBytes, st, p, q));
      } else {
        PBB_TRY(launch_kernel("stoi_segment_prep_kernel", stoi_segment_prep_kernel, (unsigned)(p.rows * p.blocks),
                              kStoiThreads, 0, st, p, q));
      }
      const unsigned ctas = stoi_ctas(p.rows * kStoiBands * p.Mmax);
      if (extended) {
        PBB_TRY(launch_kernel("estoi_segment_grad_kernel", estoi_segment_grad_kernel, ctas, kStoiThreads, 0, st, p, q));
      } else {
        PBB_TRY(launch_kernel("stoi_segment_grad_kernel", stoi_segment_grad_kernel, ctas, kStoiThreads, 0, st, p, q));
      }
      PBB_TRY(launch_kernel("stoi_spectral_grad_kernel", stoi_spectral_grad_kernel<U>,
                            (unsigned)(p.rows * 2 * ((p.Mmax + kStoiFpc - 1) / kStoiFpc)), kStoiThreads, 0, st, p, q));
    }
    // below 30 STFT frames in every row the kernel only writes zeros
    PBB_TRY(launch_kernel("stoi_removal_grad_kernel", stoi_removal_grad_kernel, stoi_ctas(p.rows * 2 * p.L),
                          kStoiThreads, 0, st, p, q));
    if (s.resample) {
      PBB_TRY(launch_kernel("stoi_resample_grad_kernel", stoi_resample_grad_kernel, stoi_ctas(p.rows * 2 * p.n),
                            kStoiThreads, 0, st, p, q));
    }
    return 0;
  };
  if (s.resample) return run(double{});
  return run(T{});
}

static int stoi_backward_call(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
                              const double* taps, int taps_per_phase, long long pre_remove, const double* window,
                              const int* bands, const double* twiddle, long long group, void* workspace,
                              size_t workspace_bytes, int extended, const double* grad_out, double* grad_x,
                              double* grad_y, void* stream) {
  StoiShape s;
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(y != nullptr, 2, "y is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64, 3, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(rows > 0 && rows <= 0x7fffffffll / 64, 4, "rows out of range");
  PBB_CHECK_ARG(stoi_shape(n, up, down, &s), 5,
                "n must be in [1, PBB_STOI_MAX_SAMPLES], up / down in lowest terms, and ceil(n up / down) in "
                "(PBB_STOI_FRAME, PBB_STOI_MAX_RESAMPLED]");
  PBB_CHECK_ARG(!s.resample || taps != nullptr, 8, "taps is null");
  PBB_CHECK_ARG(!s.resample || taps_per_phase > 0, 9, "taps_per_phase must be positive");
  PBB_CHECK_ARG(pre_remove >= 0, 10, "pre_remove must not be negative");
  PBB_CHECK_ARG(window != nullptr && bands != nullptr && twiddle != nullptr, 11, "a table is null");
  PBB_CHECK_ARG(group > 0 && group <= PBB_STOI_MAX_GROUP, 14, "group must be in [1, PBB_STOI_MAX_GROUP]");
  PBB_CHECK_ARG(extended == 0 || extended == 1, 17, "extended must be 0 or 1");
  PBB_CHECK_ARG(workspace != nullptr &&
                    workspace_bytes >= pbb_stoi_backward_workspace_bytes(group, n, up, down, extended),
                15, "workspace too small (pbb_stoi_backward_workspace_bytes)");
  PBB_CHECK_ARG(grad_out != nullptr, 18, "grad_out is null");
  if (!grad_x && !grad_y) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const StoiBackLayout l = stoi_back_layout(group, s, extended);
  char* w = static_cast<char*>(workspace);
  const size_t esz = dtype == PBB_F32 ? sizeof(float) : sizeof(double);
  for (long long g0 = 0; g0 < rows; g0 += group) {
    const long long g = rows - g0 < group ? rows - g0 : group;
    StoiParams p{};
    p.x = static_cast<const char*>(x) + (size_t)g0 * n * esz;
    p.y = static_cast<const char*>(y) + (size_t)g0 * n * esz;
    p.rows = g;
    p.n = n;
    p.L = s.L;
    p.F = s.F;
    p.Mmax = s.Mmax;
    p.blocks = s.blocks;
    p.up = up;
    p.down = down;
    p.tpp = taps_per_phase;
    p.pre_remove = pre_remove;
    p.taps = taps;
    p.window = window;
    p.bands = bands;
    p.tw = reinterpret_cast<const double2*>(twiddle);
    p.sig = s.resample ? reinterpret_cast<double*>(w + l.sig) : nullptr;
    p.energy = reinterpret_cast<double*>(w + l.energy);
    p.kept = reinterpret_cast<int*>(w + l.kept);
    p.km = reinterpret_cast<long long*>(w + l.km);
    p.tob = reinterpret_cast<double*>(w + l.tob);
    p.row0 = g0;
    p.terms = extended ? kStoiSeg : kStoiBands;
    StoiGrad q{};
    q.gout = grad_out + g0;
    q.Jmax = stoi_jmax(s);
    q.chains = (grad_x ? 1 : 0) | (grad_y ? 2 : 0);
    q.rank = reinterpret_cast<int*>(w + l.rank);
    q.tbar = reinterpret_cast<double*>(w + l.tbar);
    q.seg = reinterpret_cast<double*>(w + l.seg);
    q.fbar = reinterpret_cast<double*>(w + l.fbar);
    q.sbar = p.sig;
    q.gx = grad_x ? grad_x + (size_t)g0 * n : nullptr;
    q.gy = grad_y ? grad_y + (size_t)g0 * n : nullptr;
    const int rc = dtype == PBB_F32 ? stoi_backward_group<float>(p, q, s, extended, st)
                                    : stoi_backward_group<double>(p, q, s, extended, st);
    if (rc) return rc;
  }
  return 0;
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_stoi_workspace_bytes(long long group, long long n, int up, int down) {
  StoiShape s;
  if (group <= 0 || group > PBB_STOI_MAX_GROUP || !stoi_shape(n, up, down, &s)) return 0;
  return stoi_layout(group, s).total;
}

int pbb_stoi(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
             const double* taps, int taps_per_phase, long long pre_remove, const double* window, const int* bands,
             const double* twiddle, long long group, void* workspace, size_t workspace_bytes, double* out,
             long long* frames, double* resampled, double* energies, long long* status, void* stream) {
  return stoi_call(x, y, dtype, rows, n, up, down, taps, taps_per_phase, pre_remove, window, bands, twiddle, group,
                   workspace, workspace_bytes, out, frames, resampled, energies, status, stream, false);
}

int pbb_estoi(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
              const double* taps, int taps_per_phase, long long pre_remove, const double* window, const int* bands,
              const double* twiddle, long long group, void* workspace, size_t workspace_bytes, double* out,
              long long* frames, double* resampled, double* energies, long long* status, void* stream) {
  return stoi_call(x, y, dtype, rows, n, up, down, taps, taps_per_phase, pre_remove, window, bands, twiddle, group,
                   workspace, workspace_bytes, out, frames, resampled, energies, status, stream, true);
}

size_t pbb_stoi_backward_workspace_bytes(long long group, long long n, int up, int down, int extended) {
  StoiShape s;
  if (group <= 0 || group > PBB_STOI_MAX_GROUP || (extended != 0 && extended != 1) || !stoi_shape(n, up, down, &s))
    return 0;
  return stoi_back_layout(group, s, extended).total;
}

int pbb_stoi_backward(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
                      const double* taps, int taps_per_phase, long long pre_remove, const double* window,
                      const int* bands, const double* twiddle, long long group, void* workspace,
                      size_t workspace_bytes, int extended, const double* grad_out, double* grad_x, double* grad_y,
                      void* stream) {
  return stoi_backward_call(x, y, dtype, rows, n, up, down, taps, taps_per_phase, pre_remove, window, bands, twiddle,
                            group, workspace, workspace_bytes, extended, grad_out, grad_x, grad_y, stream);
}

}  // extern "C"
