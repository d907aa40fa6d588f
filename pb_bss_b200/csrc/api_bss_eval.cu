// C-ABI entry points for BSS Eval, pb_bss/evaluation/module_mir_eval.py -- see include/pbb.h and csrc/bss_eval.cuh.
#include "common.cuh"
#include "prof.cuh"
#include "bss_eval.cuh"

namespace pbb {

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static BssShape bss_shape(long long T, int K, int E) {
  BssShape s{};
  s.T = T;
  s.K = K;
  s.E = E;
  s.S = K + E;
  s.N = K * kBssL;
  long long span = (T + kCorrParts - 1) / kCorrParts;
  span = (span + kCorrChunk - 1) / kCorrChunk * kCorrChunk;
  s.span = span;
  s.parts = (int)((T + span - 1) / span);
  s.tiles = (T + kBssL - 1 + kProjTile - 1) / kProjTile;
  return s;
}

static int sums_width(int E) { return E > 8 ? 16 : 8; }

struct BssLayout {
  size_t flags, part, R, G, Gb, sums, total;  // byte offsets
};

static BssLayout bss_layout(long long group, const BssShape& s) {
  BssLayout l;
  l.flags = 0;
  l.part = align256(l.flags + (size_t)group * sizeof(int));
  l.R = align256(l.part + (size_t)group * s.K * s.parts * s.S * kBssL * sizeof(double));
  l.G = align256(l.R + (size_t)group * s.K * s.S * kBssL * sizeof(double));
  l.Gb = align256(l.G + (size_t)group * s.N * (s.N + kRhsPad) * sizeof(double));
  const size_t gb = s.K > 1 ? (size_t)group * s.K * kBssL * (kBssL + kRhsPad) * sizeof(double) : 0;
  l.sums = align256(l.Gb + gb);
  l.total = l.sums + (size_t)group * s.tiles * (s.K + 1) * 3 * sums_width(s.E) * sizeof(double);
  return l;
}

static bool valid_shape(long long T, int K, int E) {
  return K >= 1 && K <= PBB_BSS_EVAL_MAX_SOURCES && (E == K || E == K + 1) && T >= 1 &&
         T <= PBB_BSS_EVAL_MAX_SAMPLES;
}

// Blocked LU of `mats` augmented matrices, then the back substitution of their right-hand columns
static int lu_solve(LuBatch b, long long mats, cudaStream_t st) {
  for (int k0 = 0; k0 < b.n; k0 += kPanel) {
    PBB_TRY(launch_kernel("bss_lu_panel_kernel", bss_lu_panel_kernel, (unsigned)mats, 512, 0, st, b, k0));
    const int cols = b.ncols - k0 - kPanel, rows = b.n - k0 - kPanel;
    if (cols > 0) {
      PBB_TRY(launch_kernel("bss_lu_trsm_kernel", bss_lu_trsm_kernel, dim3((cols + 127) / 128, (unsigned)mats), 128, 0,
                            st, b, k0));
    }
    if (cols > 0 && rows > 0) {
      PBB_TRY(launch_kernel("bss_lu_update_kernel", bss_lu_update_kernel,
                            dim3((cols + 63) / 64, (rows + 63) / 64, (unsigned)mats), 128, 0, st, b, k0));
    }
  }
  return launch_kernel("bss_backsub_kernel", bss_backsub_kernel, (unsigned)mats, 256, 0, st, b);
}

template <int NS>
static int corr_launch(const double* x, const BssShape& s, long long g, double* part, cudaStream_t st) {
  return launch_kernel("bss_corr_kernel", bss_corr_kernel<NS>, dim3((unsigned)s.parts, (unsigned)s.K, (unsigned)g), 256,
                       0, st, x, s, part);
}

template <int NS>
static int project_launch(const double* x, const BssShape& s, long long g, const double* G, const double* Gb,
                          double* sums, cudaStream_t st) {
  const size_t smem = sizeof(ProjSmem<NS>);
  PBB_CUDA(cudaFuncSetAttribute(bss_project_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel("bss_project_kernel", bss_project_kernel<NS>, dim3((unsigned)s.tiles, (unsigned)g), 256, smem,
                       st, x, s, G, Gb, sums);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_bss_eval_workspace_bytes(long long group, int K, int E, long long T) {
  if (group <= 0 || group > PBB_BSS_EVAL_MAX_GROUP || !valid_shape(T, K, E)) return 0;
  return bss_layout(group, bss_shape(T, K, E)).total;
}

int pbb_bss_eval(const double* x, long long items, int K, int E, long long T, int compute_permutation,
                 long long group, void* workspace, size_t workspace_bytes, double* sdr, double* sir, double* sar,
                 long long* selection, double* pairs, long long* status, void* stream) {
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(items > 0, 2, "items must be positive");
  PBB_CHECK_ARG(K >= 1 && K <= PBB_BSS_EVAL_MAX_SOURCES, 3, "K must be in [1, PBB_BSS_EVAL_MAX_SOURCES]");
  PBB_CHECK_ARG(E == K || E == K + 1, 4, "E must be K or K + 1");
  PBB_CHECK_ARG(T >= 1 && T <= PBB_BSS_EVAL_MAX_SAMPLES, 5, "T must be in [1, PBB_BSS_EVAL_MAX_SAMPLES]");
  PBB_CHECK_ARG(compute_permutation || E == K, 6, "E = K + 1 needs compute_permutation");
  PBB_CHECK_ARG(group > 0 && group <= PBB_BSS_EVAL_MAX_GROUP, 7, "group must be in [1, PBB_BSS_EVAL_MAX_GROUP]");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_bss_eval_workspace_bytes(group, K, E, T), 8,
                "workspace too small (pbb_bss_eval_workspace_bytes)");
  PBB_CHECK_ARG(sdr != nullptr && sir != nullptr && sar != nullptr, 10, "sdr, sir or sar is null");
  PBB_CHECK_ARG(selection != nullptr || !compute_permutation, 13, "selection is null");
  PBB_CHECK_ARG(status != nullptr, 15, "status is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const BssShape s = bss_shape(T, K, E);
  const BssLayout l = bss_layout(group, s);
  char* w = static_cast<char*>(workspace);
  int* flags = reinterpret_cast<int*>(w + l.flags);
  double* part = reinterpret_cast<double*>(w + l.part);
  double* R = reinterpret_cast<double*>(w + l.R);
  double* G = reinterpret_cast<double*>(w + l.G);
  double* Gb = K > 1 ? reinterpret_cast<double*>(w + l.Gb) : nullptr;
  double* sums = reinterpret_cast<double*>(w + l.sums);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(long long), st));
  for (long long i0 = 0; i0 < items; i0 += group) {
    const long long g = items - i0 < group ? items - i0 : group;
    const double* xg = x + i0 * s.S * T;
    PBB_CUDA(cudaMemsetAsync(flags, 0, (size_t)g * sizeof(int), st));
    PBB_TRY(launch_kernel("bss_check_kernel", bss_check_kernel, dim3((unsigned)s.S, (unsigned)g), 256, 0, st, xg, T,
                          s.S, flags));
    const int ns = (s.S + 7) / 8;
    int rc = ns == 1 ? corr_launch<1>(xg, s, g, part, st)
                     : ns == 2 ? corr_launch<2>(xg, s, g, part, st) : corr_launch<3>(xg, s, g, part, st);
    if (rc) return rc;
    {
      const long long n = g * s.K * s.S * kBssL;
      PBB_TRY(launch_kernel("bss_corr_reduce_kernel", bss_corr_reduce_kernel, (unsigned)((n + 255) / 256), 256, 0, st,
                            part, s, g, R));
    }
    {
      const long long n = g * s.N * (long long)(s.N + kRhsPad);
      PBB_TRY(launch_kernel("bss_assemble_kernel", bss_assemble_kernel, (unsigned)((n + 255) / 256), 256, 0, st, R, s,
                            g, G, Gb));
    }
    rc = lu_solve(LuBatch{G, s.N, s.N + kRhsPad, s.N + E, 1, flags}, g, st);
    if (rc) return rc;
    if (K > 1) {
      rc = lu_solve(LuBatch{Gb, kBssL, kBssL + kRhsPad, kBssL + E, K, flags}, g * K, st);
      if (rc) return rc;
    }
    rc = E > 8 ? project_launch<2>(xg, s, g, G, Gb, sums, st) : project_launch<1>(xg, s, g, G, Gb, sums, st);
    if (rc) return rc;
    PBB_TRY(launch_kernel("bss_ratio_kernel", bss_ratio_kernel, (unsigned)g, 256, 0, st, sums, s, compute_permutation,
                          flags, i0, sdr, sir, sar, selection, pairs));
    PBB_TRY(launch_kernel("bss_status_kernel", bss_status_kernel, 1, 32, 0, st, flags, g, i0, status));
  }
  return 0;
}

}  // extern "C"
