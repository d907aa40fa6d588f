// C-ABI entry points for SRMR, pb_bss/evaluation/module_srmr.py -- see include/pbb.h, csrc/srmr.cuh and
// csrc/fft_large.cuh.
#include "common.cuh"
#include "prof.cuh"
#include "srmr.cuh"

namespace pbb {

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int vad_tiles(long long N) { return (int)((N + kVadTile - 1) / kVadTile); }

template <class T>
static int vad_launch(VadParams p, int normalise, cudaStream_t st) {
  const unsigned ctas = (unsigned)(p.rows * p.tiles), rows = (unsigned)p.rows;
  PBB_TRY(launch_kernel("srmr_vad_max_kernel", vad_tile_kernel<T, VAD_MAX>, ctas, kVadThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_threshold_kernel", vad_row_kernel<T, ROW_THRESHOLD>, rows, kVadRowThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_edges_kernel", vad_tile_kernel<T, VAD_EDGES>, ctas, kVadThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_row_edges_kernel", vad_row_kernel<T, ROW_EDGES>, rows, kVadRowThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_count_kernel", vad_tile_kernel<T, VAD_COUNT>, ctas, kVadThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_offsets_kernel", vad_row_kernel<T, ROW_OFFSETS>, rows, kVadRowThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_compact_kernel", vad_tile_kernel<T, VAD_COMPACT>, ctas, kVadThreads, 0, st, p));
  PBB_TRY(launch_kernel("srmr_vad_mean_kernel", vad_row_kernel<T, ROW_MEAN>, rows, kVadRowThreads, 0, st, p));
  if (normalise) {
    PBB_TRY(launch_kernel("srmr_vad_moments_kernel", vad_norm_kernel<VAD_MOMENTS>, ctas, kVadThreads, 0, st, p));
    PBB_TRY(launch_kernel("srmr_vad_std_kernel", vad_row_kernel<T, ROW_STD>, rows, kVadRowThreads, 0, st, p));
    PBB_TRY(launch_kernel("srmr_vad_normalise_kernel", vad_norm_kernel<VAD_NORMALISE>, ctas, kVadThreads, 0, st, p));
  }
  return 0;
}

struct HilbertLayout {
  FlShape sh;
  size_t tw1, tw2, ks, fft, total;  // byte offsets
};

static HilbertLayout hilbert_layout(long long rows, long long N, long long group) {
  HilbertLayout l;
  l.sh = fl_shape(pbb_srmr_fft_log2(N) - 1);
  l.tw1 = 0;
  l.tw2 = align256(l.tw1 + 2 * (size_t)l.sh.P1() * sizeof(double2));
  l.ks = align256(l.tw2 + 2 * (size_t)l.sh.P2() * sizeof(double2));
  l.fft = align256(l.ks + (size_t)rows * l.sh.P() * sizeof(double));
  l.total = l.fft + (size_t)group * l.sh.P() * sizeof(double2);
  return l;
}

template <class K, class... Args>
static int smem_launch(K kernel, const char* name, long long ctas, size_t smem, cudaStream_t st, Args... args) {
  if (ctas > 0x7fffffffll) {
    set_error("argument: %lld CTAs exceed the grid", ctas);
    return -1;
  }
  PBB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return launch_kernel(name, kernel, (unsigned)ctas, kFlThreads, smem, st, args...);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_srmr_vad_workspace_bytes(long long rows, long long N) {
  if (rows <= 0 || N <= 0) return 0;
  return 5 * align256((size_t)rows * vad_tiles(N) * 8);
}

int pbb_srmr_vad(const void* x, int dtype, long long rows, long long N, double gap, int normalise, void* workspace,
                 size_t workspace_bytes, double* out, long long* nr, double* stats, void* stream) {
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64, 2, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(rows > 0 && rows <= 0x7fffffffll / 1024, 3, "rows out of range");
  PBB_CHECK_ARG(N > 0 && N <= PBB_SRMR_MAX_SAMPLES, 4, "N must be in [1, PBB_SRMR_MAX_SAMPLES]");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_srmr_vad_workspace_bytes(rows, N), 7,
                "workspace too small (pbb_srmr_vad_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr, 9, "out is null");
  PBB_CHECK_ARG(nr != nullptr, 10, "nr is null");
  PBB_CHECK_ARG(stats != nullptr, 11, "stats is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  VadParams p{};
  p.x = x;
  p.rows = rows;
  p.N = N;
  p.tiles = vad_tiles(N);
  p.gap = gap;
  const size_t part = align256((size_t)rows * p.tiles * 8);
  char* w = static_cast<char*>(workspace);
  p.tmax = reinterpret_cast<double*>(w);
  p.first = reinterpret_cast<long long*>(w + part);
  p.last = reinterpret_cast<long long*>(w + 2 * part);
  p.count = reinterpret_cast<long long*>(w + 3 * part);
  p.psum = reinterpret_cast<double*>(w + 4 * part);
  p.stats = stats;
  p.nr = nr;
  p.out = out;
  PBB_CUDA(cudaMemsetAsync(out, 0, (size_t)rows * N * sizeof(double), st));
  if (dtype == PBB_F32) return vad_launch<float>(p, normalise, st);
  return vad_launch<double>(p, normalise, st);
}

int pbb_srmr_fft_log2(long long N) {
  int l = 1;
  while ((1ll << l) < 2 * N - 1) ++l;
  return l;
}

size_t pbb_srmr_hilbert_workspace_bytes(long long rows, long long N, long long group) {
  if (rows <= 0 || N <= 0 || N > PBB_SRMR_MAX_SAMPLES || group <= 0) return 0;
  return hilbert_layout(rows, N, group).total;
}

int pbb_srmr_hilbert(double* y, long long rows, long long N, int n, const long long* nr, long long group,
                     void* workspace, size_t workspace_bytes, void* stream) {
  PBB_CHECK_ARG(y != nullptr, 1, "y is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(N > 0 && N <= PBB_SRMR_MAX_SAMPLES, 3, "N must be in [1, PBB_SRMR_MAX_SAMPLES]");
  PBB_CHECK_ARG(n > 0, 4, "n must be positive");
  PBB_CHECK_ARG(nr != nullptr, 5, "nr is null");
  PBB_CHECK_ARG(group > 0, 6, "group must be positive");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_srmr_hilbert_workspace_bytes(rows, N, group), 7,
                "workspace too small (pbb_srmr_hilbert_workspace_bytes)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const HilbertLayout l = hilbert_layout(rows, N, group);
  const FlShape sh = l.sh;
  char* w = static_cast<char*>(workspace);
  double2* tw1 = reinterpret_cast<double2*>(w + l.tw1);
  double2* tw2 = reinterpret_cast<double2*>(w + l.tw2);
  double* ks = reinterpret_cast<double*>(w + l.ks);
  double2* ws = reinterpret_cast<double2*>(w + l.fft);
  PBB_TRY(launch_kernel("fl_stage_table_kernel", fl_stage_table_kernel, (2 * sh.P1() + 255) / 256, 256, 0, st, tw1,
                        sh.logP1 + 1));
  PBB_TRY(launch_kernel("fl_stage_table_kernel", fl_stage_table_kernel, (2 * sh.P2() + 255) / 256, 256, 0, st, tw2,
                        sh.logP2 + 1));
  const size_t col_smem = 2 * (size_t)sh.cols * sh.P1() * sizeof(double2);
  const size_t row_smem = 4 * (size_t)sh.P2() * sizeof(double2);
  const FlForwardStore fwd{ws, sh.logP, sh.logP2};
  // the kernel spectrum of every row
  for (long long g0 = 0; g0 < rows; g0 += group) {
    const long long g = rows - g0 < group ? rows - g0 : group;
    int rc = smem_launch(fl_column_kernel<-1, HilbertKernelLoad, FlForwardStore>, "srmr_hilbert_kernel_column_kernel",
                         g * sh.col_tiles(), col_smem, st, sh, (const double2*)tw1,
                         HilbertKernelLoad{nr, g0, 2 * sh.P()}, fwd);
    if (rc) return rc;
    rc = smem_launch(fl_row_pair_kernel<KernelSpectrumOp>, "srmr_hilbert_kernel_row_kernel", g * sh.row_pairs(),
                     row_smem, st, sh, (const double2*)tw2, ws, KernelSpectrumOp{ks, sh, g0});
    if (rc) return rc;
  }
  // every sequence: forward, multiply, inverse, envelope
  const long long seqs = (long long)n * rows;
  for (long long g0 = 0; g0 < seqs; g0 += group) {
    const long long g = seqs - g0 < group ? seqs - g0 : group;
    int rc = smem_launch(fl_column_kernel<-1, HilbertSignalLoad, FlForwardStore>, "srmr_hilbert_column_kernel",
                         g * sh.col_tiles(), col_smem, st, sh, (const double2*)tw1,
                         HilbertSignalLoad{y, nr, g0, rows, N}, fwd);
    if (rc) return rc;
    rc = smem_launch(fl_row_pair_kernel<ConvolveOp>, "srmr_hilbert_row_kernel", g * sh.row_pairs(), row_smem, st, sh,
                     (const double2*)tw2, ws, ConvolveOp{ks, sh, g0, rows});
    if (rc) return rc;
    rc = smem_launch(fl_column_kernel<1, FlWorkspaceLoad, EnvelopeStore>, "srmr_hilbert_envelope_kernel",
                     g * sh.col_tiles(), col_smem, st, sh, (const double2*)tw1, FlWorkspaceLoad{ws, sh.logP},
                     EnvelopeStore{y, nr, g0, rows, N, sh.logP2});
    if (rc) return rc;
  }
  return 0;
}

size_t pbb_srmr_means_workspace_bytes(long long rows, long long N, int n, int hop) {
  if (rows <= 0 || N <= 0 || n <= 0 || hop <= 0) return 0;
  const long long blocks = (N + hop - 1) / hop + 3;
  return (size_t)rows * n * 8 * blocks * 6 * sizeof(double);
}

int pbb_srmr_means(const double* env, long long rows, long long N, int n, const long long* nr, int hop,
                   const double* coef, const double* transition, const double* window, void* workspace,
                   size_t workspace_bytes, double* means, void* stream) {
  PBB_CHECK_ARG(env != nullptr, 1, "env is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(N > 0 && N <= PBB_SRMR_MAX_SAMPLES, 3, "N must be in [1, PBB_SRMR_MAX_SAMPLES]");
  PBB_CHECK_ARG(n > 0, 4, "n must be positive");
  PBB_CHECK_ARG(nr != nullptr, 5, "nr is null");
  PBB_CHECK_ARG(hop > 0, 6, "hop must be positive");
  PBB_CHECK_ARG(coef != nullptr && transition != nullptr && window != nullptr, 7, "a table is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_srmr_means_workspace_bytes(rows, N, n, hop), 10,
                "workspace too small (pbb_srmr_means_workspace_bytes)");
  PBB_CHECK_ARG(means != nullptr, 12, "means is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ModParams p{};
  p.env = env;
  p.nr = nr;
  p.rows = rows;
  p.N = N;
  p.seqs = rows * n;
  p.n = n;
  p.S = hop;
  p.blocks = (int)((N + hop - 1) / hop + 3);
  p.coef = coef;
  p.trans = transition;
  p.window = window;
  p.state = static_cast<double*>(workspace);
  p.quarter = p.state + p.seqs * 8 * p.blocks * 2;
  p.means = means;
  const long long units = p.seqs * 8 * p.blocks, filters = p.seqs * 8;
  if ((units + 255) / 256 > 0x7fffffffll) {
    set_error("argument: %lld blocks exceed the grid", units);
    return -1;
  }
  PBB_TRY(launch_kernel("srmr_block_state_kernel", srmr_block_kernel<false>, (unsigned)((units + 255) / 256), 256, 0,
                        st, p));
  PBB_TRY(launch_kernel("srmr_carry_kernel", srmr_carry_kernel, (unsigned)((filters + 255) / 256), 256, 0, st, p));
  PBB_TRY(launch_kernel("srmr_block_energy_kernel", srmr_block_kernel<true>, (unsigned)((units + 255) / 256), 256, 0,
                        st, p));
  return launch_kernel("srmr_mean_kernel", srmr_mean_kernel, (unsigned)((filters + 255) / 256), 256, 0, st, p);
}

int pbb_srmr_ratio(const double* means, long long rows, int n, const double* erb, const double* cutoff, double* out,
                   void* stream) {
  PBB_CHECK_ARG(means != nullptr, 1, "means is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(n > 0, 3, "n must be positive");
  PBB_CHECK_ARG(erb != nullptr && cutoff != nullptr, 4, "erb or cutoff is null");
  PBB_CHECK_ARG(out != nullptr, 6, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("srmr_ratio_kernel", srmr_ratio_kernel, (unsigned)((rows + 127) / 128), 128, 0, st, means, rows,
                       n, erb, cutoff, out);
}

}  // extern "C"
