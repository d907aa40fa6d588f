// C-ABI entry points for the oracle masks (pb_bss/extraction/mask_module.py) and the array geometry
// (pb_bss/extraction/beamform_utils.py) -- see include/pbb.h and csrc/mask.cuh.
#include "common.cuh"
#include "mask.cuh"
#include "prof.cuh"

namespace pbb {

static bool layout_ok(const pbb_mask_layout* L) {
  if (L == nullptr || L->nd < 0 || L->nd > PBB_MASK_MAX_DIMS) return false;
  for (int a = 0; a < L->nd; ++a)
    if (L->shape[a] < 1) return false;
  return true;
}

static long long layout_count(const pbb_mask_layout* L) {
  long long n = 1;
  for (int a = 0; a < L->nd; ++a) n *= L->shape[a];
  return n;
}

static unsigned grid_for(long long n, int threads) {
  long long g = (n + threads - 1) / threads;
  if (g > (1ll << 20)) g = 1ll << 20;
  return (unsigned)(g < 1 ? 1 : g);
}

static bool dtype_ok(int dtype) {
  return dtype == PBB_C64 || dtype == PBB_C128 || dtype == PBB_F32 || dtype == PBB_F64;
}

// returns fn(TI*) with the signal pointer cast to its element type
template <class Fn>
static int with_input(int dtype, const void* p, Fn&& fn) {
  switch (dtype) {
    case PBB_C128: return fn(reinterpret_cast<const double2*>(p));
    case PBB_C64: return fn(reinterpret_cast<const float2*>(p));
    case PBB_F64: return fn(reinterpret_cast<const double*>(p));
    default: return fn(reinterpret_cast<const float*>(p));
  }
}

static bool is32(int dtype) { return dtype == PBB_C64 || dtype == PBB_F32; }

static size_t sel_state_offset(long long rows, long long n) { return ((size_t)rows * n * sizeof(double) + 255) & ~(size_t)255; }
static size_t sel_hist_offset(long long rows, long long n) {
  return sel_state_offset(rows, n) + (((size_t)rows * 2 * sizeof(SelState) + 255) & ~(size_t)255);
}

template <class TI, class TO>
static int row_select_launch(const TI* x, int D, long long sD, const pbb_mask_layout* rows,
                             const pbb_mask_layout* elems, const RowSelParams& p, TO* out, void* scratch,
                             size_t scratch_bytes, int* status, cudaStream_t st) {
  const long long nrows = layout_count(rows), n = layout_count(elems);
  if (n <= PBB_ROW_SELECT_SHORT_MAX) {
    int R = 1;
    while (R * 2 <= 32 && (long long)R * 2 * n <= kSelTileValues) R *= 2;
    // a row stride of 1 (the frequency axis of an STFT): walk the tile row-fastest so the loads coalesce
    const int rowfast = rows->nd > 0 && rows->in_stride[rows->nd - 1] == 1 && R > 1;
    const size_t smem = (size_t)R * n * sizeof(double) + R * sizeof(double) + (size_t)kSelWarps * kSelHistBytes;
    PBB_CUDA(cudaFuncSetAttribute(row_select_short_kernel<TI, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    return launch_kernel("row_select_short_kernel", row_select_short_kernel<TI, TO>, (unsigned)((nrows + R - 1) / R),
                         kSelWarps * 32, smem, st, x, D, sD, *rows, nrows, *elems, (int)n, R, rowfast, p, out, status);
  }
  if (scratch == nullptr || scratch_bytes < pbb_row_select_scratch_bytes(nrows, n)) {
    set_error("argument: scratch too small for rows of %lld elements (pbb_row_select_scratch_bytes)", n);
    return -1;
  }
  double* vals = reinterpret_cast<double*>(scratch);
  SelState* state = reinterpret_cast<SelState*>(reinterpret_cast<unsigned char*>(scratch) + sel_state_offset(nrows, n));
  unsigned char* hist = reinterpret_cast<unsigned char*>(scratch) + sel_hist_offset(nrows, n);
  PBB_CUDA(cudaMemsetAsync(hist, 0, (size_t)nrows * kSelHistBytes, st));
  // enough CTAs per row to fill the GPU about twice, each with at least 4096 elements
  long long chunks = (264 + nrows - 1) / nrows;
  if (chunks > (n + 4095) / 4096) chunks = (n + 4095) / 4096;
  if (chunks < 1) chunks = 1;
  // the row is blockIdx.x / chunks: rows < 2^31 and chunks * rows <= rows + 263, so the grid never exceeds grid.x
  const unsigned grid = (unsigned)(chunks * nrows);
  PBB_TRY(launch_kernel("row_state_init_kernel", row_state_init_kernel, grid_for(nrows, 128), 128, 0, st, nrows, n, p,
                        state));
  PBB_TRY(launch_kernel("row_gather_kernel", row_gather_kernel<TI>, grid, 256, 0, st, x, D, sD, *rows, *elems, n,
                        (int)chunks, p, vals, state));
  const int queries = p.lorenz ? 1 : 2;
  for (int q = 0; q < queries; ++q) {
    for (int pass = 0; pass < kSelPasses; ++pass) {
      PBB_TRY(launch_kernel("row_hist_kernel", row_hist_kernel, grid, 256, 0, st, vals, n, (int)chunks, pass, q,
                            p.lorenz, state, hist));
      PBB_TRY(launch_kernel("row_decide_kernel", row_decide_kernel, (unsigned)nrows, 32, 0, st, n, pass, q, p, state,
                            hist));
    }
  }
  return launch_kernel("row_apply_kernel", row_apply_kernel<TO>, grid, 256, 0, st, vals, *rows, *elems, n, (int)chunks,
                       p, state, out, status);
}

template <class TI>
static int row_select_dispatch(int dtype, const TI* x, int D, long long sD, const pbb_mask_layout* rows,
                               const pbb_mask_layout* elems, const RowSelParams& p, void* out, void* scratch,
                               size_t scratch_bytes, int* status, cudaStream_t st) {
  if (is32(dtype))
    return row_select_launch(x, D, sD, rows, elems, p, reinterpret_cast<float*>(out), scratch, scratch_bytes, status,
                             st);
  return row_select_launch(x, D, sD, rows, elems, p, reinterpret_cast<double*>(out), scratch, scratch_bytes, status,
                           st);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

int pbb_source_mask(const void* signal, int dtype, int kind, int K, int D, long long source_stride,
                    long long sensor_stride, long long out_source_stride, const pbb_mask_layout* rest, double eps,
                    void* out, void* stream) {
  PBB_CHECK_ARG(signal != nullptr, 1, "signal is null");
  PBB_CHECK_ARG(dtype_ok(dtype), 2, "bad dtype");
  PBB_CHECK_ARG(kind >= PBB_MASK_IDEAL_BINARY && kind <= PBB_MASK_IDEAL_COMPLEX, 3, "bad mask kind");
  PBB_CHECK_ARG(K > 0, 4, "K must be positive");
  PBB_CHECK_ARG(D > 0 && (D == 1 || kind <= PBB_MASK_WIENER_LIKE), 5,
                "sensor pooling (D > 1) is defined for the binary and Wiener-like masks only");
  PBB_CHECK_ARG(layout_ok(rest), 9, "bad layout");
  PBB_CHECK_ARG(out != nullptr, 11, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long n = layout_count(rest);
  const unsigned grid = grid_for(n, 256);
  return with_input(dtype, signal, [&](auto x) {
    using TI = std::remove_const_t<std::remove_pointer_t<decltype(x)>>;
    const bool complex_out = kind == PBB_MASK_IDEAL_COMPLEX && IsComplex<TI>::value;
    if (complex_out && is32(dtype))
      return launch_kernel("source_mask_kernel", source_mask_kernel<TI, float2>, grid, 256, 0, st, x, kind, K, D,
                           source_stride, sensor_stride, out_source_stride, *rest, n, eps,
                           reinterpret_cast<float2*>(out));
    if (complex_out)
      return launch_kernel("source_mask_kernel", source_mask_kernel<TI, double2>, grid, 256, 0, st, x, kind, K, D,
                           source_stride, sensor_stride, out_source_stride, *rest, n, eps,
                           reinterpret_cast<double2*>(out));
    if (is32(dtype))
      return launch_kernel("source_mask_kernel", source_mask_kernel<TI, float>, grid, 256, 0, st, x, kind, K, D,
                           source_stride, sensor_stride, out_source_stride, *rest, n, eps,
                           reinterpret_cast<float*>(out));
    return launch_kernel("source_mask_kernel", source_mask_kernel<TI, double>, grid, 256, 0, st, x, kind, K, D,
                         source_stride, sensor_stride, out_source_stride, *rest, n, eps,
                         reinterpret_cast<double*>(out));
  });
}

size_t pbb_row_select_scratch_bytes(long long rows, long long n) {
  if (rows <= 0 || n <= 0) return 0;
  return sel_hist_offset(rows, n) + (size_t)rows * kSelHistBytes;
}

int pbb_lorenz_mask(const void* signal, int dtype, int D, long long sensor_stride, const pbb_mask_layout* rows,
                    const pbb_mask_layout* elems, double lorenz_fraction, double mask_low, double mask_high,
                    void* out, void* scratch, size_t scratch_bytes, int* status, void* stream) {
  PBB_CHECK_ARG(signal != nullptr, 1, "signal is null");
  PBB_CHECK_ARG(dtype_ok(dtype), 2, "bad dtype");
  PBB_CHECK_ARG(D > 0, 3, "D must be positive");
  PBB_CHECK_ARG(layout_ok(rows) && layout_count(rows) < (1ll << 31), 5, "bad row layout");
  PBB_CHECK_ARG(layout_ok(elems), 6, "bad element layout");
  PBB_CHECK_ARG(out != nullptr, 10, "out is null");
  PBB_CHECK_ARG(status != nullptr, 13, "status is null");
  RowSelParams p{};
  p.lorenz = 1;
  p.fraction = lorenz_fraction;
  p.mask_low = mask_low;
  p.mask_high = mask_high;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int rc = with_input(dtype, signal, [&](auto x) {
    return row_select_dispatch(dtype, x, D, sensor_stride, rows, elems, p, out, scratch, scratch_bytes, status, st);
  });
  if (rc == -1) return -11;
  return rc;
}

int pbb_quantile_mask(const void* signal, int dtype, const pbb_mask_layout* rows, const pbb_mask_layout* elems,
                      long long k_lower, long long k_upper, double gamma, double one_minus_gamma, int below,
                      double mask_low, double mask_high, void* out, void* scratch, size_t scratch_bytes,
                      void* stream) {
  PBB_CHECK_ARG(signal != nullptr, 1, "signal is null");
  PBB_CHECK_ARG(dtype_ok(dtype), 2, "bad dtype");
  PBB_CHECK_ARG(layout_ok(rows) && layout_count(rows) < (1ll << 31), 3, "bad row layout");
  PBB_CHECK_ARG(layout_ok(elems), 4, "bad element layout");
  const long long n = layout_ok(elems) ? layout_count(elems) : 0;
  PBB_CHECK_ARG(k_lower >= 0 && k_lower < n, 5, "k_lower out of range");
  PBB_CHECK_ARG(k_upper >= k_lower && k_upper < n, 6, "k_upper out of range");
  PBB_CHECK_ARG(out != nullptr, 12, "out is null");
  RowSelParams p{};
  p.lorenz = 0;
  p.below = below != 0;
  p.f32 = is32(dtype);
  p.k_lower = k_lower;
  p.k_upper = k_upper;
  p.gamma = gamma;
  p.one_minus_gamma = one_minus_gamma;
  p.mask_low = mask_low;
  p.mask_high = mask_high;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int rc = with_input(dtype, signal, [&](auto x) {
    return row_select_dispatch(dtype, x, 1, 0, rows, elems, p, out, scratch, scratch_bytes, nullptr, st);
  });
  if (rc == -1) return -13;
  return rc;
}

int pbb_biased_binary_mask(const void* signal, int dtype, long long component_stride, long long out_component_stride,
                           const pbb_mask_layout* rest, int L, const double* speech_div, const double* noise_div,
                           const unsigned char* force, void* out, void* stream) {
  PBB_CHECK_ARG(signal != nullptr, 1, "signal is null");
  PBB_CHECK_ARG(dtype_ok(dtype), 2, "bad dtype");
  PBB_CHECK_ARG(layout_ok(rest), 5, "bad layout");
  PBB_CHECK_ARG(L > 0, 6, "L must be positive");
  PBB_CHECK_ARG(speech_div && noise_div && force, 7, "threshold arrays are null");
  PBB_CHECK_ARG(out != nullptr, 10, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long n = layout_count(rest);
  return with_input(dtype, signal, [&](auto x) {
    using TI = std::remove_const_t<std::remove_pointer_t<decltype(x)>>;
    return launch_kernel("biased_binary_kernel", biased_binary_kernel<TI>, grid_for(n, 256), 256, 0, st, x,
                         component_stride, out_component_stride, *rest, n, L, speech_div, noise_div, force,
                         reinterpret_cast<unsigned char*>(out));
  });
}

int pbb_steering_vector(const double* tdoa, int A, int M, const double* freq, int F, int normalize, void* out,
                        void* stream) {
  PBB_CHECK_ARG(tdoa != nullptr, 1, "tdoa is null");
  PBB_CHECK_ARG(A > 0 && M > 0, 2, "bad shape");
  PBB_CHECK_ARG(freq != nullptr, 4, "freq is null");
  PBB_CHECK_ARG(F > 0, 5, "F must be positive");
  PBB_CHECK_ARG(out != nullptr, 7, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("steering_vector_kernel", steering_vector_kernel, grid_for((long long)A * F, 128), 128, 0, st,
                       tdoa, A, M, freq, F, normalize, reinterpret_cast<double2*>(out));
}

int pbb_diffuse_noise_coherence(const double* distances, int D, const double* freq, int F, double sound_velocity,
                                double* out, void* stream) {
  PBB_CHECK_ARG(distances != nullptr, 1, "distances is null");
  PBB_CHECK_ARG(D > 0, 2, "D must be positive");
  PBB_CHECK_ARG(freq != nullptr, 3, "freq is null");
  PBB_CHECK_ARG(F > 0, 4, "F must be positive");
  PBB_CHECK_ARG(out != nullptr, 6, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("diffuse_coherence_kernel", diffuse_coherence_kernel, grid_for((long long)F * D * D, 256), 256,
                       0, st, distances, D, freq, F, sound_velocity, out);
}

int pbb_array_geometry(int mode, const double* points, int S, const double* sensor, int M, int reference_channel,
                       double sound_velocity, double* out, void* stream) {
  PBB_CHECK_ARG(mode == 0 || mode == 1, 1, "mode must be 0 (near field) or 1 (far field)");
  PBB_CHECK_ARG(points != nullptr, 2, "points is null");
  PBB_CHECK_ARG(S > 0, 3, "S must be positive");
  PBB_CHECK_ARG(sensor != nullptr, 4, "sensor is null");
  PBB_CHECK_ARG(M > 0, 5, "M must be positive");
  PBB_CHECK_ARG(mode == 0 || (reference_channel >= 0 && reference_channel < M), 6, "reference_channel out of range");
  PBB_CHECK_ARG(out != nullptr, 8, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("array_geometry_kernel", array_geometry_kernel, grid_for((long long)S * M, 128), 128, 0, st,
                       mode, points, S, sensor, M, reference_channel, sound_velocity, out);
}

}  // extern "C"
