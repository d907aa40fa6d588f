// C-ABI entry points for SI-SDR and the invasive SxR, pb_bss/evaluation/module_si_sdr.py and sxr_module.py -- see
// include/pbb.h and csrc/sxr.cuh.
#include <algorithm>

#include "common.cuh"
#include "prof.cuh"
#include "sxr.cuh"

namespace pbb {

static bool rows_ok(long long rows, long long n) {
  return rows >= 0 && n >= 0 && rows <= 0x7fffffffll && rows * sxr_chunks(n) <= 0x7fffffffll;
}

template <class T>
static int mean_square_launch(const void* x, long long rows, long long n, double* partial, double* out,
                              cudaStream_t st) {
  const long long chunks = sxr_chunks(n);
  if (chunks > 0) {
    PBB_TRY(launch_kernel("mean_square_chunk_kernel", mean_square_chunk_kernel<T>, (unsigned)(rows * chunks),
                          kSxrThreads, 0, st, static_cast<const T*>(x), n, chunks, partial));
  }
  return launch_kernel("mean_square_row_kernel", mean_square_row_kernel, (unsigned)rows, kSxrThreads, 0, st, partial, n,
                       chunks, out);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

size_t pbb_mean_square_workspace_bytes(long long rows, long long n) {
  if (!rows_ok(rows, n)) return 0;
  return (size_t)(rows * sxr_chunks(n)) * sizeof(double);
}

int pbb_mean_square(const void* x, int dtype, long long rows, long long n, void* workspace, size_t workspace_bytes,
                    double* out, void* stream) {
  PBB_CHECK_ARG(x != nullptr || n == 0 || rows == 0, 1, "x is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64 || dtype == PBB_I16 || dtype == PBB_I32 || dtype == PBB_I64 ||
                    dtype == PBB_C64 || dtype == PBB_C128,
                2, "dtype must be PBB_F32, PBB_F64, PBB_I16, PBB_I32, PBB_I64, PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(rows_ok(rows, n), 3, "rows and n must be non-negative and rows * chunks below 2^31");
  const size_t need = pbb_mean_square_workspace_bytes(rows, n);
  PBB_CHECK_ARG((workspace != nullptr || need == 0) && workspace_bytes >= need, 5,
                "workspace too small (pbb_mean_square_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr || rows == 0, 7, "out is null");
  if (rows == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double* partial = static_cast<double*>(workspace);
  switch (dtype) {
    case PBB_F32: return mean_square_launch<float>(x, rows, n, partial, out, st);
    case PBB_F64: return mean_square_launch<double>(x, rows, n, partial, out, st);
    case PBB_I16: return mean_square_launch<short>(x, rows, n, partial, out, st);
    case PBB_I32: return mean_square_launch<int>(x, rows, n, partial, out, st);
    case PBB_I64: return mean_square_launch<long long>(x, rows, n, partial, out, st);
    case PBB_C64: return mean_square_launch<float2>(x, rows, n, partial, out, st);
    default: return mean_square_launch<double2>(x, rows, n, partial, out, st);
  }
}

size_t pbb_si_sdr_workspace_bytes(long long rows, long long n) {
  if (!rows_ok(rows, n)) return 0;
  return (size_t)(rows * sxr_chunks(n) * 4 + rows) * sizeof(double);
}

int pbb_si_sdr(const double* reference, const double* estimation, const long long* reference_offsets,
               const long long* estimation_offsets, long long rows, long long n, void* workspace,
               size_t workspace_bytes, double* out, void* stream) {
  PBB_CHECK_ARG(reference != nullptr || n == 0 || rows == 0, 1, "reference is null");
  PBB_CHECK_ARG(estimation != nullptr || n == 0 || rows == 0, 2, "estimation is null");
  PBB_CHECK_ARG((reference_offsets != nullptr && estimation_offsets != nullptr) || rows == 0, 3, "an offset table is null");
  PBB_CHECK_ARG(rows_ok(rows, n), 5, "rows and n must be non-negative and rows * chunks below 2^31");
  PBB_CHECK_ARG(workspace_bytes >= pbb_si_sdr_workspace_bytes(rows, n) && (workspace != nullptr || rows == 0), 7,
                "workspace too small (pbb_si_sdr_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr || rows == 0, 9, "out is null");
  if (rows == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long chunks = sxr_chunks(n);
  double* p1 = static_cast<double*>(workspace);
  double* p2 = p1 + rows * chunks * 2;
  double* alpha = p2 + rows * chunks * 2;
  const unsigned grid = (unsigned)(rows * chunks);
  if (chunks > 0) {
    PBB_TRY(launch_kernel("si_sdr_pass1_kernel", si_sdr_pass1_kernel, grid, kSxrThreads, 0, st, reference, estimation,
                          reference_offsets, estimation_offsets, n, chunks, p1));
  }
  PBB_TRY(launch_kernel("si_sdr_alpha_kernel", si_sdr_alpha_kernel, (unsigned)rows, kSxrThreads, 0, st, p1, chunks,
                        alpha));
  if (chunks > 0) {
    PBB_TRY(launch_kernel("si_sdr_pass2_kernel", si_sdr_pass2_kernel, grid, kSxrThreads, 0, st, reference, estimation,
                          reference_offsets, estimation_offsets, n, chunks, alpha, p2));
  }
  return launch_kernel("si_sdr_ratio_kernel", si_sdr_ratio_kernel, (unsigned)rows, kSxrThreads, 0, st, p2, chunks, out);
}

size_t pbb_si_sdr_backward_workspace_bytes(long long rows, long long n) {
  if (!rows_ok(rows, n)) return 0;
  return pbb_si_sdr_workspace_bytes(rows, n) + (size_t)(2 * rows) * sizeof(double);
}

int pbb_si_sdr_backward(const double* reference, const double* estimation, const long long* reference_offsets,
                        const long long* estimation_offsets, long long rows, long long n, const double* grad_out,
                        long long reference_rows, const long long* reference_row_start,
                        const long long* reference_row_index, long long estimation_rows,
                        const long long* estimation_row_start, const long long* estimation_row_index, void* workspace,
                        size_t workspace_bytes, double* grad_reference, double* grad_estimation, void* stream) {
  PBB_CHECK_ARG(reference != nullptr || n == 0 || rows == 0, 1, "reference is null");
  PBB_CHECK_ARG(estimation != nullptr || n == 0 || rows == 0, 2, "estimation is null");
  PBB_CHECK_ARG((reference_offsets != nullptr && estimation_offsets != nullptr) || rows == 0, 3, "an offset table is null");
  PBB_CHECK_ARG(rows_ok(rows, n), 5, "rows and n must be non-negative and rows * chunks below 2^31");
  PBB_CHECK_ARG(grad_out != nullptr || rows == 0, 7, "grad_out is null");
  PBB_CHECK_ARG(grad_reference == nullptr || (reference_rows >= 0 && reference_rows <= rows &&
                                              (rows == 0 || (reference_row_start && reference_row_index))),
                8, "bad reference row table");
  PBB_CHECK_ARG(grad_estimation == nullptr || (estimation_rows >= 0 && estimation_rows <= rows &&
                                               (rows == 0 || (estimation_row_start && estimation_row_index))),
                11, "bad estimation row table");
  PBB_CHECK_ARG(workspace_bytes >= pbb_si_sdr_backward_workspace_bytes(rows, n) && (workspace != nullptr || rows == 0),
                14, "workspace too small (pbb_si_sdr_backward_workspace_bytes)");
  if (rows == 0 || n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long chunks = sxr_chunks(n);
  double* p1 = static_cast<double*>(workspace);
  double* p2 = p1 + rows * chunks * 2;
  double* alpha = p2 + rows * chunks * 2;
  double* coef = alpha + rows;
  const unsigned grid = (unsigned)(rows * chunks);
  // alpha, P and Q exactly as pbb_si_sdr forms them
  PBB_TRY(launch_kernel("si_sdr_pass1_kernel", si_sdr_pass1_kernel, grid, kSxrThreads, 0, st, reference, estimation,
                        reference_offsets, estimation_offsets, n, chunks, p1));
  PBB_TRY(launch_kernel("si_sdr_alpha_kernel", si_sdr_alpha_kernel, (unsigned)rows, kSxrThreads, 0, st, p1, chunks,
                        alpha));
  PBB_TRY(launch_kernel("si_sdr_pass2_kernel", si_sdr_pass2_kernel, grid, kSxrThreads, 0, st, reference, estimation,
                        reference_offsets, estimation_offsets, n, chunks, alpha, p2));
  PBB_TRY(launch_kernel("si_sdr_backward_row_kernel", si_sdr_backward_row_kernel, (unsigned)rows, kSxrThreads, 0, st,
                        p2, chunks, grad_out, coef));
  const auto blocks = [](long long count) {
    return (unsigned)std::min<long long>((count + kSxrThreads - 1) / kSxrThreads, 1ll << 20);
  };
  if (grad_estimation && estimation_rows > 0) {
    PBB_TRY(launch_kernel("si_sdr_backward_kernel", si_sdr_backward_kernel<true>, blocks(estimation_rows * n),
                          kSxrThreads, 0, st, reference, estimation, reference_offsets, estimation_offsets, n, alpha,
                          coef, estimation_rows, estimation_row_start, estimation_row_index, grad_estimation));
  }
  if (grad_reference && reference_rows > 0) {
    PBB_TRY(launch_kernel("si_sdr_backward_kernel", si_sdr_backward_kernel<false>, blocks(reference_rows * n),
                          kSxrThreads, 0, st, reference, estimation, reference_offsets, estimation_offsets, n, alpha,
                          coef, reference_rows, reference_row_start, reference_row_index, grad_reference));
  }
  return 0;
}

int pbb_input_sxr(const double* S, const double* N, int K, int D, int average_sources, int average_channels,
                  double* sdr, double* sir, double* snr, void* stream) {
  PBB_CHECK_ARG(S != nullptr, 1, "S is null");
  PBB_CHECK_ARG(N != nullptr, 2, "N is null");
  PBB_CHECK_ARG(K >= 1 && K <= PBB_SXR_MAX_K, 3, "K must be in [1, PBB_SXR_MAX_K]");
  PBB_CHECK_ARG(D >= 1 && D <= PBB_SXR_MAX_D, 4, "D must be in [1, PBB_SXR_MAX_D]");
  PBB_CHECK_ARG(sdr != nullptr && sir != nullptr && snr != nullptr, 7, "an output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch_kernel("input_sxr_kernel", input_sxr_kernel, 1, 1, 0, st, S, N, K, D, average_sources != 0,
                       average_channels != 0, sdr, sir, snr);
}

static int output_sxr_ctas(int K_source, int K_target) {
  const long long P = sxr_perm_count(K_target, K_source);
  return (int)std::min<long long>((P + kSxrThreads - 1) / kSxrThreads, kSxrPermCtas);
}

size_t pbb_output_sxr_workspace_bytes(int K_source, int K_target) {
  if (K_source < 1 || K_target < K_source || K_target > PBB_SXR_MAX_K) return 0;
  return (size_t)output_sxr_ctas(K_source, K_target) * (sizeof(double) + sizeof(long long));
}

int pbb_output_sxr(const double* S, const double* N, int K_source, int K_target, int average_sources, void* workspace,
                   size_t workspace_bytes, double* sdr, double* sir, double* snr, long long* selection, void* stream) {
  PBB_CHECK_ARG(S != nullptr, 1, "S is null");
  PBB_CHECK_ARG(N != nullptr, 2, "N is null");
  PBB_CHECK_ARG(K_source >= 1 && K_source <= K_target && K_target <= PBB_SXR_MAX_K, 3,
                "need 1 <= K_source <= K_target <= PBB_SXR_MAX_K");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_output_sxr_workspace_bytes(K_source, K_target), 6,
                "workspace too small (pbb_output_sxr_workspace_bytes)");
  PBB_CHECK_ARG(sdr != nullptr && sir != nullptr && snr != nullptr && selection != nullptr, 8, "an output is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int ctas = output_sxr_ctas(K_source, K_target);
  double* best = static_cast<double*>(workspace);
  long long* best_idx = reinterpret_cast<long long*>(best + ctas);
  PBB_TRY(launch_kernel("output_sxr_search_kernel", output_sxr_search_kernel, ctas, kSxrThreads, 0, st, S, K_source,
                        K_target, sxr_perm_count(K_target, K_source), best, best_idx));
  return launch_kernel("output_sxr_kernel", output_sxr_kernel, 1, 1, 0, st, S, N, K_source, K_target, best, best_idx,
                       ctas, average_sources != 0, sdr, sir, snr, selection);
}

}  // extern "C"
