// C-ABI entry points for the building blocks of pb_bss.distribution.mixture_model_utils / utils, pb_bss.utils and
// pb_bss.evaluation.sxr_module -- see include/pbb.h and csrc/mm_utils.cuh:
//   pbb_affiliation_nd      log_pdf_to_affiliation for any K and any strides   (mixture_model_utils.py:7-55)
//   pbb_axis_sum            sum / mean over a set of axes                        (:133-203, sxr_module.py:13-14)
//   pbb_unit_norm           _unit_norm for every vector ord                      (distribution/utils.py:223-256)
//   pbb_reduce_workspace_bytes  the partials of the chunked reductions of both
//   pbb_force_hermitian     (A + A^H) / 2                                        (distribution/utils.py:318-330)
//   pbb_abs_square          re^2 + im^2                                          (utils.py:314-336)
//   pbb_labels_to_one_hot   one-hot in its final layout                          (utils.py:234-311)
//   pbb_scale_nd            N *= factor                                          (sxr_module.py:51-78)
#include <cstring>

#include "common.cuh"
#include "mm_utils.cuh"
#include "prof.cuh"

namespace pbb {

static bool layout_ok(const pbb_nd_layout* L, long long* count) {
  if (L == nullptr || L->nd < 0 || L->nd > PBB_ND_MAX_DIMS) return false;
  long long n = 1;
  for (int d = 0; d < L->nd; ++d) {
    if (L->shape[d] < 0) return false;
    n *= L->shape[d];
  }
  *count = n;
  return true;
}

static unsigned blocks_for(long long n) { return (unsigned)((n + kNdThreads - 1) / kNdThreads); }

static bool is_float(int dtype) { return dtype == PBB_F32 || dtype == PBB_F64; }
static bool is_float_or_complex(int dtype) { return is_float(dtype) || dtype == PBB_C64 || dtype == PBB_C128; }

static long long red_chunks(long long outs, long long n) {
  const long long len = red_chunk_len(outs, n);
  return (n + len - 1) / len > 1 ? (n + len - 1) / len : 1;
}

template <class T, bool CPLX, class TO>
static int reduce_launch(const void* x, const double* mul, const pbb_nd_layout& O, const pbb_nd_layout& R,
                         long long outs, long long n, const RedOp& op, double* partial, void* out, cudaStream_t st) {
  const long long len = red_chunk_len(outs, n), chunks = red_chunks(outs, n);
  const bool warp = len >= 32;
  const long long threads = outs * chunks * (warp ? 32 : 1);
  const auto kern = warp ? reduce_kernel<T, CPLX, TO, true> : reduce_kernel<T, CPLX, TO, false>;
  PBB_TRY(launch_kernel(warp ? "reduce_kernel<warp>" : "reduce_kernel", kern, blocks_for(threads), kNdThreads, 0, st,
                        static_cast<const T*>(x), mul, O, R, outs, n, len, chunks, op, partial, static_cast<TO*>(out)));
  if (chunks > 1)
    PBB_TRY(launch_kernel("red_finish_kernel", red_finish_kernel<TO>, blocks_for(outs * 32), kNdThreads, 0, st, partial,
                          O, outs, chunks, op, static_cast<TO*>(out)));
  return 0;
}

template <class TO>
static int reduce_dispatch(const void* x, int dtype, const double* mul, const pbb_nd_layout& O,
                           const pbb_nd_layout& R, long long outs, long long n, const RedOp& op, double* partial,
                           void* out, cudaStream_t st) {
  switch (dtype) {
    case PBB_F32: return reduce_launch<float, false, TO>(x, mul, O, R, outs, n, op, partial, out, st);
    case PBB_F64: return reduce_launch<double, false, TO>(x, mul, O, R, outs, n, op, partial, out, st);
    case PBB_C64: return reduce_launch<float, true, TO>(x, mul, O, R, outs, n, op, partial, out, st);
    default: return reduce_launch<double, true, TO>(x, mul, O, R, outs, n, op, partial, out, st);
  }
}

template <class T, bool CPLX>
static int divide_launch(const void* x, const double* norm, const pbb_nd_layout& L, long long total, void* out,
                         cudaStream_t st) {
  return launch_kernel("scale_nd_kernel<divide>", scale_nd_kernel<T, CPLX, true>, blocks_for(total), kNdThreads, 0, st,
                       static_cast<const T*>(x), norm, L, total, static_cast<T*>(out));
}

template <class T, bool CPLX>
static int force_hermitian_launch(const void* a, long long total, int D, void* out, cudaStream_t st) {
  return launch_kernel("force_hermitian_kernel", force_hermitian_kernel<T, CPLX>, blocks_for(total), kNdThreads, 0, st,
                       static_cast<const T*>(a), total, D, static_cast<T*>(out));
}

template <class T, bool CPLX>
static int abs_square_launch(const void* x, long long n, void* out, cudaStream_t st) {
  return launch_kernel("abs_square_kernel", abs_square_kernel<T, CPLX>, blocks_for(n), kNdThreads, 0, st,
                       static_cast<const T*>(x), n, static_cast<T*>(out));
}

template <class E>
static int one_hot_launch(const long long* labels, long long outer, long long inner, int C, const void* one,
                          void* out, int* status, cudaStream_t st) {
  E v;
  std::memcpy(&v, one, sizeof(E));
  return launch_kernel("one_hot_kernel", one_hot_kernel<E>, blocks_for(outer * C * inner), kNdThreads, 0, st, labels,
                       outer, inner, C, v, static_cast<E*>(out), status);
}

template <class T, bool CPLX>
static int scale_launch(const void* x, const double* f, const pbb_nd_layout& L, long long total, void* out,
                        cudaStream_t st) {
  return launch_kernel("scale_nd_kernel", scale_nd_kernel<T, CPLX, false>, blocks_for(total), kNdThreads, 0, st,
                       static_cast<const T*>(x), f, L, total, static_cast<T*>(out));
}

}  // namespace pbb

using namespace pbb;

extern "C" {

int pbb_affiliation_nd(const void* log_pdf, int dtype, const double* weight, const uint8_t* mask,
                       const pbb_nd_layout* columns, int K, const long long* class_stride, double affiliation_eps,
                       void* out, void* stream) {
  long long cols = 0;
  PBB_CHECK_ARG(is_float(dtype), 2, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(layout_ok(columns, &cols), 5, "bad layout");
  PBB_CHECK_ARG(K >= 0, 6, "need K >= 0");
  PBB_CHECK_ARG(class_stride != nullptr, 7, "class_stride is null");
  PBB_CHECK_ARG((log_pdf != nullptr && out != nullptr) || cols == 0 || K == 0, 1, "log_pdf / out is null");
  if (cols == 0 || K == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long* cs = class_stride;
  if (dtype == PBB_F64)
    return launch_kernel("affiliation_nd_kernel", affiliation_nd_kernel<double>, blocks_for(cols), kNdThreads, 0, st,
                         static_cast<const double*>(log_pdf), weight, mask, *columns, cols, K, cs[0], cs[1], cs[2],
                         cs[3], DBL_MIN, affiliation_eps, static_cast<double*>(out));
  return launch_kernel("affiliation_nd_kernel", affiliation_nd_kernel<float>, blocks_for(cols), kNdThreads, 0, st,
                       static_cast<const float*>(log_pdf), weight, mask, *columns, cols, K, cs[0], cs[1], cs[2], cs[3],
                       (double)FLT_MIN, affiliation_eps, static_cast<float*>(out));
}

size_t pbb_reduce_workspace_bytes(long long outs, long long n) {
  if (outs < 0 || n < 0) return 0;
  const long long chunks = red_chunks(outs, n);
  return (size_t)((chunks > 1 ? outs * chunks : 0) + outs) * sizeof(double);
}

int pbb_axis_sum(const void* x, int dtype, const double* multiplier, const pbb_nd_layout* outer,
                 const pbb_nd_layout* reduced, int square, double divisor, void* out, int out_dtype, void* workspace,
                 size_t workspace_bytes, void* stream) {
  long long outs = 0, n = 0;
  PBB_CHECK_ARG(is_float_or_complex(dtype), 2, "dtype must be PBB_F32, PBB_F64, PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(layout_ok(outer, &outs), 4, "bad outer layout");
  PBB_CHECK_ARG(layout_ok(reduced, &n), 5, "bad reduced layout");
  PBB_CHECK_ARG(square == 1 || is_float(dtype), 6, "a complex x is summed as |x|^2 (square = 1)");
  PBB_CHECK_ARG(out != nullptr || outs == 0, 8, "out is null");
  PBB_CHECK_ARG(is_float(out_dtype), 9, "out_dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(workspace_bytes >= pbb_reduce_workspace_bytes(outs, n) &&
                    (workspace != nullptr || pbb_reduce_workspace_bytes(outs, n) == 0),
                10, "workspace too small (pbb_reduce_workspace_bytes)");
  PBB_CHECK_ARG(x != nullptr || outs == 0 || n == 0, 1, "x is null");
  if (outs == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RedOp op{square ? kTermSquare : kTermValue, kPostDivide, 0.0, divisor, 0.0, 0};
  double* partial = static_cast<double*>(workspace);
  if (out_dtype == PBB_F32)
    return reduce_dispatch<float>(x, dtype, multiplier, *outer, *reduced, outs, n, op, partial, out, st);
  return reduce_dispatch<double>(x, dtype, multiplier, *outer, *reduced, outs, n, op, partial, out, st);
}

int pbb_unit_norm(const void* x, int dtype, const pbb_nd_layout* rows, long long n, long long x_stride,
                  long long out_stride, double ord, double eps, int eps_style, void* out, void* workspace,
                  size_t workspace_bytes, void* stream) {
  long long nrows = 0;
  PBB_CHECK_ARG(is_float_or_complex(dtype), 2, "dtype must be PBB_F32, PBB_F64, PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(layout_ok(rows, &nrows), 3, "bad layout");
  PBB_CHECK_ARG(n >= 0, 4, "need n >= 0");
  PBB_CHECK_ARG(!std::isnan(ord), 7, "ord is NaN");
  PBB_CHECK_ARG(eps_style >= 0 && eps_style <= 2, 9, "eps_style must be 0 (plus), 1 (max) or 2 (where)");
  PBB_CHECK_ARG(rows->nd < PBB_ND_MAX_DIMS, 3, "need rows.nd < PBB_ND_MAX_DIMS (the vector axis is added)");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_reduce_workspace_bytes(nrows, n), 11,
                "workspace too small (pbb_reduce_workspace_bytes)");
  PBB_CHECK_ARG((x != nullptr && out != nullptr) || nrows == 0 || n == 0, 1, "x / out is null");
  if (nrows == 0 || n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int term = ord == 2.0 ? kTermSquare : ord == 1.0 ? kTermAbs : ord == 0.0 ? kTermNonzero
                   : std::isinf(ord) ? (ord > 0 ? kTermMax : kTermMin) : kTermPow;
  const RedOp op{term, kPostNorm, ord, 1.0, eps, eps_style};
  // the norms (rows, contiguous) after the partials
  const long long chunks = red_chunks(nrows, n);
  double* partial = static_cast<double*>(workspace);
  double* norm = partial + (chunks > 1 ? nrows * chunks : 0);
  pbb_nd_layout O = *rows, R{}, D{};
  for (int d = 0; d < O.nd; ++d) O.stride[1][d] = 0;
  long long s = 1;  // operand 2: the norms, contiguous over the rows
  for (int d = O.nd - 1; d >= 0; --d) { O.stride[2][d] = s; s *= O.shape[d]; }
  R.nd = 1;
  R.shape[0] = n;
  R.stride[0][0] = x_stride;
  int rc = reduce_dispatch<double>(x, dtype, nullptr, O, R, nrows, n, op, partial, norm, st);
  if (rc) return rc;
  // out = x / norm over (rows, n): operands 0 x, 1 the norm (stride 0 along the vector), 2 out
  D.nd = O.nd + 1;
  for (int d = 0; d < O.nd; ++d) {
    D.shape[d] = O.shape[d];
    D.stride[0][d] = rows->stride[0][d];
    D.stride[1][d] = O.stride[2][d];
    D.stride[2][d] = rows->stride[1][d];
  }
  D.shape[O.nd] = n;
  D.stride[0][O.nd] = x_stride;
  D.stride[1][O.nd] = 0;
  D.stride[2][O.nd] = out_stride;
  const long long total = nrows * n;
  switch (dtype) {
    case PBB_F32: return divide_launch<float, false>(x, norm, D, total, out, st);
    case PBB_F64: return divide_launch<double, false>(x, norm, D, total, out, st);
    case PBB_C64: return divide_launch<float, true>(x, norm, D, total, out, st);
    default: return divide_launch<double, true>(x, norm, D, total, out, st);
  }
}

int pbb_force_hermitian(const void* a, int dtype, long long batch, int D, void* out, void* stream) {
  PBB_CHECK_ARG(is_float_or_complex(dtype), 2, "dtype must be PBB_F32, PBB_F64, PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(batch >= 0, 3, "need batch >= 0");
  PBB_CHECK_ARG(D >= 0, 4, "need D >= 0");
  PBB_CHECK_ARG((a != nullptr && out != nullptr) || batch == 0 || D == 0, 1, "a / out is null");
  const long long total = batch * D * D;
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (dtype) {
    case PBB_F32: return force_hermitian_launch<float, false>(a, total, D, out, st);
    case PBB_F64: return force_hermitian_launch<double, false>(a, total, D, out, st);
    case PBB_C64: return force_hermitian_launch<float, true>(a, total, D, out, st);
    default: return force_hermitian_launch<double, true>(a, total, D, out, st);
  }
}

int pbb_abs_square(const void* x, int dtype, long long n, void* out, void* stream) {
  PBB_CHECK_ARG(is_float_or_complex(dtype) || dtype == PBB_I32 || dtype == PBB_I64, 2,
                "dtype must be PBB_F32, PBB_F64, PBB_C64, PBB_C128, PBB_I32 or PBB_I64");
  PBB_CHECK_ARG(n >= 0, 3, "need n >= 0");
  PBB_CHECK_ARG((x != nullptr && out != nullptr) || n == 0, 1, "x / out is null");
  if (n == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (dtype) {
    case PBB_F32: return abs_square_launch<float, false>(x, n, out, st);
    case PBB_F64: return abs_square_launch<double, false>(x, n, out, st);
    case PBB_C64: return abs_square_launch<float, true>(x, n, out, st);
    case PBB_C128: return abs_square_launch<double, true>(x, n, out, st);
    case PBB_I32: return abs_square_launch<int, false>(x, n, out, st);
    default: return abs_square_launch<long long, false>(x, n, out, st);
  }
}

int pbb_labels_to_one_hot(const long long* labels, long long outer, long long inner, int C, int elem_size,
                          const void* one, void* out, int* status, void* stream) {
  PBB_CHECK_ARG(outer >= 0 && inner >= 0, 2, "need outer, inner >= 0");
  PBB_CHECK_ARG(C >= 0, 4, "need C >= 0");
  PBB_CHECK_ARG(elem_size == 1 || elem_size == 2 || elem_size == 4 || elem_size == 8 || elem_size == 16, 5,
                "elem_size must be 1, 2, 4, 8 or 16");
  PBB_CHECK_ARG(one != nullptr, 6, "one is null");
  PBB_CHECK_ARG(status != nullptr, 8, "status is null");
  const long long total = outer * C * inner;
  PBB_CHECK_ARG((labels != nullptr && out != nullptr) || total == 0, 1, "labels / out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PBB_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  if (total == 0) return 0;
  switch (elem_size) {
    case 1: return one_hot_launch<uint8_t>(labels, outer, inner, C, one, out, status, st);
    case 2: return one_hot_launch<uint16_t>(labels, outer, inner, C, one, out, status, st);
    case 4: return one_hot_launch<uint32_t>(labels, outer, inner, C, one, out, status, st);
    case 8: return one_hot_launch<unsigned long long>(labels, outer, inner, C, one, out, status, st);
    default: return one_hot_launch<Bytes16>(labels, outer, inner, C, one, out, status, st);
  }
}

int pbb_scale_nd(const void* x, int dtype, const double* factor, const pbb_nd_layout* layout, void* out,
                 void* stream) {
  long long total = 0;
  PBB_CHECK_ARG(is_float_or_complex(dtype), 2, "dtype must be PBB_F32, PBB_F64, PBB_C64 or PBB_C128");
  PBB_CHECK_ARG(layout_ok(layout, &total), 4, "bad layout");
  PBB_CHECK_ARG((x != nullptr && factor != nullptr && out != nullptr) || total == 0, 1, "x / factor / out is null");
  if (total == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (dtype) {
    case PBB_F32: return scale_launch<float, false>(x, factor, *layout, total, out, st);
    case PBB_F64: return scale_launch<double, false>(x, factor, *layout, total, out, st);
    case PBB_C64: return scale_launch<float, true>(x, factor, *layout, total, out, st);
    default: return scale_launch<double, true>(x, factor, *layout, total, out, st);
  }
}

}  // extern "C"
