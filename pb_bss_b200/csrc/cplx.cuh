// Complex fp64 helpers and the power-of-two input scaling shared by the small-matrix solvers
// (linalg_kernels.cuh, wpe.cuh).
#pragma once
#include "common.cuh"

namespace pbb {

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cmulc(double2 a, double2 b) {  // a * conj(b)
  return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
__device__ __forceinline__ double2 cdiv(double2 a, double2 b) {
  const double d = b.x * b.x + b.y * b.y;
  return make_double2((a.x * b.x + a.y * b.y) / d, (a.y * b.x - a.x * b.y) / d);
}

// ---- input scaling -------------------------------------------------------------
// The Jacobi rotation test (|a_pq|^2 > eps^2 |a_pp a_qq| and > 1e-300), the Cholesky and cdiv square the entries:
// above ~1e154 those squares overflow, below ~1e-150 they fall under 1e-300 or underflow, and the result is silently
// wrong (the diagonal comes back as the eigenvalues).  The kernels below therefore work on the matrix times 2^-e,
// e = even_exponent(max |entry|), so that its largest entry lies in [1, 4), and undo the scaling afterwards.  Scaling
// by a power of two is exact: results at ordinary scales do not change, and w(2^k A) = 2^k w(A) bit for bit for even k.
// e is even so that a Cholesky factor scales by the exact power 2^(e/2).  0 for a zero or non-finite maximum.
__device__ __forceinline__ int even_exponent(double amax) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (!(amax > 0.0) || !isfinite(amax)) return 0;
  return ilogb(amax) & ~1;  // floor to even, also for negative exponents
}
__device__ __forceinline__ double cabs_max(double m, double2 v) { return fmax(m, fmax(fabs(v.x), fabs(v.y))); }
__device__ __forceinline__ double2 cscalbn(double2 v, int e) { return make_double2(scalbn(v.x, e), scalbn(v.y, e)); }

}  // namespace pbb
