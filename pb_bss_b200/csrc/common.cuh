// Shared device/host helpers for the pb_bss_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <utility>

#include "../../include/pbb.h"

namespace pbb {

constexpr double kTiny = DBL_MIN;  // np.finfo(np.float64).tiny

// ---- host-side error reporting (pbb_last_error) ---------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define PBB_CHECK_ARG(cond, idx, msg)                         \
  do {                                                        \
    if (!(cond)) {                                            \
      ::pbb::set_error("argument %d: %s", (idx), (msg));      \
      return -(idx);                                          \
    }                                                         \
  } while (0)

#define PBB_CUDA(call)                                        \
  do {                                                        \
    cudaError_t _e = (call);                                  \
    if (_e != cudaSuccess) return ::pbb::cuda_fail(_e, #call);\
  } while (0)

// propagates a nonzero status (a launch_kernel result, say) to the caller
#define PBB_TRY(...)                                          \
  do {                                                        \
    if (int _r = (__VA_ARGS__)) return _r;                    \
  } while (0)

// ---- launches with one attribute (host) ------------------------------------------
// Configuration of a launch with one launch attribute, for launch_ex (prof.cuh) and
// cudaOccupancyMaxActiveClusters.  cfg points at attr, so the object is not copied.
struct AttrLaunch {
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr{};
  AttrLaunch(dim3 grid, dim3 block, size_t smem, cudaStream_t st) {
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
  }
  AttrLaunch(const AttrLaunch&) = delete;
  AttrLaunch& operator=(const AttrLaunch&) = delete;
};

// a 1-D grid launched in clusters of `cluster` CTAs
struct ClusterLaunch : AttrLaunch {
  ClusterLaunch(unsigned ctas, unsigned threads, size_t smem, unsigned cluster, cudaStream_t st)
      : AttrLaunch(dim3(ctas), dim3(threads), smem, st) {
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
  }
};

// a cooperative launch: all CTAs co-resident (grid_barrier), or the launch fails
struct CoopLaunch : AttrLaunch {
  CoopLaunch(dim3 grid, dim3 block, size_t smem, cudaStream_t st) : AttrLaunch(grid, block, smem, st) {
    attr.id = cudaLaunchAttributeCooperative;
    attr.val.cooperative = 1;
  }
};

// ---- dtype dispatch (host) ---------------------------------------------------------
// fn(ct) with a value of the storage type (double2 for PBB_C128, float2 for PBB_C64) standing for the type
template <class Fn>
static int with_ct(int dtype, Fn&& fn) {
  return dtype == PBB_C128 ? fn(double2{}) : fn(float2{});
}

// ---- compile-time loop -----------------------------------------------------
template <class F, int... I>
__device__ __forceinline__ void static_for_impl(F&& f, std::integer_sequence<int, I...>) {
  (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  static_for_impl(static_cast<F&&>(f), std::make_integer_sequence<int, N>{});
}

// ---- slot table -------------------------------------------------------------
// A Hermitian D x D outer product z z^H has D*D real degrees of freedom
// ("slots"): D real diagonals and D(D-1)/2 complex off-diagonal entries.  A slot
// is (d, e, kind) with psi(d,e) = conj(z_d) * z_e (d may be larger than e: the
// scatter matrix entry [d][e] is conj(psi), entry [e][d] is psi, and the
// quadratic form picks up 2 Re(Binv[d][e] psi) either way).
//
// Even D: the channels form M = D/2 pairs P_0..P_{M-1}.  The slots are split
// into M groups with IDENTICAL local structure, so M warps can run the same
// instruction stream on different channels:
//   group g owns pair P_g = (a0, a1):          |a0|^2, |a1|^2, (a0,a1)
//   full cross with P_{g+1+j}, j < (M-1)/2:    (a0,b0) (a0,b1) (a1,b0) (a1,b1)
//   if M is even, half cross with P_{g+M/2}:   (a0,c0) (a1,c1), where the lower
//   half of the groups takes c in order and the upper half takes it swapped,
//   which tiles the 2x2 cross block of the two pairs exactly once.
// D=8: 4 groups x 16 slots (6 channels each); D=6: 3 x 12; D=4: 2 x 8.
// Odd D: plain upper-triangle order (only the generic kernels use it).
struct SlotInfo { int d, e, kind; };  // kind: 0 = diagonal, 1 = real part, 2 = imaginary part

struct GroupShape {
  int M, nfull, half, nloc, nsg;
};
__host__ __device__ constexpr GroupShape group_shape(int D) {
  const int M = D / 2;
  const int nfull = (M - 1) / 2;
  const int half = (M % 2 == 0) ? 1 : 0;
  return {M, nfull, half, 2 + 2 * nfull + 2 * half, 4 + 8 * nfull + 4 * half};
}
// Row layout of a ring stage of the observation in shared memory: rows 0..D-1
// are the channels; the rows after that repeat the first channels (pair-swapped
// when M is even) so that group g finds its NLOC local channels in the
// CONSECUTIVE rows 2g .. 2g+NLOC-1 -- one base address plus compile-time
// offsets for every group.  The repeated rows exist on chip only: global memory
// holds the D channel rows, and stage_g2s (em_persistent.cuh) copies the
// repeated ones from there.
//   D=8: rows = 0 1 2 3 4 5 6 7 | 1 0 3 2      D=6: 0..5 | 0 1      D=4: 0..3 | 1 0
__host__ __device__ constexpr int stage_rows(int D) {
  const GroupShape gs = group_shape(D);
  return 2 * (gs.M - 1) + gs.nloc;
}
__host__ __device__ constexpr int row_channel(int D, int r) {
  if (r < D) return r;
  const int x = r - D;
  return (D / 2) % 2 == 0 ? (x ^ 1) : x;
}
// channel of local index l of group g (0,1 = own pair; then the full crosses; last two = half cross)
__host__ __device__ constexpr int group_channel(int D, int g, int l) { return row_channel(D, 2 * g + l); }
// local slot i of a group -> (local x, local y, kind)
__host__ __device__ constexpr SlotInfo group_local_slot(int D, int i) {
  const GroupShape gs = group_shape(D);
  if (i == 0) return {0, 0, 0};
  if (i == 1) return {1, 1, 0};
  if (i < 4) return {0, 1, i - 1};
  const int r = i - 4;
  if (r < 8 * gs.nfull) {
    const int j = r / 8, q = (r % 8) / 2, kind = 1 + (r % 2);
    return {q / 2, 2 + 2 * j + (q % 2), kind};
  }
  const int h = r - 8 * gs.nfull;  // 0..3
  return {h / 2, 2 + 2 * gs.nfull + h / 2, 1 + (h % 2)};
}

__host__ __device__ constexpr SlotInfo slot_info(int D, int s) {
  if (D % 2 == 0) {
    const GroupShape gs = group_shape(D);
    const int g = s / gs.nsg, i = s % gs.nsg;
    const SlotInfo l = group_local_slot(D, i);
    return {group_channel(D, g, l.d), group_channel(D, g, l.e), l.kind};
  }
  int idx = 0;
  for (int d = 0; d < D; ++d) {
    if (idx == s) return {d, d, 0};
    ++idx;
    for (int e = d + 1; e < D; ++e) {
      if (idx == s) return {d, e, 1};
      ++idx;
      if (idx == s) return {d, e, 2};
      ++idx;
    }
  }
  return {-1, -1, -1};
}

// bitmask of channels a contiguous slot range [s0, s1) touches
__host__ __device__ constexpr unsigned slot_range_channels(int D, int s0, int s1) {
  unsigned m = 0;
  for (int s = s0; s < s1 && s < D * D; ++s) {
    SlotInfo si = slot_info(D, s);
    m |= (1u << si.d) | (1u << si.e);
  }
  return m;
}

// packed runtime table entry: d | e << 8 | kind << 16
__host__ __device__ inline int slot_pack(int D, int s) {
  SlotInfo si = slot_info(D, s);
  return si.d | (si.e << 8) | (si.kind << 16);
}

// ---- loads of the observation in either storage precision ------------------
__device__ __forceinline__ double2 ld_cplx(const double2* p) { return __ldg(p); }
__device__ __forceinline__ double2 ld_cplx(const float2* p) {
  float2 v = __ldg(p);
  return make_double2((double)v.x, (double)v.y);
}
__device__ __forceinline__ void st_cplx(double2* p, double re, double im) { *p = make_double2(re, im); }
__device__ __forceinline__ void st_cplx(float2* p, double re, double im) { *p = make_float2((float)re, (float)im); }

// |s|^2 as NumPy rounds it: two products, one sum, no FMA contraction
__device__ __forceinline__ double abs2_rn(double2 v) { return __dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y)); }

// log( 1F1(1; D; kappa) * 2 pi^D / (D-1)! )  (complex_watson.py:157-168).  Series
// for small kappa, Mardia's closed form (complex_watson.py:109-138) otherwise.
__device__ inline double cw_log_norm(double kappa, int D) {
  double lfact = 0.0;
  for (int r = 2; r < D; ++r) lfact += log((double)r);
  const double base = log(2.0) + (double)D * log(3.14159265358979323846) - lfact;
  if (kappa < 20.0) {
    double s = 1.0, term = 1.0;
    for (int n = 1; n < 400; ++n) {
      term *= kappa / (double)(D + n - 1);
      s += term;
      if (term < 1e-17 * s) break;
    }
    return base + log(s);
  }
  double part = 0.0, pw = 1.0, fr = 1.0;  // sum_{r=0}^{D-2} kappa^r / r!
  for (int r = 0; r <= D - 2; ++r) {
    if (r > 0) { pw *= kappa; fr *= (double)r; }
    part += pw / fr;
  }
  return log(2.0) + (double)D * log(3.14159265358979323846) + (1.0 - (double)D) * log(kappa) + kappa +
         log1p(-exp(-kappa) * part);
}

// ---- grid barrier -------------------------------------------------------------
// Grid-wide barrier of a cooperative launch (all CTAs are resident): a monotonic arrival counter, one atomic and a
// short acquire spin per CTA -- about a third of the latency of cooperative_groups' grid.sync() here.  The counter
// is zeroed before the launch; generation starts at 0 in every CTA.
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& generation) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ++generation;
    __threadfence();
    atomicAdd(counter, 1u);
    const unsigned target = generation * gridDim.x;
    unsigned seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
    } while (seen < target);
  }
  __syncthreads();
}

// ---- warp reductions ---------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum N per-lane values over the 32 lanes of a warp with the "halving"
// butterfly: at each of the 5 steps a lane keeps one half of its values and
// sends the other half to its partner, so N + O(log) values are exchanged in
// total instead of 5 N.  Afterwards lane l holds the totals of the indices
// reduce_base<N>(l) .. +reduce_count<N>(l) in v[0..].
template <int N> struct HalvingSizes {
  static constexpr int n1 = (N + 1) / 2, n2 = (n1 + 1) / 2, n3 = (n2 + 1) / 2,
                       n4 = (n3 + 1) / 2, n5 = (n4 + 1) / 2;
};
template <int N, int NH>
__device__ __forceinline__ void halving_step(double (&v)[N], int lane, int off) {
  // v holds 2*NH (or 2*NH-1 .. padded) live values in v[0 .. 2*NH)
  const bool upper = (lane & off) != 0;
#pragma unroll
  for (int i = 0; i < NH; ++i) {
    const double lo = v[i];
    const double hi = (i + NH < N) ? v[i + NH] : 0.0;
    const double keep = upper ? hi : lo;
    const double send = upper ? lo : hi;
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
  }
}
template <int N>
__device__ __forceinline__ void warp_reduce_halving(double (&v)[N], int lane) {
  using S = HalvingSizes<N>;
  // live counts: N -> n1 -> n2 -> n3 -> n4 -> n5 ; zero-pad the tail first
  halving_step<N, S::n1>(v, lane, 16);
#pragma unroll
  for (int i = S::n1; i < N; ++i) v[i] = 0.0;
  halving_step<N, S::n2>(v, lane, 8);
#pragma unroll
  for (int i = S::n2; i < S::n1; ++i) v[i] = 0.0;
  halving_step<N, S::n3>(v, lane, 4);
#pragma unroll
  for (int i = S::n3; i < S::n2; ++i) v[i] = 0.0;
  halving_step<N, S::n4>(v, lane, 2);
#pragma unroll
  for (int i = S::n4; i < S::n3; ++i) v[i] = 0.0;
  halving_step<N, S::n5>(v, lane, 1);
}
// Index range [lo, hi) of the totals lane `lane` holds in v[0 .. hi-lo) after
// warp_reduce_halving<N> (hi - lo <= HalvingSizes<N>::n5; may be empty).
template <int N>
__device__ __forceinline__ void reduce_range(int lane, int& lo, int& hi) {
  using S = HalvingSizes<N>;
  lo = 0; hi = N;
  const int nh[5] = {S::n1, S::n2, S::n3, S::n4, S::n5};
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int bit = (lane >> (4 - k)) & 1;
    if (bit) lo = lo + nh[k]; else hi = min(hi, lo + nh[k]);
  }
  if (hi < lo) hi = lo;
}

}  // namespace pbb
