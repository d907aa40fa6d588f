// Power-of-two complex FFTs of up to 2^22 points in global memory (fp64), for sequences too long for one CTA's
// shared memory, built from the shared-memory stages of fft_stages.cuh (those of fft.cuh).  Four-step: P = P1 P2
// points, P2 = 2^min(log2 P, kFlLogRow), n = P2 n1 + n2 in, k = k1 + P1 k2 out.
//
//   column pass  for every column n2: the P1-point FFT over n1 of a[P2 n1 + n2], times exp(-2 pi i n2 k1 / P), stored
//                as row k1 of a (P1, P2) workspace (several adjacent columns per CTA, so global accesses are runs)
//   row pass     the P2-point FFT of every row k1: X[k1 + P1 k2] at workspace[k1][k2] ("transposed" order)
//
// The inverse runs the same steps backwards on the transposed order: P2-point inverse FFTs of the rows, times
// exp(+2 pi i n2 k1 / P), then P1-point inverse FFTs of the columns, which give x[P2 n1 + n2].  The real-FFT split of a
// 2P-point real sequence pairs the bins k and P - k, which lie in the rows k1 and P1 - k1, so a row-pass CTA owns such
// a pair of rows (kernels below take the per-bin work as a functor).  Twiddles are sincospi of exactly reduced
// arguments, (a b mod P) / P, not recurrences.
#pragma once
#include "fft_stages.cuh"

namespace pbb {

constexpr int kFlThreads = 256;
constexpr int kFlLogRow = 11;         // rows of at most 2048 points: two rows and their scratch are 128 KB
constexpr int kFlColPoints = 4096;    // points per column-pass CTA (cols * P1), also 128 KB with scratch

struct FlShape {
  int logP, logP1, logP2, cols;       // cols: adjacent columns per column-pass CTA
  __host__ __device__ int P1() const { return 1 << logP1; }
  __host__ __device__ int P2() const { return 1 << logP2; }
  __host__ __device__ long long P() const { return 1ll << logP; }
  __host__ __device__ int col_tiles() const { return P2() / cols; }
  __host__ __device__ int row_pairs() const { return P1() / 2 + 1; }  // k1 = 0 .. P1 / 2
};

inline FlShape fl_shape(int logP) {
  FlShape s;
  s.logP = logP;
  s.logP2 = logP < kFlLogRow ? logP : kFlLogRow;
  s.logP1 = logP - s.logP2;
  const int c = kFlColPoints >> s.logP1;
  s.cols = c < s.P2() ? c : s.P2();
  return s;
}

// exp(SIGN 2 pi i (a b mod P) / P)
template <int SIGN>
__device__ __forceinline__ double2 fl_twiddle(long long a, long long b, int logP) {
  const long long r = (a * b) & ((1ll << logP) - 1);
  double s, c;
  sincospi(ldexp((double)r, 1 - logP), &s, &c);
  return make_double2(c, SIGN * s);
}

// tw[k] = (cos 2 pi k / S, sin 2 pi k / S), k < S: the stage table of fft_stage for S / 2-point transforms
__global__ void fl_stage_table_kernel(double2* tw, int logS) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < (1 << logS)) {
    double s, c;
    sincospi(ldexp((double)k, 1 - logS), &s, &c);
    tw[k] = make_double2(c, s);
  }
}

// Column pass over the sequences of one group (blockIdx.x = sequence * col_tiles + tile).  ld(seq, n) gives input
// point n; st(seq, n2, i, v) takes point i of column n2 of the transform (forward: k1, inverse: n1).
template <int DIR, class Load, class Store>
__global__ void __launch_bounds__(kFlThreads) fl_column_kernel(FlShape sh, const double2* __restrict__ tw1, Load ld,
                                                               Store st) {
  extern __shared__ double2 smem[];
  const int P1 = sh.P1(), P2 = sh.P2(), cols = sh.cols, tiles = sh.col_tiles();
  const long long seq = blockIdx.x / tiles;
  const int c0 = (int)(blockIdx.x % tiles) * cols;
  double2* A = smem;
  double2* B = smem + cols * P1;
  for (int e = threadIdx.x; e < cols * P1; e += blockDim.x) {
    const int c = e % cols, n1 = e / cols;
    A[c * P1 + n1] = ld(seq, (long long)P2 * n1 + c0 + c);
  }
  __syncthreads();
  const double2* Z = fft_shared<DIR>(A, B, sh.logP1, cols, tw1);
  for (int e = threadIdx.x; e < cols * P1; e += blockDim.x) {
    const int c = e % cols, i = e / cols;
    st(seq, c0 + c, i, Z[c * P1 + i]);
  }
}

// Loader of the inverse column pass: point n = P2 k1 + n2 of a sequence's workspace, which is its row k1 and column n2.
struct FlWorkspaceLoad {
  const double2* ws;
  int logP;
  __device__ double2 operator()(long long seq, long long n) const { return ws[(seq << logP) + n]; }
};

// Row pass over the sequences of one group (blockIdx.x = sequence * row_pairs + pair): the forward P2-point FFTs of
// rows k1 and P1 - k1 of ws (one row when they coincide), then op(...) on the spectrum.  op.kInverse: op writes the
// new spectrum into the scratch buffer, which is inverse-transformed, multiplied by exp(+2 pi i n2 k1 / P) and written
// back over the rows; otherwise op stores what it needs itself.
template <class Op>
__global__ void __launch_bounds__(kFlThreads) fl_row_pair_kernel(FlShape sh, const double2* __restrict__ tw2,
                                                                 double2* ws, Op op) {
  extern __shared__ double2 smem[];
  const int P1 = sh.P1(), P2 = sh.P2(), pairs = sh.row_pairs();
  const long long seq = blockIdx.x / pairs;
  const int k1 = (int)(blockIdx.x % pairs), kb = (P1 - k1) & (P1 - 1);
  const int rows = kb == k1 ? 1 : 2;
  double2* A = smem;
  double2* B = smem + 2 * P2;
  double2* w = ws + (seq << sh.logP);
  for (int e = threadIdx.x; e < rows * P2; e += blockDim.x) {
    const int r = e >> sh.logP2, k2 = e & (P2 - 1);
    A[e] = w[(long long)(r ? kb : k1) * P2 + k2];
  }
  __syncthreads();
  double2* Z = fft_shared<-1>(A, B, sh.logP2, rows, tw2);
  double2* O = Z == A ? B : A;
  for (int e = threadIdx.x; e < rows * P2; e += blockDim.x) {
    const int r = e >> sh.logP2, k2 = e & (P2 - 1);
    const int kr = r ? kb : k1;
    // bin k = kr + P1 k2 and its partner P - k (mod P) = kp + P1 k2p, in the other row of the pair
    const int pr = rows == 2 ? 1 - r : r, kp = pr ? kb : k1;
    const int k2p = kr == 0 ? (P2 - k2) & (P2 - 1) : P2 - 1 - k2;
    op(seq, kr, k2, kp, k2p, Z[e], Z[(pr << sh.logP2) + k2p], O + e);
  }
  if (!Op::kInverse) return;
  __syncthreads();
  const double2* X = fft_shared<1>(O, Z, sh.logP2, rows, tw2);
  for (int e = threadIdx.x; e < rows * P2; e += blockDim.x) {
    const int r = e >> sh.logP2, n2 = e & (P2 - 1);
    const int kr = r ? kb : k1;
    w[(long long)kr * P2 + n2] = cmul(X[e], fl_twiddle<1>(n2, kr, sh.logP));
  }
}

}  // namespace pbb
