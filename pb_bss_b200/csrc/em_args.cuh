// Argument block of the per-iteration EM kernels, shared by the API translation units.
#pragma once
#include "common.cuh"

namespace pbb {

constexpr int kMaxK = 20;  // cacgmm.py:249

enum EmMode { kModeM = 0, kModeEM = 1, kModeE = 2 };

struct EmArgs {
  const void* z;   // (F, D, zs): rows zero padded to zs frames
  int zs;
  int F, T, D, K;
  int mode;          // EmMode
  int model_kind;    // 0 = cACG, 1 = complex Watson (coef = slots of m m^H, ew = kappa, ld = log norm)
  int softmax_fast;  // integer-power softmax is safe (see em_softmax)
  const double* coef;
  const double* ld;
  const double* w;
  const double* ew;
  const double* w_time;     // frequency-tied weights (K, T) [w_time_st = 1] or (K) [w_time_st = 0], or null
  int w_time_st;
  const uint8_t* activity;  // (F, K, T) or null
  double aff_eps;
  const double* aff_in;    // (F, K, T), mode M
  const double* q_in;      // (F, K, T) or null (= 1), mode M
  const double* saliency;  // (F, T) or null
  double* part;            // (F, NCH, K, NS + 1), modes M / EM
  double* aff_out;         // (F, K, T) or null
  double* q_out;           // (F, K, T) or null
  double* loglik_part;     // (F, NCH) or null
  int nch;
  int frames_per_block;    // multiple of 32
  int f0;                  // first bin of the launch: launch_em covers F > 65535 bins (gridDim.y) in several launches
};

// host launcher (defined in api_cacgmm.cu): fills nch / frames_per_block, launches the EM
// kernel for the shape, returns nch (> 0) or an error code (<= 0)
int launch_em(EmArgs a, int dtype, int frames_per_block, cudaStream_t st);

}  // namespace pbb
