// C-ABI entry points for the STFT / iSTFT of nara_wpe.utils and the Griffin-Lim / MISI phase reconstruction of
// pb_bss/transform/griffin_lim_module.py, and the gammatone filterbank of pb_bss/transform/gammatone.py -- see
// include/pbb.h, csrc/fft.cuh and csrc/gammatone.cuh.
#include "common.cuh"
#include "fft.cuh"
#include "gammatone.cuh"
#include "prof.cuh"

namespace pbb {

static int log2_size(int size) {
  if (size < kFftMinSize || size > kFftMaxSize || (size & (size - 1)) != 0) return -1;
  int l = 0;
  while ((1 << l) < size) ++l;
  return l;
}

static int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      n = 132;
  }
  return n;
}

static int frames_per_cta(int size, long long rows, int frames) {
  return pbb_stft_frames_per_cta(size, rows, frames, sm_count());
}

template <class P>
static int fft_launch(void (*kernel)(P), const char* name, long long rows, int frames, int fpc, int size, const P& p,
                      cudaStream_t st) {
  const size_t smem = (size_t)fpc * size * sizeof(double2);  // two buffers of fpc * size / 2 points
  PBB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const long long ctas = rows * ((frames + fpc - 1) / fpc);
  if (ctas > 0x7fffffffll) {
    set_error("argument: %lld CTAs exceed the grid", ctas);
    return -1;
  }
  return launch_kernel(name, kernel, (unsigned)ctas, kFftThreads, smem, st, p);
}

struct GtShape {
  long long chunks, groups;
};

static GtShape gammatone_shape(long long N, int L) {
  const long long C = (N + L - 1) / L;
  return {C, (C + kGtGroup - 1) / kGtGroup};
}

template <class T>
static int gammatone_launch(const GtParams& p, cudaStream_t st) {
  const long long ctas = (p.total + 31) / 32 * ((p.n + kGtFilters - 1) / kGtFilters);
  if (ctas > 0x7fffffffll || p.rows * p.n > 0x7fffffffll) {
    set_error("argument: %lld CTAs exceed the grid", ctas);
    return -1;
  }
  GtParams q = p;
  if (p.chunks > 1) {
    PBB_TRY(launch_kernel("gammatone_chunk_state_kernel", gammatone_chunk_kernel<T, false>, (unsigned)ctas, kGtThreads,
                          0, st, q));
    const long long units = p.groups < kGtGroup ? p.groups : kGtGroup;
    PBB_TRY(launch_kernel("gammatone_carry_kernel", gammatone_carry_kernel, (unsigned)(p.rows * p.n),
                          (unsigned)((units * 8 + 31) / 32 * 32), 0, st, q));
  }
  return launch_kernel("gammatone_output_kernel", gammatone_chunk_kernel<T, true>, (unsigned)ctas, kGtThreads, 0, st,
                       q);
}

}  // namespace pbb

using namespace pbb;

extern "C" {

// Frames per CTA: as many as the 64 KB shared-memory budget allows, halved while the grid would not give every SM
// two CTAs.
int pbb_stft_frames_per_cta(int size, long long rows, int frames, int sms) {
  PBB_CHECK_ARG(log2_size(size) > 0, 1, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(frames > 0, 3, "frames must be positive");
  PBB_CHECK_ARG(sms > 0, 4, "sms must be positive");
  int fpc = kFftFrameBudget / size;
  while (fpc > 1 && rows * ((frames + fpc - 1) / fpc) < 2ll * sms) fpc /= 2;
  return fpc;
}

int pbb_stft(const void* x, int dtype, long long rows, long long n, int size, int shift, int window_length,
             int offset, int frames, const double* window, const double* twiddle, void* out, void* stream) {
  const int logN = log2_size(size);
  // an empty CUDA tensor has a null data pointer; with n = 0 no sample is read
  PBB_CHECK_ARG(x != nullptr || n == 0, 1, "x is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64, 2, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(rows > 0, 3, "rows must be positive");
  PBB_CHECK_ARG(n >= 0, 4, "n must be non-negative");
  PBB_CHECK_ARG(logN > 0, 5, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(window_length >= 1 && window_length <= size, 7, "window_length must be in [1, size]");
  PBB_CHECK_ARG(shift >= 1 && shift <= window_length, 6, "shift must be in [1, window_length]");
  PBB_CHECK_ARG(offset >= 0 && offset < window_length, 8, "offset must be in [0, window_length)");
  PBB_CHECK_ARG(frames > 0, 9, "frames must be positive");
  PBB_CHECK_ARG(window != nullptr, 10, "window is null");
  PBB_CHECK_ARG(twiddle != nullptr, 11, "twiddle is null");
  PBB_CHECK_ARG(out != nullptr, 12, "out is null");
  StftParams p{};
  p.x = x;
  p.rows = rows;
  p.n = n;
  p.logM = logN - 1;
  p.shift = shift;
  p.wl = window_length;
  p.offset = offset;
  p.frames = frames;
  p.fpc = frames_per_cta(size, rows, frames);
  p.tiles = (frames + p.fpc - 1) / p.fpc;
  p.window = window;
  p.tw = reinterpret_cast<const double2*>(twiddle);
  p.out = reinterpret_cast<double2*>(out);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PBB_F32) return fft_launch(stft_kernel<float, STFT_PLAIN>, "stft_kernel", rows, frames, p.fpc, size, p, st);
  return fft_launch(stft_kernel<double, STFT_PLAIN>, "stft_kernel", rows, frames, p.fpc, size, p, st);
}

int pbb_griffin_lim_stft(const double* x_hat, int K, long long n, const double* y, const void* X, int size, int shift,
                         int window_length, int offset, int frames, const double* window, const double* twiddle,
                         void* X_dash_dash, void* X_dash, void* stream) {
  const int logN = log2_size(size);
  PBB_CHECK_ARG(x_hat != nullptr || n == 0, 1, "x_hat is null");
  PBB_CHECK_ARG(K > 0, 2, "K must be positive");
  PBB_CHECK_ARG(n >= 0, 3, "n must be non-negative");
  PBB_CHECK_ARG(X != nullptr, 5, "X is null");
  PBB_CHECK_ARG(logN > 0, 6, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(window_length >= 1 && window_length <= size, 8, "window_length must be in [1, size]");
  PBB_CHECK_ARG(shift >= 1 && shift <= window_length, 7, "shift must be in [1, window_length]");
  PBB_CHECK_ARG(offset >= 0 && offset < window_length, 9, "offset must be in [0, window_length)");
  PBB_CHECK_ARG(frames > 0, 10, "frames must be positive");
  PBB_CHECK_ARG(window != nullptr, 11, "window is null");
  PBB_CHECK_ARG(twiddle != nullptr, 12, "twiddle is null");
  PBB_CHECK_ARG(X_dash_dash != nullptr, 13, "X_dash_dash is null");
  PBB_CHECK_ARG(X_dash != nullptr, 14, "X_dash is null");
  StftParams p{};
  p.x = x_hat;
  p.rows = K;
  p.n = n;
  p.logM = logN - 1;
  p.shift = shift;
  p.wl = window_length;
  p.offset = offset;
  p.frames = frames;
  p.fpc = frames_per_cta(size, K, frames);
  p.tiles = (frames + p.fpc - 1) / p.fpc;
  p.window = window;
  p.tw = reinterpret_cast<const double2*>(twiddle);
  p.X = reinterpret_cast<const double2*>(X);
  p.y = y;
  p.out = reinterpret_cast<double2*>(X_dash_dash);
  p.out_dash = reinterpret_cast<double2*>(X_dash);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (y != nullptr)
    return fft_launch(stft_kernel<double, STFT_MISI>, "stft_misi_kernel", K, frames, p.fpc, size, p, st);
  return fft_launch(stft_kernel<double, STFT_GRIFFIN_LIM>, "stft_griffin_lim_kernel", K, frames, p.fpc, size, p, st);
}

size_t pbb_istft_workspace_bytes(long long rows, int frames, int window_length) {
  if (rows <= 0 || frames <= 0 || window_length <= 0) return 0;
  return (size_t)rows * frames * window_length * sizeof(double);
}

int pbb_istft(const void* X, long long rows, int frames, int size, int shift, int window_length, int crop,
              long long n_out, const double* synthesis_window, const double* twiddle, void* workspace,
              size_t workspace_bytes, double* out, void* stream) {
  const int logN = log2_size(size);
  PBB_CHECK_ARG(X != nullptr, 1, "X is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(frames > 0, 3, "frames must be positive");
  PBB_CHECK_ARG(logN > 0, 4, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(window_length >= 1 && window_length <= size, 6, "window_length must be in [1, size]");
  PBB_CHECK_ARG(shift >= 1 && shift <= window_length, 5, "shift must be in [1, window_length]");
  const long long full = (long long)frames * shift + window_length - shift;
  PBB_CHECK_ARG(crop >= 0, 7, "crop must be non-negative");
  PBB_CHECK_ARG(n_out >= 0 && crop + n_out <= full, 8, "crop + n_out exceeds frames * shift + window_length - shift");
  PBB_CHECK_ARG(synthesis_window != nullptr, 9, "synthesis_window is null");
  PBB_CHECK_ARG(twiddle != nullptr, 10, "twiddle is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_istft_workspace_bytes(rows, frames, window_length), 11,
                "workspace too small (pbb_istft_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr || n_out == 0, 13, "out is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  IstftParams p{};
  p.X = reinterpret_cast<const double2*>(X);
  p.rows = rows;
  p.logM = logN - 1;
  p.wl = window_length;
  p.frames = frames;
  p.fpc = frames_per_cta(size, rows, frames);
  p.tiles = (frames + p.fpc - 1) / p.fpc;
  p.synthesis = synthesis_window;
  p.tw = reinterpret_cast<const double2*>(twiddle);
  p.framebuf = reinterpret_cast<double*>(workspace);
  const int rc = fft_launch(istft_frames_kernel, "istft_frames_kernel", rows, frames, p.fpc, size, p, st);
  if (rc != 0 || n_out == 0) return rc;
  long long blocks = (rows * n_out + 255) / 256;
  if (blocks > 4ll * 32 * sm_count()) blocks = 4ll * 32 * sm_count();
  return launch_kernel("overlap_add_kernel", overlap_add_kernel, (unsigned)blocks, 256, 0, st, p.framebuf, rows, frames,
                       window_length, shift, crop, n_out, out);
}

int pbb_istft_backward(const double* grad_out, long long rows, int frames, int size, int shift, int window_length,
                       int crop, long long n_out, const double* synthesis_window, const double* twiddle,
                       void* grad_X, void* stream) {
  const int logN = log2_size(size);
  PBB_CHECK_ARG(grad_out != nullptr || n_out == 0, 1, "grad_out is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(frames > 0, 3, "frames must be positive");
  PBB_CHECK_ARG(logN > 0, 4, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(window_length >= 1 && window_length <= size, 6, "window_length must be in [1, size]");
  PBB_CHECK_ARG(shift >= 1 && shift <= window_length, 5, "shift must be in [1, window_length]");
  const long long full = (long long)frames * shift + window_length - shift;
  PBB_CHECK_ARG(crop >= 0, 7, "crop must be non-negative");
  PBB_CHECK_ARG(n_out >= 0 && crop + n_out <= full, 8, "crop + n_out exceeds frames * shift + window_length - shift");
  PBB_CHECK_ARG(synthesis_window != nullptr, 9, "synthesis_window is null");
  PBB_CHECK_ARG(twiddle != nullptr, 10, "twiddle is null");
  PBB_CHECK_ARG(grad_X != nullptr, 11, "grad_X is null");
  StftParams p{};
  p.x = grad_out;
  p.rows = rows;
  p.n = n_out;
  p.logM = logN - 1;
  p.shift = shift;
  p.wl = window_length;
  p.offset = crop;
  p.frames = frames;
  p.fpc = frames_per_cta(size, rows, frames);
  p.tiles = (frames + p.fpc - 1) / p.fpc;
  p.window = synthesis_window;
  p.tw = reinterpret_cast<const double2*>(twiddle);
  p.out = reinterpret_cast<double2*>(grad_X);
  return fft_launch(istft_backward_kernel, "istft_backward_kernel", rows, frames, p.fpc, size, p,
                    reinterpret_cast<cudaStream_t>(stream));
}

size_t pbb_stft_backward_workspace_bytes(long long rows, int frames, int window_length) {
  return pbb_istft_workspace_bytes(rows, frames, window_length);
}

int pbb_stft_backward(const void* grad_X, long long rows, long long n, int size, int shift, int window_length,
                      int offset, int frames, const double* window, const double* twiddle, void* workspace,
                      size_t workspace_bytes, double* grad_x, void* stream) {
  const int logN = log2_size(size);
  PBB_CHECK_ARG(grad_X != nullptr, 1, "grad_X is null");
  PBB_CHECK_ARG(rows > 0, 2, "rows must be positive");
  PBB_CHECK_ARG(n >= 0, 3, "n must be non-negative");
  PBB_CHECK_ARG(logN > 0, 4, "size must be a power of two in [64, 4096]");
  PBB_CHECK_ARG(window_length >= 1 && window_length <= size, 6, "window_length must be in [1, size]");
  PBB_CHECK_ARG(shift >= 1 && shift <= window_length, 5, "shift must be in [1, window_length]");
  PBB_CHECK_ARG(offset >= 0 && offset < window_length, 7, "offset must be in [0, window_length)");
  PBB_CHECK_ARG(frames > 0, 8, "frames must be positive");
  PBB_CHECK_ARG(window != nullptr, 9, "window is null");
  PBB_CHECK_ARG(twiddle != nullptr, 10, "twiddle is null");
  PBB_CHECK_ARG(workspace != nullptr && workspace_bytes >= pbb_stft_backward_workspace_bytes(rows, frames, window_length),
                11, "workspace too small (pbb_stft_backward_workspace_bytes)");
  PBB_CHECK_ARG(grad_x != nullptr || n == 0, 13, "grad_x is null");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  IstftParams p{};
  p.X = reinterpret_cast<const double2*>(grad_X);
  p.rows = rows;
  p.logM = logN - 1;
  p.wl = window_length;
  p.frames = frames;
  p.fpc = frames_per_cta(size, rows, frames);
  p.tiles = (frames + p.fpc - 1) / p.fpc;
  p.synthesis = window;
  p.tw = reinterpret_cast<const double2*>(twiddle);
  p.framebuf = reinterpret_cast<double*>(workspace);
  const int rc = fft_launch(stft_backward_kernel, "stft_backward_kernel", rows, frames, p.fpc, size, p, st);
  if (rc != 0 || n == 0) return rc;
  // sample s of row r sums the frames t covering padded position s + offset; samples no frame covers get 0
  long long blocks = (rows * n + 255) / 256;
  if (blocks > 4ll * 32 * sm_count()) blocks = 4ll * 32 * sm_count();
  return launch_kernel("overlap_add_kernel", overlap_add_kernel, (unsigned)blocks, 256, 0, st, p.framebuf, rows, frames,
                       window_length, shift, offset, n, grad_x);
}

int pbb_gammatone_chunk_length(long long rows, int n, long long N) {
  int L = PBB_GAMMATONE_CHUNK_MAX;
  if (rows <= 0 || n <= 0 || N <= 0) return L;
  while (L > PBB_GAMMATONE_CHUNK_MIN && rows * n * ((N + L - 1) / L) < PBB_GAMMATONE_MIN_CHUNKS) L /= 2;
  return L;
}

size_t pbb_gammatone_workspace_bytes(long long rows, int n, long long N) {
  if (rows <= 0 || n <= 0 || N <= 0) return 0;
  const GtShape s = gammatone_shape(N, pbb_gammatone_chunk_length(rows, n, N));
  if (s.chunks == 1) return 0;
  return (size_t)(rows * n) * (size_t)(s.chunks + s.groups) * 8 * sizeof(double);
}

int pbb_gammatone(const void* x, int dtype, long long rows, long long N, int n, const double* coef,
                  const double* transition, int chunk_length, void* workspace, size_t workspace_bytes, double* out,
                  void* stream) {
  PBB_CHECK_ARG(x != nullptr, 1, "x is null");
  PBB_CHECK_ARG(dtype == PBB_F32 || dtype == PBB_F64, 2, "dtype must be PBB_F32 or PBB_F64");
  PBB_CHECK_ARG(rows > 0, 3, "rows must be positive");
  PBB_CHECK_ARG(N > 0, 4, "N must be positive");
  PBB_CHECK_ARG(n > 0, 5, "n must be positive");
  PBB_CHECK_ARG(coef != nullptr, 6, "coef is null");
  PBB_CHECK_ARG(transition != nullptr, 7, "transition is null");
  PBB_CHECK_ARG(chunk_length == pbb_gammatone_chunk_length(rows, n, N), 8,
                "chunk_length must be pbb_gammatone_chunk_length(rows, n, N)");
  const size_t need = pbb_gammatone_workspace_bytes(rows, n, N);
  PBB_CHECK_ARG(need == 0 || (workspace != nullptr && workspace_bytes >= need), 9,
                "workspace too small (pbb_gammatone_workspace_bytes)");
  PBB_CHECK_ARG(out != nullptr, 11, "out is null");
  const GtShape s = gammatone_shape(N, chunk_length);
  GtParams p{};
  p.x = x;
  p.rows = rows;
  p.N = N;
  p.chunks = s.chunks;
  p.total = rows * s.chunks;
  p.groups = s.groups;
  p.n = n;
  p.L = chunk_length;
  p.coef = coef;
  p.trans = transition;
  p.state = static_cast<double*>(workspace);
  p.group = p.state + rows * n * s.chunks * 8;
  p.out = out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == PBB_F32) return gammatone_launch<float>(p, st);
  return gammatone_launch<double>(p, st);
}

}  // extern "C"
