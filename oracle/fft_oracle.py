"""Long-double restatements of the FFT paths of pb_bss_b200 (stft / istft, one Griffin-Lim / MISI step, the Hilbert
envelope of SRMR), the error bounds the device kernels are held to, and a float64 model of the kernels' arithmetic
that sizes those bounds without a GPU.

The restatements follow oracle/transform_oracle.py and srmr's ``np.abs(scipy.signal.hilbert(x))``, with every
transform in ``np.longdouble`` (NumPy's and SciPy's pocketfft compute in the input's precision; the 64-bit mantissa
of x86 long double agrees with an mpmath DFT to about 1e-18).  Inputs and windows stay float64, as the device reads
them; only the transforms and the overlap-add are done in long double.

The model (``model_stft`` / ``model_istft``) is the arithmetic of csrc/fft_stages.cuh and csrc/fft.cuh restated in
float64 NumPy and vectorised over frames: the size/2-point complex transform of the even/odd-packed frame in radix-4
Stockham stages (one radix-2 stage when log2(size/2) is odd) with the same twiddle table, then the real split;
inversely the split, the inverse stages, the synthesis window and the overlap-add in increasing t.  It is not bitwise
equal to the device (the compiler contracts products into FMAs), but it makes the same roundings in the same order
of operations, so its error against the oracle is what a correct kernel achieves.

Bounds (u = 2^-53):

* forward, per frame: ||X_t - X*_t||_2 <= C_F u log2(size) ||X*_t||_2; a frame that is exactly zero is exactly zero.
* inverse, per output sample: |x_m - x*_m| <= C_I u log2(size) sum_t |w_s[m - t shift]| rms(irfft X_t), over the
  frames t that cover m.
* envelope, per row: ||e - e*||_2 <= C_F u log2(M) ||a*||_2, a* the analytic signal, M the real FFT length.
* Griffin-Lim / MISI: X_dash_dash has the forward bound; X_dash per bin
  |X'_k - X'*_k| <= |X_k| min(2, 2 eps_t / |X''*_k|), eps_t the frame's forward bound.
"""
import numpy as np
import scipy.signal

from . import transform_oracle as TO

LD = np.longdouble
U = 2.0 ** -53
C_F = 2.0
# with C_I = 1 the model's worst inverse ratio is about 2.6 over the shapes of tests/test_fft_oracle.py and 3.7 over
# the larger sample of tests/test_fft_kernels_gpu.py (a per-sample maximum, so it grows slowly with the number of
# samples; largest at shift = wl).  C_I = 10 keeps the model at least 2x inside the bound and the bound within 10x of
# what the algorithm achieves
C_I = 10.0


def twiddles(size):
    """The host table of pb_bss_b200.transform.fourier: (cos + i sin)(2 pi k / size), k < size."""
    k = 2 * np.pi * np.arange(size) / size
    return np.cos(k) + 1j * np.sin(k)


def _frames(x, size, shift, wl, fading, pad):
    """(..., T, wl) float64 frames of x (before the window), zero outside the signal."""
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[-1]
    T = TO.num_frames(L, size, shift, wl, fading, pad)
    off = wl - shift if fading else 0
    padded = np.zeros(x.shape[:-1] + (max(T - 1, 0) * shift + wl,))
    n = max(min(L, padded.shape[-1] - off), 0)
    padded[..., off:off + n] = x[..., :n]
    idx = np.arange(T)[:, None] * shift + np.arange(wl)[None, :]
    return padded[..., idx]


# ---- long-double oracle ----------------------------------------------------------------------------------------------
def stft(x, size, shift, window_length=None, fading=True, pad=True, symmetric_window=False):
    """TO.stft with the frame product and the rfft in long double: (..., T, size // 2 + 1) complex long double."""
    wl = window_length or size
    w = TO.analysis_window(size, window_length=wl, symmetric_window=symmetric_window)
    return np.fft.rfft(_frames(x, size, shift, wl, fading, pad).astype(LD) * w.astype(LD), n=size, axis=-1)


def _overlap_add(frames, shift):
    """sum_t frames[..., t, m - t shift] into (..., T shift + wl - shift), in increasing t."""
    T, wl = frames.shape[-2:]
    out = np.zeros(frames.shape[:-2] + (T * shift + wl - shift,), dtype=frames.dtype)
    for t in range(T):
        out[..., t * shift:t * shift + wl] += frames[..., t, :]
    return out


def istft_parts(X, size, shift, window_length=None, fading=True):
    """TO.istft in long double and the per-sample scale of the inverse bound:
    (x*, sum_t |w_s[m - t shift]| rms(irfft X_t)), both cropped like the output."""
    wl = window_length or size
    ws = TO.synthesis_window(TO.analysis_window(size, window_length=wl), shift)
    y = np.fft.irfft(np.asarray(X).astype(np.clongdouble), n=size, axis=-1)
    rms = np.sqrt(np.mean(np.square(y), axis=-1, keepdims=True))
    x = _overlap_add(y[..., :wl] * ws.astype(LD), shift)
    scale = _overlap_add((rms * np.abs(ws)).astype(np.float64), shift)
    if fading:
        c = wl - shift
        x, scale = x[..., c:x.shape[-1] - c], scale[..., c:scale.shape[-1] - c]
    return x, scale


def misi_signal(x_hat, y):
    """MISI's x in float64, formed exactly as NumPy does."""
    return x_hat + (y - np.sum(x_hat, axis=0)) / x_hat.shape[0]


def griffin_lim_step(x_hat, X, y, size, shift, fading):
    """(X_dash_dash*, X_dash*) of one Griffin-Lim (y None) or MISI step in long double: X_dash_dash = stft(x)
    (periodic Blackman, window_length = size, pad), X_dash = |X| X''/|X''| (|X| at X'' = 0)."""
    x = x_hat if y is None else misi_signal(x_hat, y)
    Xdd = stft(x, size, shift, fading=fading)
    mag = np.abs(np.asarray(X).astype(np.clongdouble))
    h = np.abs(Xdd)
    phase = np.where(h > 0, Xdd / np.where(h > 0, h, 1), 1)
    return Xdd, mag * phase


def analytic(x):
    """scipy.signal.hilbert of each row in long double."""
    return scipy.signal.hilbert(np.asarray(x, dtype=np.float64).astype(LD), axis=-1)


# ---- bounds ----------------------------------------------------------------------------------------------------------
def forward_ratio(X, ref, size):
    """Per-frame ||X_t - X*_t|| / (C_F u log2(size) ||X*_t||) and the mask of exact-zero reference frames (where the
    ratio is 0 if X_t is exactly zero, inf otherwise)."""
    err = np.sqrt(np.sum(np.abs(np.asarray(X).astype(np.clongdouble) - ref) ** 2, axis=-1)).astype(np.float64)
    nrm = np.sqrt(np.sum(np.abs(ref) ** 2, axis=-1)).astype(np.float64)
    zero = nrm == 0
    ratio = np.where(zero, np.where(err == 0, 0.0, np.inf), err / (C_F * U * np.log2(size) * np.where(zero, 1, nrm)))
    return ratio, zero


def inverse_ratio(x, ref, scale, size, c_i=None):
    """Per-sample |x_m - x*_m| / (C_I u log2(size) scale_m), 0 / inf where the scale is 0."""
    c = C_I if c_i is None else c_i
    err = np.abs(np.asarray(x).astype(LD) - ref).astype(np.float64)
    zero = scale == 0
    return np.where(zero, np.where(err == 0, 0.0, np.inf), err / (c * U * np.log2(size) * np.where(zero, 1, scale)))


def envelope_ratio(e, a, M):
    """||e - |a||| / (C_F u log2(M) ||a||) of one row."""
    err = float(np.sqrt(np.sum((np.asarray(e).astype(LD) - np.abs(a)) ** 2)))
    nrm = float(np.sqrt(np.sum(np.abs(a) ** 2)))
    if nrm == 0:
        return 0.0 if err == 0 else np.inf
    return err / (C_F * U * max(np.log2(M), 1.0) * nrm)


def dash_ratio(Xd, X, Xdd_ref, size):
    """Per-bin |X'_k - X'*_k| / (|X_k| min(2, 2 eps_t / |X''*_k|)) at the bins of frames that are not exactly zero
    (where X'' is exactly zero, X' must be |X| + 0j: checked separately)."""
    h = np.abs(Xdd_ref)
    nrm = np.sqrt(np.sum(h ** 2, axis=-1, keepdims=True))
    eps = C_F * U * np.log2(size) * nrm
    phase = np.where(h > 0, Xdd_ref / np.where(h > 0, h, 1), 1)
    ref = np.abs(np.asarray(X).astype(np.clongdouble)) * phase
    err = np.abs(np.asarray(Xd).astype(np.clongdouble) - ref)
    with np.errstate(divide='ignore', invalid='ignore'):
        lim = np.abs(X) * np.minimum(2.0, 2 * eps / h).astype(np.float64)
        r = np.where(lim > 0, err.astype(np.float64) / np.where(lim > 0, lim, 1), np.where(err == 0, 0.0, np.inf))
    live = np.broadcast_to(nrm > 0, r.shape)
    return r[live]


# ---- float64 model of the kernels ------------------------------------------------------------------------------------
def _stage(src, logM, logNs, R, DIR, tw):
    """fft_stage<R, DIR> over every frame of src (F, M)."""
    logR = 2 if R == 4 else 1
    lognb = logM - logR
    nb, Ns = 1 << lognb, 1 << logNs
    tshift = logM + 1 - logNs - logR
    j = np.arange(nb)
    jm = j & (Ns - 1)
    v = [src[:, j + (r << lognb)] for r in range(R)]
    step = jm << tshift
    for r in range(1, R):
        w = tw[r * step]
        v[r] = v[r] * (np.conj(w) if DIR < 0 else w)
    if R == 2:
        v = [v[0] + v[1], v[0] - v[1]]
    else:
        s02, d02, s13, d13 = v[0] + v[2], v[0] - v[2], v[1] + v[3], v[1] - v[3]
        jd13 = 1j * d13  # exact: a swap and a sign
        v = [s02 + s13, d02 - jd13 if DIR < 0 else d02 + jd13, s02 - s13, d02 + jd13 if DIR < 0 else d02 - jd13]
    dst = np.empty_like(src)
    base = (j - jm) * R + jm
    for r in range(R):
        dst[:, base + (r << logNs)] = v[r]
    return dst


def _fft_shared(a, logM, DIR, tw):
    logNs = 0
    while logNs + 2 <= logM:
        a = _stage(a, logM, logNs, 4, DIR, tw)
        logNs += 2
    if logNs < logM:
        a = _stage(a, logM, logNs, 2, DIR, tw)
    return a


def model_rfft(f, size):
    """The forward body of stft_kernel in float64 on windowed real frames f (N, size): (N, size // 2 + 1) complex128."""
    M, logM = size // 2, int(np.log2(size)) - 1
    tw = twiddles(size)
    z = _fft_shared(f[:, 0::2] + 1j * f[:, 1::2], logM, -1, tw)
    k = np.arange(1, M)
    a, b = z[:, k], z[:, M - k]
    fe = 0.5 * (a.real + b.real) + 1j * (0.5 * (a.imag - b.imag))
    fo = 0.5 * (a.imag + b.imag) + 1j * (-0.5 * (a.real - b.real))
    out = np.empty((f.shape[0], M + 1), dtype=np.complex128)
    out[:, 0] = z[:, 0].real + z[:, 0].imag
    out[:, M] = z[:, 0].real - z[:, 0].imag
    out[:, 1:M] = fe + np.conj(tw[k]) * fo
    return out


def model_stft(x, size, shift, window_length=None, fading=True, pad=True):
    """stft_kernel's arithmetic in float64: (..., T, size // 2 + 1) complex128."""
    wl = window_length or size
    fr = _frames(x, size, shift, wl, fading, pad)
    lead, T = fr.shape[:-2], fr.shape[-2]
    f = np.zeros((int(np.prod(lead, dtype=np.int64)) * T, size))
    f[:, :wl] = fr.reshape(-1, wl) * TO.analysis_window(size, window_length=wl)
    return model_rfft(f, size).reshape(lead + (T, size // 2 + 1))


def model_irfft(Xf, size):
    """The inverse body of istft_frames_kernel in float64 on spectra Xf (N, size // 2 + 1): (N, size) real frames,
    irfft(Xf, n=size)."""
    M, logM = size // 2, int(np.log2(size)) - 1
    tw = twiddles(size)
    k = np.arange(1, M)
    a, b = Xf[:, k], Xf[:, M - k]
    fe = 0.5 * (a.real + b.real) + 1j * (0.5 * (a.imag - b.imag))
    fo = (0.5 * (a.real - b.real) + 1j * (0.5 * (a.imag + b.imag))) * tw[k]
    z = np.empty((Xf.shape[0], M), dtype=np.complex128)
    z[:, 0] = 0.5 * (Xf[:, 0].real + Xf[:, M].real) + 1j * (0.5 * (Xf[:, 0].real - Xf[:, M].real))
    z[:, 1:] = (fe.real - fo.imag) + 1j * (fe.imag + fo.real)
    v = _fft_shared(z, logM, 1, tw)
    y = np.empty((Xf.shape[0], size))
    y[:, 0::2], y[:, 1::2] = v.real / M, v.imag / M
    return y


def model_istft(X, size, shift, window_length=None, fading=True):
    """istft_frames_kernel + overlap_add_kernel's arithmetic in float64."""
    wl = window_length or size
    X = np.asarray(X, dtype=np.complex128)
    lead, T = X.shape[:-2], X.shape[-2]
    y = model_irfft(X.reshape(-1, size // 2 + 1), size)
    ws = TO.synthesis_window(TO.analysis_window(size, window_length=wl), shift)
    out = _overlap_add((ws * y[:, :wl]).reshape(lead + (T, wl)), shift)
    if fading:
        c = wl - shift
        out = out[..., c:out.shape[-1] - c]
    return out


# ---- test signals ----------------------------------------------------------------------------------------------------
def spread_signal(shape, wl, seed, zero_runs=True):
    """Gaussian noise under a slow envelope spanning 120 dB (1 to 1e-6 in amplitude, period 16 windows), with a run of
    exact zeros longer than 2 wl + 8 in every row when the row is long enough."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape)
    n = shape[-1]
    m = np.arange(n)
    phase = rng.random(shape[:-1] + (1,))
    x *= 10.0 ** (-3.0 * (1 + np.cos(2 * np.pi * (m / (16 * wl) + phase))))
    run = 2 * wl + 8
    if zero_runs and n >= 2 * run:
        x[..., n // 3:n // 3 + run] = 0.0
    return x
