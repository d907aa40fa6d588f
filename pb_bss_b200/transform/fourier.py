"""STFT and iSTFT on the device with the signatures of nara_wpe.utils.stft / istft, the two ends of the separation
pipeline (STFT -> fit -> predict -> alignment -> PSD -> beamformer -> iSTFT).

The contract is restated in oracle/transform_oracle.py; it has not been checked against nara_wpe itself, which is not
a dependency.  Every FFT runs in the hand-written fp64 kernels of csrc/fft.cuh (no cuFFT); ``size`` is a power of two
in [64, 4096].  numpy in -> numpy out, CUDA tensors in -> CUDA tensors out.

``stft`` and ``istft`` are differentiable: a CUDA tensor that requires grad gets a graph whose backward runs the
device kernels of pbb_stft_backward / pbb_istft_backward (fp64, returned in the input's dtype).  Double backward
raises.
"""
import numpy as np
import scipy.signal
import torch
from torch.autograd.function import once_differentiable

from .. import _device, _lib

MIN_SIZE, MAX_SIZE = 64, 4096

_windows = {}
_twiddles = {}


def _check(size, shift, window_length):
    if not (isinstance(size, (int, np.integer)) and MIN_SIZE <= size <= MAX_SIZE and size & (size - 1) == 0):
        raise ValueError(f'size must be a power of two in [{MIN_SIZE}, {MAX_SIZE}], got {size}')
    wl = window_length or size
    if not 1 <= wl <= size:
        raise ValueError(f'window_length must be in [1, size = {size}], got {wl}')
    if not 1 <= shift <= wl:
        raise ValueError(f'shift must be in [1, window_length = {wl}], got {shift}')
    return int(size), int(shift), int(wl)


def _analysis_window(window, wl, symmetric_window):
    """window(wl + 1)[:-1] (or window(wl)), computed on the host with SciPy and cached on the device."""
    key = (window, wl, bool(symmetric_window), _device.device())
    w = _windows.get(key)
    if w is None:
        host = np.asarray(window(wl) if symmetric_window else window(wl + 1)[:-1], dtype=np.float64)
        w = _windows[key] = _device.to_device(host)
    return w


def _synthesis_window(window, wl, shift, symmetric_window):
    """w_a / sum_{|i| <= (wl - 1) // shift} roll_zeropad(w_a, i shift)^2 (nara_wpe's biorthogonal window)."""
    key = (window, wl, bool(symmetric_window), shift, _device.device())
    w = _windows.get(key)
    if w is None:
        wa = np.asarray(window(wl) if symmetric_window else window(wl + 1)[:-1], dtype=np.float64)
        den = np.zeros(wl)
        for i in range(-((wl - 1) // shift), (wl - 1) // shift + 1):
            s = i * shift
            den[max(s, 0):wl + min(s, 0)] += wa[max(-s, 0):wl - max(s, 0)] ** 2
        w = _windows[key] = _device.to_device(wa / den)
    return w


def _twiddle(size):
    """(cos, sin)(2 pi k / size), k < size, from NumPy, as size double pairs."""
    key = (size, _device.device())
    tw = _twiddles.get(key)
    if tw is None:
        k = 2 * np.pi * np.arange(size) / size
        tw = _twiddles[key] = _device.to_device(np.stack([np.cos(k), np.sin(k)], axis=-1))
    return tw


def num_frames(length, size, shift, wl, fading, pad):
    lp = length + (2 * (wl - shift) if fading else 0)
    if pad:
        return 1 if lp <= wl else -(-(lp - wl) // shift) + 1
    return 0 if lp < wl else (lp - wl) // shift + 1


def stft(time_signal, size=1024, shift=256, axis=-1, window=scipy.signal.windows.blackman, window_length=None,
         fading=True, pad=True, symmetric_window=False):
    """nara_wpe.utils.stft: (..., n) real -> (..., T, size // 2 + 1) complex128, the frame axis where ``axis`` was.

    With ``fading``, window_length - shift zeros pad both ends; ``pad=True`` zero-pads the end to
    T = ceil((n - window_length) / shift) + 1 frames (one when the padded signal is shorter than the window),
    ``pad=False`` cuts the remainder.  Each frame is multiplied by the window and transformed with
    ``rfft(frame, n=size)``.  The padding is never materialised.  float32 input gives complex128 (the float64 window
    promotes), as in NumPy."""
    size, shift, wl = _check(size, shift, window_length)
    like_numpy = not _device.is_tensor(time_signal)
    x = np.asarray(time_signal) if like_numpy else time_signal
    if np.iscomplexobj(x) if like_numpy else x.is_complex():
        raise TypeError(f'stft of a real signal, got {x.dtype}')
    ndim = x.ndim if like_numpy else x.dim()
    axis = axis % ndim
    if like_numpy:
        x = np.moveaxis(x, axis, -1)
        x = x.astype(np.float32 if x.dtype == np.float32 else np.float64, copy=False)
    else:
        x = torch.movedim(x, axis, -1)
        x = x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)
    xd = _device.to_device(x)
    T = num_frames(xd.shape[-1], size, shift, wl, fading, pad)
    out = _Stft.apply(xd, size, shift, wl, wl - shift if fading else 0, T,
                      _analysis_window(window, wl, symmetric_window))
    out = torch.movedim(out, (-2, -1), (axis, axis + 1))
    return _device.to_host(out, like_numpy) if like_numpy else out.contiguous()


def istft(stft_signal, size=1024, shift=256, window=scipy.signal.windows.blackman, fading=True, window_length=None,
          symmetric_window=False):
    """nara_wpe.utils.istft: (..., T, size // 2 + 1) -> (..., T shift + wl - shift) float64, less wl - shift samples at
    each end with ``fading``.  Each frame is irfft(X_t, n=size)[:wl] times the biorthogonal synthesis window (the
    imaginary parts of the DC and Nyquist bins are ignored, as np.fft.irfft does), overlap-added in increasing t.
    The input is read as complex128."""
    size, shift, wl = _check(size, shift, window_length)
    like_numpy = not _device.is_tensor(stft_signal)
    X = _device.to_device(stft_signal, torch.complex128)
    assert X.dim() >= 2 and X.shape[-1] == size // 2 + 1, tuple(X.shape)
    out = _Istft.apply(X, size, shift, wl, wl - shift if fading else 0,
                       _synthesis_window(window, wl, shift, symmetric_window))
    return _device.to_host(out, like_numpy)


class _Stft(torch.autograd.Function):
    """(rows..., n) float32 / float64 -> (rows..., T, size // 2 + 1) complex128 by pbb_stft; backward pbb_stft_backward."""

    @staticmethod
    def forward(ctx, xd, size, shift, wl, offset, T, window):
        lead, n = tuple(xd.shape[:-1]), xd.shape[-1]
        out = _device.empty(lead + (T, size // 2 + 1), torch.complex128)
        rows = int(np.prod(lead, dtype=np.int64))
        if out.numel():
            dtype = _lib.PBB_F32 if xd.dtype == torch.float32 else _lib.PBB_F64
            _device.call('pbb_stft', xd, dtype, rows, n, size, shift, wl, offset, T, window, _twiddle(size), out)
        ctx.args = (lead, n, rows, size, shift, wl, offset, T, window, xd.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        lead, n, rows, size, shift, wl, offset, T, window, dtype = ctx.args
        gx = _device.empty(lead + (n,), torch.float64)
        if rows and T:
            g = grad.to(torch.complex128).contiguous()
            lib = _lib.load()
            nbytes = lib.pbb_stft_backward_workspace_bytes(rows, T, wl)
            ws = _device.workspace(nbytes)
            _device.call('pbb_stft_backward', g, rows, n, size, shift, wl, offset, T, window, _twiddle(size), ws,
                         nbytes, gx)
        else:
            gx.zero_()
        return gx.to(dtype), None, None, None, None, None, None


class _Istft(torch.autograd.Function):
    """(rows..., T, size // 2 + 1) complex128 -> (rows..., n_out) float64 by pbb_istft; backward pbb_istft_backward."""

    @staticmethod
    def forward(ctx, X, size, shift, wl, crop, synthesis):
        lead, T = tuple(X.shape[:-2]), X.shape[-2]
        n_out = max(T * shift + wl - shift - 2 * crop, 0)
        out = _device.empty(lead + (n_out,), torch.float64)
        rows = int(np.prod(lead, dtype=np.int64))
        if rows and T:
            lib = _lib.load()
            nbytes = lib.pbb_istft_workspace_bytes(rows, T, wl)
            ws = _device.workspace(nbytes)
            _device.call('pbb_istft', X, rows, T, size, shift, wl, crop, n_out, synthesis, _twiddle(size), ws, nbytes,
                         out)
        else:
            out.zero_()
        ctx.args = (lead, T, rows, n_out, size, shift, wl, crop, synthesis)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        lead, T, rows, n_out, size, shift, wl, crop, synthesis = ctx.args
        gX = _device.empty(lead + (T, size // 2 + 1), torch.complex128)
        if rows and T:
            g = grad.to(torch.float64).contiguous()
            _device.call('pbb_istft_backward', g if n_out else None, rows, T, size, shift, wl, crop, n_out, synthesis,
                         _twiddle(size), gX)
        else:
            gX.zero_()
        return gX, None, None, None, None, None


def griffin_lim_stft(x_hat, X, y, size, shift, fading):
    """The STFT half of a Griffin-Lim (y is None) or MISI step on device tensors: returns
    (X_dash_dash, X_dash) = (stft(x), |X| exp(i angle(stft(x)))) with x = x_hat, or x_hat + (y - sum_k x_hat) / K.
    Only enqueues work."""
    size, shift, wl = _check(size, shift, None)
    window = scipy.signal.windows.blackman
    K, n = x_hat.shape
    T = num_frames(n, size, shift, wl, fading, True)
    if tuple(X.shape) != (K, T, size // 2 + 1):
        raise ValueError(f'operands could not be broadcast together with shapes {tuple(X.shape)} '
                         f'({K},{T},{size // 2 + 1})')
    Xdd = _device.empty((K, T, size // 2 + 1), torch.complex128)
    Xd = torch.empty_like(Xdd)
    _device.call('pbb_griffin_lim_stft', x_hat, K, n, y, X, size, shift, wl, wl - shift if fading else 0, T,
                 _analysis_window(window, wl, False), _twiddle(size), Xdd, Xd)
    return Xdd, Xd
