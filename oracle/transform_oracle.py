"""NumPy restatement of the STFT / iSTFT contract of pb_bss_b200.transform (the signatures of nara_wpe.utils.stft /
istft) and of the Griffin-Lim / MISI iteration of pb_bss/transform/griffin_lim_module.py.

Written from the contract, not from nara_wpe's source, and not checked against nara_wpe itself (it is not a
dependency).  The contract:

* window: ``window(wl + 1)[:-1]`` (periodic), or ``window(wl)`` with ``symmetric_window``; wl = window_length or size.
* stft: with ``fading``, wl - shift zeros on both ends of the time axis; ``pad=True`` zero-pads the end to
  T = ceil((L - wl) / shift) + 1 frames (1 frame when L <= wl), ``pad=False`` cuts the remainder; every frame is
  multiplied by the window and transformed with ``rfft(frame, n=size)``.  Output (..., T, size // 2 + 1) with the
  frame axis where ``axis`` was.
* istft: synthesis window w_a / sum_{|i| <= (wl - 1) // shift} roll_zeropad(w_a, i shift)^2; each frame is
  ``irfft(X_t, n=size)[:wl] * w_s``, overlap-added in increasing t (``np.add.at``) into T shift + wl - shift samples;
  with ``fading`` wl - shift samples are dropped at each end.
"""
import numpy as np
import scipy.signal


def analysis_window(size, window=scipy.signal.windows.blackman, window_length=None, symmetric_window=False):
    wl = window_length or size
    return np.asarray(window(wl) if symmetric_window else window(wl + 1)[:-1], dtype=np.float64)


def _roll_zeropad(a, shift):
    out = np.zeros_like(a)
    if shift >= 0:
        out[shift:] = a[:len(a) - shift]
    else:
        out[:shift] = a[-shift:]
    return out


def synthesis_window(analysis, shift):
    wl = len(analysis)
    den = np.zeros(wl)
    for i in range(-((wl - 1) // shift), (wl - 1) // shift + 1):
        den += _roll_zeropad(analysis, i * shift) ** 2
    return analysis / den


def num_frames(length, size, shift, window_length=None, fading=True, pad=True):
    wl = window_length or size
    lp = length + (2 * (wl - shift) if fading else 0)
    if pad:
        return 1 if lp <= wl else -(-(lp - wl) // shift) + 1
    return 0 if lp < wl else (lp - wl) // shift + 1


def stft(time_signal, size=1024, shift=256, axis=-1, window=scipy.signal.windows.blackman, window_length=None,
         fading=True, pad=True, symmetric_window=False):
    x = np.asarray(time_signal)
    axis = axis % x.ndim
    wl = window_length or size
    w = analysis_window(size, window, window_length, symmetric_window)
    x = np.moveaxis(x, axis, -1)
    L = x.shape[-1]
    T = num_frames(L, size, shift, window_length, fading, pad)
    off = wl - shift if fading else 0
    padded = np.zeros(x.shape[:-1] + (max(T - 1, 0) * shift + wl,), dtype=x.dtype)
    n = min(L, padded.shape[-1] - off)
    padded[..., off:off + n] = x[..., :n]
    idx = np.arange(T)[:, None] * shift + np.arange(wl)[None, :]
    frames = padded[..., idx] * w
    out = np.fft.rfft(frames, n=size, axis=-1)
    return np.moveaxis(out, (-2, -1), (axis, axis + 1))


def istft(stft_signal, size=1024, shift=256, window=scipy.signal.windows.blackman, fading=True, window_length=None,
          symmetric_window=False):
    X = np.asarray(stft_signal)
    assert X.shape[-1] == size // 2 + 1, X.shape
    wl = window_length or size
    ws = synthesis_window(analysis_window(size, window, window_length, symmetric_window), shift)
    T = X.shape[-2]
    out = np.zeros(X.shape[:-2] + (T * shift + wl - shift,))
    frames = ws * np.real(np.fft.irfft(X, n=size))[..., :wl]
    for t in range(T):
        out[..., t * shift:t * shift + wl] += frames[..., t, :]
    if fading:
        out = out[..., wl - shift:out.shape[-1] - (wl - shift)]
    return out


def griffin_lim(X, y=None, first_guess='istft', size=512, shift=128, fading=False, steps=1, misi=False):
    """x_hat, X_dash, X_dash_dash after `steps` iterations of Griffin-Lim (misi=False) or MISI (misi=True):
    X_dash_dash = stft(x), X_dash = |X| exp(i angle(X_dash_dash)), x_hat = istft(X_dash), where x = x_hat for
    Griffin-Lim and x = x_hat + (y - sum_k x_hat) / K for MISI.  First guess: istft(X), or y / K for every k."""
    st = dict(size=size, shift=shift, fading=fading)
    K = X.shape[0]
    x_hat = istft(X, **st) if first_guess == 'istft' else np.repeat(y[None, :] / K, K, axis=0)
    X_dash = X_dash_dash = X
    for _ in range(steps):
        x = x_hat + (y - np.sum(x_hat, axis=0)) / K if misi else x_hat
        X_dash_dash = stft(x, **st)
        X_dash = np.abs(X) * np.exp(1j * np.angle(X_dash_dash))
        x_hat = istft(X_dash, **st)
    return x_hat, X_dash, X_dash_dash
