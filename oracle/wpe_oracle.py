"""NumPy restatement of the WPE dereverberation contract of pb_bss_b200.wpe (the signatures of nara_wpe.wpe's
``wpe`` (``wpe_v8``), ``get_power``, ``get_power_inverse`` and ``build_y_tilde``).

Written from nara_wpe's interface and the published algorithm (T. Nakatani et al., "Speech dereverberation based on
variance-normalized delayed linear prediction", IEEE TASLP 18(7), 2010; T. Yoshioka and T. Nakatani, "Generalization
of multi-channel linear prediction methods for blind MIMO impulse response shortening", IEEE TASLP 20(10), 2012).
It has NOT been checked against nara_wpe itself, which is not a dependency.  The contract, for Y of shape
(..., D, T) complex, every leading index an independent problem:

* get_power: lambda_t = mean over D of |X_dt|^2; psd_context = c > 0 (an integer) averages frames t - c .. t + c
  that exist (no zero padding); psd_context = inf broadcasts the mean over all frames; negative raises ValueError.
* get_power_inverse: 1 / maximum(lambda, 1e-10 max lambda), the max over the whole array passed in.
* build_y_tilde: (..., taps D, T); row k D + d at frame t is Y_{d, t - delay - k}, zero where that index is < 0.
* wpe: X = Y, then ``iterations`` times: w = get_power_inverse(X) (per leading index), R = sum_S w_t Yt_t Yt_t^H,
  P = sum_S w_t Yt_t Y_t^H, G = stable_solve(R, P), X = Y - G^H Yt.  S is every frame ('full') or
  t >= delay + taps - 1 ('valid').  stable_solve is np.linalg.solve, and np.linalg.lstsq(R, P)[0] where that raises.
"""
import numpy as np


def _check_context(psd_context):
    if psd_context < 0:
        raise ValueError(f'psd_context must be >= 0 or inf, got {psd_context}')


def window_mean(x, c):
    """Moving mean over the last axis, frames t - c .. t + c that exist (nara_wpe's window_mean with (c, c))."""
    x = np.asarray(x, dtype=np.float64)
    T = x.shape[-1]
    csum = np.concatenate([np.zeros(x.shape[:-1] + (1,)), np.cumsum(x, axis=-1)], axis=-1)
    t = np.arange(T)
    lo, hi = np.maximum(t - c, 0), np.minimum(t + c, T - 1) + 1
    return (csum[..., hi] - csum[..., lo]) / (hi - lo)


def get_power(signal, psd_context=0):
    _check_context(psd_context)
    power = np.mean(np.abs(signal) ** 2, axis=-2)
    if np.isposinf(psd_context):
        return np.broadcast_to(np.mean(power, axis=-1, keepdims=True), power.shape).copy()
    if psd_context > 0:
        return window_mean(power, int(psd_context))
    return power


def get_power_inverse(signal, psd_context=0):
    power = get_power(signal, psd_context)
    eps = 1e-10 * np.max(power)
    with np.errstate(divide='ignore'):
        return 1 / np.maximum(power, eps)


def build_y_tilde(Y, taps, delay):
    Y = np.asarray(Y)
    *lead, D, T = Y.shape
    out = np.zeros(tuple(lead) + (taps * D, T), dtype=Y.dtype)
    for k in range(taps):
        s = delay + k
        if s < T:
            out[..., k * D:(k + 1) * D, s:] = Y[..., :, :T - s]
    return out


def stable_solve(R, P):
    try:
        return np.linalg.solve(R, P), False
    except np.linalg.LinAlgError:
        return np.linalg.lstsq(R, P, rcond=None)[0], True


def wpe_bin(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode='full', details=False):
    """One (D, T) problem in complex128.  details: also the last (w, R, P, G) and whether any solve fell back."""
    Y = np.asarray(Y, dtype=np.complex128)
    D, T = Y.shape
    Yt = build_y_tilde(Y, taps, delay)
    s = slice(delay + taps - 1, None) if statistics_mode == 'valid' else slice(None)
    X, last, fell = Y.copy(), None, False
    for _ in range(iterations):
        with np.errstate(invalid='ignore'):
            w = get_power_inverse(X, psd_context)
            R = (Yt[:, s] * w[s]) @ Yt[:, s].conj().T
            P = (Yt[:, s] * w[s]) @ Y[:, s].conj().T
        G, f = stable_solve(R, P)
        fell |= f
        X = Y - G.conj().T @ Yt
        last = (w, R, P, G)
    return (X, last, fell) if details else X


def wpe(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode='full', inplace=False):
    if statistics_mode not in ('full', 'valid'):
        raise ValueError(f'statistics_mode must be full or valid, got {statistics_mode!r}')
    _check_context(psd_context)
    Y = np.asarray(Y)
    flat = Y.reshape((-1,) + Y.shape[-2:])
    X = np.stack([wpe_bin(y, taps, delay, iterations, psd_context, statistics_mode) for y in flat])
    X = X.reshape(Y.shape).astype(Y.dtype)
    if inplace:
        Y[...] = X
        return Y
    return X
