"""NumPy restatement of the frame-online WPE contract of pb_bss_b200.wpe: nara_wpe.wpe's ``online_wpe_step`` and
``get_power_online``, and ``online_wpe``, the step loop over a whole stream (which nara_wpe does not have).

Written from nara_wpe's interface and the published recursive least-squares form of WPE (T. Yoshioka and
T. Nakatani, "Generalization of multi-channel linear prediction methods for blind MIMO impulse response shortening",
IEEE TASLP 20(10), 2012; J. Caroselli et al., "Adaptive multichannel dereverberation for automatic speech
recognition", Interspeech 2017).  It has NOT been checked against nara_wpe itself, which is not a dependency.

n = taps D.  For bin f the window w at the current frame t holds the taps frames t - delay - 1 - k, k < taps, at
index d taps + k (nara_wpe's ``buffer[:-delay-1][::-1].transpose(1, 2, 0).reshape(F, taps*D)``), and one step is

    pred = y_t - G^H w,   u = Q w,   den = alpha lambda + w^H u,   k = u / den,
    Q'   = (Q - k (w^H Q)) / alpha,   G' = G + k pred^H.

``online_wpe`` runs it for every frame of Y (T, F, D) from a history of taps + delay frames (zeros, Q = I, G = 0 by
default), with lambda = the mean of |.|^2 over the D channels and the taps + delay + 1 frames of the buffer.
"""
import collections

import numpy as np

OnlineState = collections.namedtuple('OnlineState', ['history', 'inv_cov', 'filter_taps'])


def window(input_buffer, taps, delay):
    """(F, taps D) window of a (taps + delay + 1, F, D) buffer, index d taps + k = frame -delay - 2 - k."""
    buf = np.asarray(input_buffer)
    if buf.shape[0] != taps + delay + 1:
        raise ValueError(f'input_buffer needs taps + delay + 1 = {taps + delay + 1} frames, got {buf.shape[0]}')
    F, D = buf.shape[1:]
    return buf[:-delay - 1][::-1].transpose(1, 2, 0).reshape(F, taps * D)


def online_wpe_step(input_buffer, power_estimate, inv_cov, filter_taps, alpha, taps, delay):
    """nara_wpe.wpe.online_wpe_step: (prediction (F, D), inv_cov_k (F, n, n), filter_taps_k (F, n, D))."""
    buf = np.asarray(input_buffer)
    w = window(buf, taps, delay)
    pred = buf[-1] - np.einsum('fid,fi->fd', np.conjugate(filter_taps), w)
    nominator = np.einsum('fij,fj->fi', inv_cov, w)
    denominator = (alpha * np.asarray(power_estimate)).astype(w.dtype)
    denominator = denominator + np.einsum('fi,fi->f', np.conjugate(w), nominator)
    kalman_gain = nominator / denominator[:, None]
    inv_cov_k = inv_cov - np.einsum('fj,fjm,fi->fim', np.conjugate(w), inv_cov, kalman_gain, optimize='optimal')
    inv_cov_k = inv_cov_k / alpha
    filter_taps_k = filter_taps + np.einsum('fi,fm->fim', kalman_gain, np.conjugate(pred))
    return pred, inv_cov_k, filter_taps_k


def get_power_online(signal):
    """nara_wpe.wpe.get_power_online: (F,) mean over D and T of |signal (F, D, T)|^2."""
    return np.mean(np.abs(np.asarray(signal)) ** 2, axis=(-2, -1))


def initial_state(F, D, taps, delay, dtype=np.complex128):
    """zeros, Q = I, G = 0; Q and G in complex128, or in dtype where that is wider (np.clongdouble)"""
    n = taps * D
    cd = np.result_type(dtype, np.complex128)
    return OnlineState(np.zeros((taps + delay, F, D), dtype),
                       np.broadcast_to(np.eye(n, dtype=cd), (F, n, n)).copy(),
                       np.zeros((F, n, D), cd))


def online_wpe(Y, taps, delay, alpha, state=None, details=False):
    """Y (T, F, D) -> (Z (T, F, D), state); every frame is one online_wpe_step with lambda = get_power_online of its
    buffer.  The recursion runs in complex128, or in Y's dtype where that is wider (np.clongdouble: the long-double
    reference).  details: also kappa(Q_t) per bin and frame (Q_t = R_t^-1, so this is kappa(R_t)), shape (T, F),
    the ratio of the extreme eigenvalue moduli of a complex128 copy of the Hermitian Q_t (its 2-norm condition
    number)."""
    Y = np.asarray(Y)
    T, F, D = Y.shape
    cd = np.result_type(Y.dtype, np.complex128)
    if state is None:
        state = initial_state(F, D, taps, delay, Y.dtype)
    hist = np.asarray(state.history, dtype=cd)
    Q = np.asarray(state.inv_cov, dtype=cd)
    G = np.asarray(state.filter_taps, dtype=cd)
    stream = np.concatenate([hist, Y.astype(cd)])
    L = taps + delay + 1
    Z = np.empty((T, F, D), cd)
    kappa = np.empty((T, F))
    with np.errstate(invalid='ignore', divide='ignore'):
        for t in range(T):
            buf = stream[t:t + L]
            power = get_power_online(buf.transpose(1, 2, 0))
            Z[t], Q, G = online_wpe_step(buf, power, Q, G, alpha, taps, delay)
            if details:
                lam = np.abs(np.linalg.eigvalsh(Q.astype(np.complex128)))
                kappa[t] = lam.max(axis=-1) / lam.min(axis=-1)
    out = OnlineState(stream[T:].astype(Y.dtype), Q, G)
    Z = Z.astype(Y.dtype)
    return (Z, out, kappa) if details else (Z, out)
