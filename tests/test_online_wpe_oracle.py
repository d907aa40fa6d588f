"""The frame-online WPE oracle (oracle/wpe_online_oracle.py) against independent facts: a scalar-loop restatement of
the step, the window layout, the closed form of the recursive least-squares recursion, get_power and chunking."""
import numpy as np
import pytest

from oracle import wpe_online_oracle as O
from oracle import wpe_oracle as W

EPS = np.finfo(np.float64).eps


def _y(shape, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _step_loops(buf, power, Q, G, alpha, taps, delay):
    """The step written with explicit loops over bins and indices."""
    L, F, D = buf.shape
    n = taps * D
    pred, Qk, Gk = np.empty((F, D), complex), np.empty((F, n, n), complex), np.empty((F, n, D), complex)
    for f in range(F):
        w = np.zeros(n, complex)
        for d in range(D):
            for k in range(taps):
                w[d * taps + k] = buf[L - delay - 2 - k, f, d]
        for d in range(D):
            pred[f, d] = buf[-1, f, d] - sum(np.conj(G[f, i, d]) * w[i] for i in range(n))
        u = np.array([sum(Q[f, i, j] * w[j] for j in range(n)) for i in range(n)])
        den = alpha * power[f] + sum(np.conj(w[i]) * u[i] for i in range(n))
        k = u / den
        v = np.array([sum(np.conj(w[j]) * Q[f, j, m] for j in range(n)) for m in range(n)])
        for i in range(n):
            for m in range(n):
                Qk[f, i, m] = (Q[f, i, m] - k[i] * v[m]) / alpha
            for d in range(D):
                Gk[f, i, d] = G[f, i, d] + k[i] * np.conj(pred[f, d])
    return pred, Qk, Gk


@pytest.mark.parametrize('F,D,taps,delay,alpha', [(1, 1, 1, 0, 1.0), (3, 2, 3, 1, 0.99), (2, 3, 2, 2, 0.9)])
def test_step_matches_scalar_loops(F, D, taps, delay, alpha):
    n = taps * D
    buf = _y((taps + delay + 1, F, D), 1)
    A = _y((F, n, n), 2)
    Q = A @ A.conj().transpose(0, 2, 1) + n * np.eye(n)
    G = _y((F, n, D), 3)
    power = np.random.default_rng(4).random(F) + 0.5
    got = O.online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    want = _step_loops(buf, power, Q, G, alpha, taps, delay)
    for g, w in zip(got, want):
        np.testing.assert_allclose(g, w, rtol=1e-12, atol=1e-12 * np.abs(w).max())


def test_window_index_is_d_taps_plus_k():
    taps, delay, D = 3, 2, 4
    L = taps + delay + 1
    for d in range(D):
        for k in range(taps):
            buf = np.zeros((L, 1, D), complex)
            buf[L - delay - 2 - k, 0, d] = 1
            w = O.window(buf, taps, delay)[0]
            assert np.flatnonzero(w).tolist() == [d * taps + k]
            # and through the step: u = Q w = e_{d taps + k} with Q = I
            Q = np.eye(taps * D)[None].astype(complex)
            _, Qk, _ = O.online_wpe_step(buf, np.ones(1), Q, np.zeros((1, taps * D, D)), 1.0, taps, delay)
            i = d * taps + k
            assert Qk[0, i, i] == 0.5


def test_wrong_buffer_length_raises():
    with pytest.raises(ValueError):
        O.online_wpe_step(np.zeros((5, 1, 2), complex), np.ones(1), np.eye(6)[None], np.zeros((1, 6, 2)), 1.0, 3, 2)


@pytest.mark.parametrize('alpha', [1.0, 0.99, 0.9])
def test_closed_form(alpha):
    """Q_t = R_t^-1 and G_t = R_t^-1 sum_s alpha^(t-s) w_s y_s^H / lambda_s with
    R_t = alpha^t I + sum_s alpha^(t-s) w_s w_s^H / lambda_s, to n eps kappa(R_t)."""
    T, F, D, taps, delay = 40, 2, 2, 3, 1
    n, L = taps * D, taps + delay + 1
    Y = _y((T, F, D), 5)
    Q = np.broadcast_to(np.eye(n, dtype=complex), (F, n, n)).copy()
    G = np.zeros((F, n, D), complex)
    stream = np.concatenate([np.zeros((L - 1, F, D)), Y])
    R = np.broadcast_to(np.eye(n, dtype=complex), (F, n, n)).copy()
    P = np.zeros((F, n, D), complex)
    for t in range(T):
        buf = stream[t:t + L]
        lam = np.mean(np.abs(buf) ** 2, axis=(0, 2))
        _, Q, G = O.online_wpe_step(buf, lam, Q, G, alpha, taps, delay)
        w = O.window(buf, taps, delay)
        R = alpha * R + np.einsum('fi,fj->fij', w, w.conj()) / lam[:, None, None]
        P = alpha * P + np.einsum('fi,fd->fid', w, buf[-1].conj()) / lam[:, None, None]
        for f in range(F):
            kappa = np.linalg.cond(R[f])
            Rinv = np.linalg.inv(R[f])
            tol = n * EPS * kappa
            assert np.abs(Q[f] - Rinv).max() <= tol * np.abs(Rinv).max()
            Gw = np.linalg.solve(R[f], P[f])
            assert np.abs(G[f] - Gw).max() <= tol * max(np.abs(Gw).max(), 1.0)


def test_get_power_online_is_get_power_inf():
    x = _y((5, 3, 17), 6)
    np.testing.assert_allclose(O.get_power_online(x), W.get_power(x, np.inf)[..., 0], rtol=1e-14)


@pytest.mark.parametrize('cuts', [[1], [3], [5, 6, 20], list(range(1, 30))])
def test_chunked_equals_one_call(cuts):
    T, F, D, taps, delay, alpha = 30, 2, 2, 3, 2, 0.99
    Y = _y((T, F, D), 7)
    Z, st = O.online_wpe(Y, taps, delay, alpha)
    parts, state = [], None
    for a, b in zip([0] + cuts, cuts + [T]):
        z, state = O.online_wpe(Y[a:b], taps, delay, alpha, state)
        parts.append(z)
    np.testing.assert_array_equal(np.concatenate(parts), Z)
    for a, b in zip(state, st):
        np.testing.assert_array_equal(a, b)
