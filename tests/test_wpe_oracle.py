"""The WPE oracle (oracle/wpe_oracle.py) against independent facts: explicit loops, brute-force means, the normal
equations of the weighted least-squares problem and the special cases its arithmetic implies."""
import numpy as np
import pytest

from oracle import wpe_oracle as W


def _y(shape, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


@pytest.mark.parametrize('taps,delay', [(1, 0), (3, 2), (5, 0), (2, 7)])
def test_build_y_tilde_matches_a_loop(taps, delay):
    Y = _y((2, 3, 4, 9))
    out = W.build_y_tilde(Y, taps, delay)
    assert out.shape == (2, 3, taps * 4, 9)
    for k in range(taps):
        for d in range(4):
            for t in range(9):
                s = t - delay - k
                want = Y[..., d, s] if s >= 0 else 0
                np.testing.assert_array_equal(out[..., k * 4 + d, t], want)


@pytest.mark.parametrize('c', [1, 2, 5, 9, 30])
def test_window_mean_matches_brute_force(c):
    x = np.random.default_rng(1).random((3, 10))
    want = np.stack([[x[i, max(0, t - c):t + c + 1].mean() for t in range(10)] for i in range(3)])
    np.testing.assert_allclose(W.window_mean(x, c), want, rtol=1e-14)


def test_get_power_contexts():
    Y = _y((4, 3, 11), 2)
    lam = np.mean(np.abs(Y) ** 2, axis=-2)
    np.testing.assert_allclose(W.get_power(Y), lam, rtol=1e-15)
    np.testing.assert_allclose(W.get_power(Y, np.inf), np.broadcast_to(lam.mean(-1, keepdims=True), lam.shape),
                               rtol=1e-14)
    np.testing.assert_allclose(W.get_power(Y, 2), W.window_mean(lam, 2), rtol=1e-15)
    inv = W.get_power_inverse(Y)
    np.testing.assert_allclose(inv, 1 / np.maximum(lam, 1e-10 * lam.max()), rtol=1e-15)
    with pytest.raises(ValueError):
        W.get_power(Y, -1)


@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_last_solve_satisfies_the_normal_equations(mode):
    """X = Y - G^H Yt with G solving R G = P makes the weighted residual orthogonal to the delayed stack."""
    Y = _y((4, 300), 3)
    X, (w, R, P, G), fell = W.wpe_bin(Y, taps=5, delay=2, iterations=2, statistics_mode=mode, details=True)
    assert not fell
    Yt = W.build_y_tilde(Y, 5, 2)
    s = slice(6, None) if mode == 'valid' else slice(None)
    resid = (Yt[:, s] * w[s]) @ X[:, s].conj().T
    scale = np.abs(Yt[:, s] * w[s]) @ np.abs(X[:, s]).T
    assert np.abs(resid).max() < 1e-12 * scale.max()


def test_valid_equals_full_on_cropped_statistics():
    Y = _y((3, 120), 4)
    taps, delay = 4, 2
    tb = taps + delay - 1
    w = W.get_power_inverse(Y)
    Yt = W.build_y_tilde(Y, taps, delay)
    R = (Yt[:, tb:] * w[tb:]) @ Yt[:, tb:].conj().T
    P = (Yt[:, tb:] * w[tb:]) @ Y[:, tb:].conj().T
    want = Y - np.linalg.solve(R, P).conj().T @ Yt
    got = W.wpe(Y, taps, delay, iterations=1, statistics_mode='valid')
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * np.abs(Y).max())


def test_special_cases():
    Y = _y((3, 2, 50), 5)
    out = W.wpe(Y, iterations=0)
    np.testing.assert_array_equal(out, Y)
    assert out is not Y
    # a dead channel makes R exactly singular: the lstsq branch, finite output
    Yd = Y[0].copy()
    Yd[1] = 0
    X, _, fell = W.wpe_bin(Yd, taps=3, delay=1, details=True)
    assert fell and np.isfinite(X).all()
    # an all-zero bin is NaN in that bin only
    Yz = Y.copy()
    Yz[1] = 0
    X = W.wpe(Yz, taps=3, delay=1)
    assert np.isnan(X[1]).all() and np.isfinite(X[[0, 2]]).all()
    # 'valid' without any frame in the statistics: R = P = 0, G = 0, X = Y
    Ys = Y[:, :, :5]
    np.testing.assert_array_equal(W.wpe(Ys, taps=3, delay=3, statistics_mode='valid'), Ys)
    # in place
    Yc = Y.copy()
    assert W.wpe(Yc, taps=2, delay=1, inplace=True) is Yc
    np.testing.assert_array_equal(Yc, W.wpe(Y, taps=2, delay=1))
    with pytest.raises(ValueError):
        W.wpe(Y, statistics_mode='cropped')
