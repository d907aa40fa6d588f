"""CPU checks of the ESTOI restatement (oracle/estoi_oracle.py): against a literal loop transcription of Jensen and
Taal's per-segment measure, its invariances (d(x, x) = 1, scale invariance of the estimate), the zero-norm rule that
replaces pystoi's random noise, and the STOI stages and < 30-frame rule it shares with oracle/stoi_oracle.py; and
the argument checks pbb_estoi shares with pbb_stoi, which raise before any device work."""
import math
import warnings

import numpy as np
import pytest

from oracle import estoi_oracle as E
from oracle import stoi_oracle as S


def _normalise_rows(A):
    """Per band: minus the mean over the frames, over the root of the sum of squares (0 where that sum is zero up to
    rounding: at most TINY times the sum of squares before centring)."""
    B, N = len(A), len(A[0])
    out = [[0.0] * N for _ in range(B)]
    for b in range(B):
        mu, raw = 0.0, 0.0
        for n in range(N):
            mu += A[b][n]
            raw += A[b][n] ** 2
        mu /= N
        ss = 0.0
        for n in range(N):
            ss += (A[b][n] - mu) ** 2
        inv = 0.0 if ss <= E.TINY * raw else 1.0 / math.sqrt(ss)
        for n in range(N):
            out[b][n] = (A[b][n] - mu) * inv
    return out


def _normalise_columns(A):
    """Per frame: minus the mean over the bands, over the root of the sum of squares (0 where that sum is zero up to
    rounding)."""
    B, N = len(A), len(A[0])
    out = [[0.0] * N for _ in range(B)]
    for n in range(N):
        mu, raw = 0.0, 0.0
        for b in range(B):
            mu += A[b][n]
            raw += A[b][n] ** 2
        mu /= B
        ss = 0.0
        for b in range(B):
            ss += (A[b][n] - mu) ** 2
        inv = 0.0 if ss <= E.TINY * raw else 1.0 / math.sqrt(ss)
        for b in range(B):
            out[b][n] = (A[b][n] - mu) * inv
    return out


def loop_d(X, Y):
    """d of one 15 x 30 segment: the row- then column-normalised X and Y, (1/N) sum_n sum_b X[b, n] Y[b, n]."""
    Xn = _normalise_columns(_normalise_rows(X.tolist()))
    Yn = _normalise_columns(_normalise_rows(Y.tolist()))
    B, N = len(Xn), len(Xn[0])
    d = 0.0
    for n in range(N):
        for b in range(B):
            d += Xn[b][n] * Yn[b][n]
    return d / N


def loop_estoi(x_tob, y_tob):
    M = x_tob.shape[1]
    ds = [loop_d(x_tob[:, m:m + E.N], y_tob[:, m:m + E.N]) for m in range(M - E.N + 1)]
    return sum(ds) / len(ds)


def _envelopes(rng, M):
    """Band-envelope-like (15, M): positive, with a per-band level and slow modulation."""
    level = np.exp(rng.uniform(-3, 3, size=(15, 1)))
    mod = 1.0 + 0.8 * np.sin(np.arange(M)[None] / rng.uniform(2, 8, size=(15, 1)))
    return level * mod * rng.uniform(0.2, 1.0, size=(15, M))


def _signals(seed, n=16000, fs=10000):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    x = rng.standard_normal(n) * (1.2 + np.sin(2 * np.pi * 3 * t)) ** 2
    y = x + 0.7 * rng.standard_normal(n)
    return x, y


@pytest.mark.parametrize('seed', range(4))
def test_vectorised_segments_match_the_loop(seed):
    rng = np.random.default_rng(seed)
    xt, yt = _envelopes(rng, 36), _envelopes(rng, 36)
    yt[:, :] += 0.5 * xt
    d = E.segment_values(xt, yt)
    assert d.shape == (7,)
    for m in range(7):
        assert abs(d[m] - loop_d(xt[:, m:m + 30], yt[:, m:m + 30])) <= 1e-14
    assert abs(E.from_bands(xt, yt) - loop_estoi(xt, yt)) <= 1e-14
    assert abs(E.from_bands(xt, yt) - d.mean()) <= 1e-15


def test_full_signal_matches_the_loop():
    x, y = _signals(1)
    st = E.stages(x, y, 10000)
    assert st['M'] >= 100
    want = loop_estoi(st['x_tob'], st['y_tob'])
    assert abs(st['value'] - want) <= 1e-13
    assert abs(E.stoi(x, y, 10000, extended=True) - want) <= 1e-13
    # STOI itself is unchanged by the switch
    assert E.stoi(x, y, 10000) == S.stoi(x, y, 10000)
    assert E.stoi(x, y, 10000, extended=False) == S.stoi(x, y, 10000)
    assert E.stoi(x, y, 10000, extended=True) != S.stoi(x, y, 10000)


def test_identical_inputs_give_one():
    rng = np.random.default_rng(2)
    xt = _envelopes(rng, 80)
    assert abs(E.from_bands(xt, xt) - 1.0) <= 1e-14
    np.testing.assert_allclose(E.segment_values(xt, xt), 1.0, rtol=0, atol=1e-14)
    x, _ = _signals(3)
    assert abs(E.stoi(x, x, 10000, extended=True) - 1.0) <= 1e-14


@pytest.mark.parametrize('c', [1e-3, 0.37, 3.7, 2.0 ** 20])
def test_scaling_the_estimate_leaves_the_value(c):
    rng = np.random.default_rng(4)
    xt, yt = _envelopes(rng, 60), _envelopes(rng, 60)
    assert abs(E.from_bands(xt, c * yt) - E.from_bands(xt, yt)) <= 1e-13
    x, y = _signals(5)
    assert abs(E.stoi(x, c * y, 10000, extended=True) - E.stoi(x, y, 10000, extended=True)) <= 1e-13


def test_value_lies_in_minus_one_to_one():
    rng = np.random.default_rng(6)
    for _ in range(5):
        xt, yt = _envelopes(rng, 45), _envelopes(rng, 45)
        d = E.segment_values(xt, yt)
        assert np.all(np.abs(d) <= 1.0 + 1e-14)
        assert abs(E.from_bands(xt, -yt + 100.0) + E.from_bands(xt, yt - 100.0)) <= 1e-13


def test_zero_norm_rule_on_a_hand_built_segment():
    rng = np.random.default_rng(7)
    X = _envelopes(rng, 30)
    X[3] = 0.0                                  # an all-zero band of the reference
    Y = np.zeros((15, 30))                      # an all-zero estimate
    rows = E._normalise(X, -1)
    np.testing.assert_array_equal(rows[3], 0.0)
    np.testing.assert_allclose(np.sum(np.delete(rows, 3, 0) ** 2, axis=1), 1.0, rtol=1e-14)
    Xn = E.row_col_normalize(X)
    assert np.all(np.isfinite(Xn))
    np.testing.assert_allclose(np.sum(Xn ** 2, axis=0), 1.0, rtol=1e-14)
    Yn = E.row_col_normalize(Y)
    np.testing.assert_array_equal(Yn, 0.0)     # zeros, where 1 / sqrt(0) would give NaN
    assert E.from_bands(X, Y) == 0.0 and loop_d(X, Y) == 0.0
    assert abs(E.from_bands(X, X) - 1.0) <= 1e-14
    assert abs(E.from_bands(X, X) - loop_d(X, X)) <= 1e-14
    # the estimate zero except in one band, constant over time there: zero after the row step, so every column too
    Y[5] = 2.0 ** -3
    np.testing.assert_array_equal(E.row_col_normalize(Y), 0.0)


def test_one_non_zero_frame_normalises_to_zeros():
    """The first (or last) segment of a silent stretch of the estimate: one non-zero frame.  Every band normalises to
    the pattern (29, -1, ..., -1) / sqrt(870), so every column is constant in exact arithmetic; in floating point it
    centres to rounding noise, which the rule maps to zeros, as exact arithmetic would."""
    rng = np.random.default_rng(12)
    X = _envelopes(rng, 30)
    for n in (0, 29):
        Y = np.zeros((15, 30))
        Y[:, n] = rng.uniform(1, 40, 15)
        rows = E._normalise(Y, -1)
        want = np.full(30, -1.0 / np.sqrt(870.0))
        want[n] = 29.0 / np.sqrt(870.0)
        np.testing.assert_allclose(rows, np.broadcast_to(want, (15, 30)), rtol=1e-14)
        np.testing.assert_array_equal(E.row_col_normalize(Y), 0.0)
        assert E.from_bands(X, Y) == 0.0 and loop_d(X, Y) == 0.0
    # two non-zero frames with different spectra are an ordinary segment
    Y[:, 3] = rng.uniform(1, 40, 15)
    assert np.all(np.abs(np.sum(E.row_col_normalize(Y) ** 2, axis=0) - 1.0) <= 1e-14)
    assert abs(E.from_bands(X, Y) - loop_d(X, Y)) <= 1e-14


def test_non_finite_envelopes_propagate():
    rng = np.random.default_rng(8)
    xt, yt = _envelopes(rng, 40), _envelopes(rng, 40)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        yt[4, 20] = np.nan
        assert np.isnan(E.from_bands(xt, yt))
        yt[4, 20] = np.inf
        assert np.isnan(E.from_bands(xt, yt))


def test_estimate_silent_over_many_frames_is_finite():
    x, y = _signals(9, n=30000)
    y[8000:20000] = 0.0                         # about 90 STFT frames of digital silence in the estimate
    st = E.stages(x, y, 10000)
    assert np.sum(np.all(st['y_tob'] == 0.0, axis=0)) >= 60
    v = E.stoi(x, y, 10000, extended=True)
    assert np.isfinite(v) and abs(v - loop_estoi(st['x_tob'], st['y_tob'])) <= 1e-13


def test_fewer_than_thirty_frames_warns_and_gives_1e_5():
    rng = np.random.default_rng(10)
    x, y = rng.standard_normal(256 + 128 * 30), rng.standard_normal(256 + 128 * 30)   # M = 29
    with pytest.warns(RuntimeWarning, match='Not enough STFT frames'):
        assert E.stoi(x, y, 10000, extended=True) == 1e-5
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        x, y = rng.standard_normal(256 + 128 * 31), rng.standard_normal(256 + 128 * 31)  # M = 30: one segment
        st = E.stages(x, y, 10000)
        assert st['M'] == 30 and abs(st['value'] - loop_d(st['x_tob'], st['y_tob'])) <= 1e-14


def test_broadcasting():
    x, y = _signals(11, n=12000)
    X = np.stack([x, y])[:, None]
    Y = np.stack([y, x, 0.5 * y])[None]
    out = E.stoi(X, Y, 10000, extended=True)
    assert out.shape == (2, 3)
    for a in range(2):
        for b in range(3):
            assert out[a, b] == E.stoi(X[a, 0], Y[0, b], 10000, extended=True)
    assert np.ndim(E.stoi(x, y, 10000, extended=True)) == 0


def test_abi_rejects_bad_arguments_like_pbb_stoi():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    for name in ('pbb_stoi', 'pbb_estoi'):
        f = getattr(lib, name)
        rc = f(None, None, _lib.PBB_F64, 1, 4000, 5, 4, None, 0, 0, None, None, None, 1, None, 0, None, None, None,
               None, None, None)
        assert rc == -1 and b'x is null' in lib.pbb_last_error()
        rc = f(1, 1, _lib.PBB_F64, 1, 204, 5, 4, None, 0, 0, None, None, None, 1, None, 0, None, None, None, None,
               None, None)
        assert rc == -5
        rc = f(1, 1, 7, 1, 4000, 5, 4, None, 0, 0, None, None, None, 1, None, 0, None, None, None, None, None, None)
        assert rc == -3
