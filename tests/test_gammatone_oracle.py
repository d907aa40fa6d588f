"""CPU checks of the gammatone filterbank: the NumPy restatement (oracle/gammatone_oracle.py) and the host-side
coefficients of pb_bss_b200.transform.gammatone against the unmodified reference (tests/golden/gammatone.npz), and
the chunked scan of csrc/gammatone.cuh restated in NumPy against the sequential cascade."""
import numpy as np
import pytest

from oracle import gammatone_oracle as GO
from oracle.make_golden_gammatone import CASES
from pb_bss_b200.transform import gammatone as G

COEF_KEYS = [f'coef_{sr}_{n}_{lo}_{int(hi)}' for sr in (8000, 16000, 44100, 48000) for n in (1, 2, 23, 64)
             for lo, hi in ((125, sr / 2), (100, 6000))]


def _params(key):
    _, sr, n, lo, hi = key.split('_')
    return int(sr), int(n), float(lo), float(hi)


@pytest.mark.parametrize('key', COEF_KEYS)
def test_oracle_coefficients_match_the_reference(golden, key):
    g = golden('gammatone')
    sr, n, lo, hi = _params(key)
    cfs = GO.centre_frequencies(lo, hi, n)
    np.testing.assert_allclose(cfs, g[key + '_cfs'], rtol=1e-13, atol=0)
    A0, A11, A12, A13, A14, A2, B0, B1, B2, gain = GO.coefficients(cfs, sr)
    np.testing.assert_array_equal([A0, A2, B0], g[key + '_A0_A2_B0'])
    for name, v in zip(('A11', 'A12', 'A13', 'A14', 'B1', 'B2', 'gain'), (A11, A12, A13, A14, B1, B2, gain)):
        np.testing.assert_allclose(v, g[f'{key}_{name}'], rtol=1e-13, atol=0, err_msg=name)


@pytest.mark.parametrize('key', COEF_KEYS)
def test_device_table_matches_the_reference(golden, key):
    """The (n, 10) table pb_bss_b200 uploads: (b0, b1) of the four sections with 1 / gain in the first, a1, a2."""
    g = golden('gammatone')
    sr, n, lo, hi = _params(key)
    cfs = G.calculate_cfs(lo, hi, n)
    np.testing.assert_allclose(cfs, g[key + '_cfs'], rtol=1e-13, atol=0)
    table = G.filter_coefficients(cfs, sr)
    T, gain = g[key + '_A0_A2_B0'][0], g[key + '_gain']
    ref = np.stack([T / gain, g[key + '_A11'] / gain, np.full(n, T), g[key + '_A12'], np.full(n, T), g[key + '_A13'],
                    np.full(n, T), g[key + '_A14'], g[key + '_B1'], g[key + '_B2']], axis=1)
    np.testing.assert_allclose(table, ref, rtol=1e-13, atol=0)


def _assert_filter_outputs_close(out, ref, rel):
    """|out - ref| <= rel * max|ref| of each (filter, row)."""
    out, ref = np.asarray(out), np.asarray(ref)
    assert out.shape == ref.shape
    r = ref.reshape(ref.shape[0], -1, ref.shape[-1])
    o = out.reshape(r.shape)
    scale = np.abs(r).max(axis=-1, keepdims=True)
    assert (np.abs(o - r) <= rel * scale).all(), np.max(np.abs(o - r) / scale)


@pytest.mark.parametrize('case', sorted(CASES))
def test_oracle_filterbank_matches_the_reference(golden, case):
    g = golden('gammatone')
    sr, n, lo, hi = g[case + '_params']
    x = g[case + '_x']
    y = GO.gammatone_filterbank(x, int(sr), int(n), lo, hi)
    assert len(y) == int(n) and all(v.dtype == np.float64 and v.shape == x.shape for v in y)
    _assert_filter_outputs_close(np.stack(y), g[case + '_y'], 1e-12)


def test_frequency_scale_matches_the_reference(golden):
    g = golden('gammatone')
    np.testing.assert_allclose([G.Hz_2_ERBS(f) for f in g['hz']], g['hz_erbs'], rtol=1e-15, atol=0)
    np.testing.assert_allclose([G.ERBS_2_Hz(e) for e in g['erbs']], g['erbs_hz'], rtol=1e-15, atol=0)
    np.testing.assert_allclose(G.ERBS_2_Hz(G.Hz_2_ERBS(g['hz'])), g['hz'], rtol=1e-13, atol=1e-10)
    for case in CASES:
        sr, n, lo, hi = g[case + '_params']
        np.testing.assert_allclose(G.calculate_cfs(lo, hi or sr / 2, int(n)), g[case + '_cfs'], rtol=1e-13, atol=0)


def test_invalid_n_raises_what_the_reference_raises(golden):
    g = golden('gammatone')
    x = np.zeros(16)
    for label, n in (('zero', 0), ('negative', -1), ('float', 2.5)):
        expected = {'ZeroDivisionError': ZeroDivisionError, 'ValueError': ValueError, 'TypeError': TypeError}[
            str(g['error_' + label])]
        with pytest.raises(expected):
            G.calculate_cfs(125, 8000, n)
        with pytest.raises(expected):
            G.gammatone_filterbank(x, 16000, n)       # raised on the host, before any device work


def _chunked_scan(x, coef, L):
    """The three passes of csrc/gammatone.cuh in NumPy for one 1-D signal: zero-start chunk end states, the two-level
    carry with M and M^CARRY_GROUP from transition_matrices, and every chunk rerun from its start state."""
    n, N = coef.shape[0], len(x)
    C = -(-N // L)
    trans = G.transition_matrices(coef, L)
    M, MG = trans[:, 0], trans[:, 1]

    def run(xc, s):
        s = s.copy()
        ys = np.empty((n, len(xc)))
        for t, w0 in enumerate(xc):
            w = np.full(n, w0)
            for k in range(4):
                y = coef[:, 2 * k] * w + s[:, 2 * k]
                s[:, 2 * k] = coef[:, 2 * k + 1] * w + s[:, 2 * k + 1] - coef[:, 8] * y
                s[:, 2 * k + 1] = -coef[:, 9] * y
                w = y
            ys[:, t] = w
        return ys, s

    z = np.stack([run(x[c * L:(c + 1) * L], np.zeros((n, 8)))[1] for c in range(C)], axis=1)   # (n, C, 8)
    K = G.CARRY_GROUP
    NG = -(-C // K)
    E = [np.zeros((n, 8))] * NG
    for g in range(NG - 1):
        e = np.zeros((n, 8))
        for c in range(g * K, (g + 1) * K):
            e = np.einsum('nij,nj->ni', M, e) + z[:, c]
        E[g] = e
    S, s = [], np.zeros((n, 8))
    for g in range(NG):
        S.append(s)
        s = np.einsum('nij,nj->ni', MG, s) + E[g]
    starts = np.empty_like(z)
    for g in range(NG):
        s = S[g]
        for c in range(g * K, min((g + 1) * K, C)):
            starts[:, c] = s
            s = np.einsum('nij,nj->ni', M, s) + z[:, c]
    return np.concatenate([run(x[c * L:(c + 1) * L], starts[:, c])[0] for c in range(C)], axis=1)


@pytest.mark.parametrize('sr,L,N', [(16000, 8, 2000), (8000, 4, 700), (48000, 128, 8500)])
def test_chunked_scan_matches_the_sequential_cascade(sr, L, N):
    """Enough chunks to cross several carry groups (CARRY_GROUP chunks each) and end in a partial one; 48 kHz at the
    shortest chunk the library uses is the least accurate case."""
    x = np.random.default_rng(L).standard_normal(N)
    coef = G.filter_coefficients(G.calculate_cfs(125, sr / 2, 5), sr)
    ref = np.stack(GO.gammatone_filterbank(x, sr, 5))
    assert -(-N // L) > 2 * G.CARRY_GROUP
    _assert_filter_outputs_close(_chunked_scan(x, coef, L), ref, 1e-11)   # the device's bound


def test_chunk_length_query():
    """A host-only function of the shape: the largest power of two in [CHUNK_MIN, CHUNK_MAX] that still gives at
    least MIN_CHUNKS (row, filter, chunk) sequences."""
    lo, hi, work = 128, 1024, 65536
    for rows, n, N in ((1, 23, 160000), (8, 23, 160000), (1, 23, 2880000), (1, 1, 100), (3000, 23, 300),
                       (171, 64, 2049), (1, 23, 1 << 22)):
        L = G.chunk_length(rows, n, N)
        assert lo <= L <= hi and L & (L - 1) == 0
        assert L == lo or rows * n * -(-N // L) >= work
        assert L == hi or rows * n * -(-N // (2 * L)) < work
    assert G.chunk_length(8, 23, 160000) == 256
    assert G.chunk_length(1, 23, 2880000) == 512
