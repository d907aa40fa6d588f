"""GPU checks of SI-SDR and the invasive SxR (pb_bss_b200.evaluation.si_sdr / sxr_module): every case of
tests/golden/metrics.npz (what the reference computes), agreement with the NumPy restatement (oracle/sxr_oracle.py)
at lengths from 1 to 2^22, exact inf / nan cases, input types, broadcasting and bitwise batch independence."""
import itertools

import numpy as np
import pytest

from oracle import sxr_oracle as O
from oracle.make_golden_metrics import SNR_AXES

pytestmark = pytest.mark.gpu

RTOL = 1e-12          # end to end: the length-n sums run in another order than NumPy's
ULP = 4 * np.finfo(np.float64).eps   # from the same S and N: the same IEEE operations, CUDA's log10 within 1 ulp


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _close(got, want, rtol, atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(np.where(np.isinf(want), want, 0), np.where(np.isinf(got), got, 0))
    finite = np.isfinite(want)
    np.testing.assert_allclose(got[finite], want[finite], rtol=rtol, atol=atol)


def _scale(g, c, suffix):
    """The largest finite |dB| of a case before any average: a source mean of values of opposite sign cancels, so the
    errors of the means are relative to it."""
    v = np.concatenate([np.ravel(g[f'{c}_{key}_{suffix}']) for key in ('sdr', 'sir', 'snr')])
    v = np.abs(v[np.isfinite(v)])
    return float(v.max()) if v.size else 0.0


def _names(g, prefix, suffix):
    return sorted(k[:-len(suffix)] for k in g if k.startswith(prefix) and k.endswith(suffix))


# ---- fixtures of the reference --------------------------------------------------------------------------------------

def test_si_sdr_doctest_cases(golden):
    from pb_bss_b200.evaluation import si_sdr
    g = golden('metrics')
    for c in _names(g, 'sisdr_', '_value'):
        r, e, want = g[c + '_reference'], g[c + '_estimation'], g[c + '_value']
        got = si_sdr(r, e)
        assert isinstance(got, np.float64 if want.ndim == 0 else np.ndarray)
        _close(got, want, RTOL)
        _close(si_sdr(_cuda(r), _cuda(e)).cpu().numpy(), want, RTOL)
    assert si_sdr(g['sisdr_1_reference'], g['sisdr_1_estimation']) == np.inf
    assert np.isnan(si_sdr([1., 0], [0., 0]))


def test_input_sxr_fixtures(golden):
    from pb_bss_b200.evaluation import sxr_module as M
    g = golden('metrics')
    cases = _names(g, 'sxr_in_', '_images')
    assert len(cases) >= 14
    for c in cases:
        images, noise = g[c + '_images'], g[c + '_noise']
        _close(M.get_variance_for_zero_mean_signal(images, axis=-1), g[c + '_S'], RTOL)
        scale = max(_scale(g, c, '00'), _scale(g, c, '01'))
        for avg_s, avg_c in itertools.product((0, 1), repeat=2):
            want = [g[f'{c}_{key}_{avg_s}{avg_c}'] for key in ('sdr', 'sir', 'snr')]
            direct = M.input_sxr_from_powers(_cuda(g[c + '_S']), _cuda(g[c + '_N']), avg_s, avg_c)
            for v, w in zip(direct, want):
                _close(v.cpu().numpy(), w, ULP, atol=ULP * scale)
            for v, w in zip(M.input_sxr(images, noise, bool(avg_s), bool(avg_c)), want):
                _close(v, w, RTOL, atol=RTOL * scale)


def test_output_sxr_fixtures(golden):
    from pb_bss_b200.evaluation import sxr_module as M
    g = golden('metrics')
    cases = _names(g, 'sxr_out_', '_contribution')
    assert len(cases) >= 20
    for c in cases:
        contribution, noise = g[c + '_contribution'], g[c + '_noise']
        scale = _scale(g, c, '0')
        for avg in (0, 1):
            want = [g[f'{c}_{key}_{avg}'] for key in ('sdr', 'sir', 'snr')]
            *direct, selection = M.output_sxr_from_powers(_cuda(g[c + '_S']), _cuda(g[c + '_N']), avg)
            np.testing.assert_array_equal(selection.cpu().numpy(), g[c + '_selection'], err_msg=c)
            for v, w in zip(direct, want):
                _close(v.cpu().numpy(), w, ULP, atol=ULP * scale)
            for v, w in zip(M.output_sxr(contribution, noise, bool(avg)), want):
                _close(v, w, RTOL, atol=RTOL * scale)
            # the selection from the device's own powers
            S = M._variance(contribution, axis=-1)
            N = M._variance(noise, axis=-1)
            np.testing.assert_array_equal(M.output_sxr_from_powers(S, N, avg)[3].cpu().numpy(), g[c + '_selection'])


def test_get_snr_fixtures(golden):
    from pb_bss_b200.evaluation.sxr_module import get_snr
    g = golden('metrics')
    for i, (axis, keepdims) in enumerate(SNR_AXES):
        want = g[f'snr_{i}_value']
        got = get_snr(g['snr_X'], g['snr_N'], axis=axis, keepdims=keepdims)
        _close(got, want, RTOL)
        _close(get_snr(_cuda(g['snr_X']), _cuda(g['snr_N']), axis=axis, keepdims=keepdims).cpu().numpy(), want, RTOL)
    assert get_snr([1, 2, 3], [1, 2, 3]) == 0.0


# ---- SI-SDR against the restatement ---------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [1, 2, 3, 7, 255, 256, 257, 8191, 8192, 8193, 16385, 65537, 1 << 22])
def test_si_sdr_matches_oracle(n):
    from pb_bss_b200.evaluation import si_sdr
    rng = np.random.default_rng(n)
    r = rng.standard_normal((3, n))
    e = 0.7 * r + 10.0 ** -rng.uniform(0.5, 2.5, (3, 1)) * rng.standard_normal((3, n))
    _close(si_sdr(r, e), O.si_sdr(r, e), RTOL, atol=1e-9)


@pytest.mark.parametrize('n', [1, 5, 100, 8193, 100000])
def test_si_sdr_exact_cases(n):
    from pb_bss_b200.evaluation import si_sdr
    r = np.random.default_rng(n).standard_normal(n)
    for j in range(-4, 5):
        assert si_sdr(r, 2.0 ** j * r) == np.inf
    assert np.isnan(si_sdr(r, np.zeros(n)))
    assert np.isnan(si_sdr(np.zeros(n), r))


def test_si_sdr_broadcast_and_types():
    import torch
    from pb_bss_b200.evaluation import si_sdr
    rng = np.random.default_rng(3)
    src, obs = rng.standard_normal((2, 1, 5000)), rng.standard_normal((1, 6, 5000))
    got = si_sdr(src, obs)
    assert got.shape == (2, 6)
    np.testing.assert_array_equal(got, si_sdr(np.broadcast_to(src, (2, 6, 5000)).copy(),
                                              np.broadcast_to(obs, (2, 6, 5000)).copy()))
    _close(got, O.si_sdr(src, obs), RTOL)
    cuda = si_sdr(_cuda(src), obs)
    assert cuda.is_cuda and cuda.dtype == torch.float64
    np.testing.assert_array_equal(cuda.cpu().numpy(), got)
    with pytest.raises(AssertionError):
        si_sdr(src.astype(np.float32), obs)
    with pytest.raises(AssertionError):
        si_sdr(_cuda(src).float(), obs)
    assert si_sdr(np.zeros((0, 10)), np.zeros((0, 10))).shape == (0,)


def test_si_sdr_row_is_bitwise_batch_independent():
    from pb_bss_b200.evaluation import si_sdr
    rng = np.random.default_rng(4)
    r, e = rng.standard_normal((1000, 20001)), rng.standard_normal((1000, 20001))
    e += 3 * r
    batch = si_sdr(r, e)
    for i in (0, 517, 999):
        assert si_sdr(r[i], e[i]) == batch[i]


# ---- the powers ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', ['float32', 'float64', 'int16', 'int32', 'int64', 'complex64', 'complex128'])
def test_variance_every_dtype(dtype):
    import torch
    from pb_bss_b200.evaluation.sxr_module import get_variance_for_zero_mean_signal as var
    rng = np.random.default_rng(5)
    x = rng.standard_normal((3, 4, 9001)) * 1000
    if dtype.startswith('complex'):
        x = x + 1j * rng.standard_normal(x.shape) * 1000
    x = x.astype(dtype)
    want = O.power(x, axis=-1)
    _close(var(x, axis=-1), want, RTOL)
    got = var(_cuda(x), axis=-1)
    assert got.is_cuda and got.dtype == torch.float64
    _close(got.cpu().numpy(), want, RTOL)
    for axis, keepdims in ((None, False), (None, True), ((0, 2), True), (1, False)):
        _close(var(x, axis=axis, keepdims=keepdims), O.power(x, axis=axis, keepdims=keepdims), RTOL)


def test_variance_long_row_and_batch_independence():
    from pb_bss_b200.evaluation.sxr_module import get_variance_for_zero_mean_signal as var
    rng = np.random.default_rng(6)
    x = rng.standard_normal(1 << 24)
    got = var(x)
    assert isinstance(got, np.float64)
    _close(got, O.power(x), RTOL)
    rows = rng.standard_normal((1000, 12345))
    batch = var(rows, axis=-1)
    for i in (0, 500, 999):
        assert var(rows[i]) == batch[i]
    assert np.isnan(var(np.zeros((2, 0)), axis=-1)).all()


def test_errors():
    from pb_bss_b200.evaluation import sxr_module as M
    with pytest.raises(ValueError, match='empty sequence'):
        M.output_sxr(np.ones((3, 2, 10)), np.ones((2, 10)))
    with pytest.raises(AssertionError):
        M.input_sxr(np.ones((10, 1, 10)), np.ones((1, 10)))
    with pytest.raises(AssertionError):
        M.input_sxr(np.ones((2, 1, 10)), np.ones((2, 10)))
    r = M.input_sxr(np.ones((2, 1, 10)), np.ones((1, 10)), return_dict='input_')
    assert sorted(r) == ['input_sdr', 'input_sir', 'input_snr']
    # output_sxr tests `return_dict is True`, so a string prefix gives the tuple, as in the reference
    assert isinstance(M.output_sxr(np.ones((2, 2, 10)), np.ones((2, 10)), return_dict='x_'), M.ResultTuple)
