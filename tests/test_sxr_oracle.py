"""CPU checks of the NumPy restatement of SI-SDR and the invasive SxR (oracle/sxr_oracle.py) against what the
reference computes (tests/golden/metrics.npz): selections exactly, inf / nan in the same places, finite values to
1e-14 relative.  Also that np_sum is NumPy's summation order, on which the device kernels' bits rest."""
import itertools

import numpy as np
import pytest

from oracle import sxr_oracle as O
from oracle.make_golden_metrics import SNR_AXES, wrapper_images

RTOL = 1e-14


def _same(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(np.isinf(got) & (got > 0), np.isinf(want) & (want > 0))
    np.testing.assert_array_equal(np.isinf(got) & (got < 0), np.isinf(want) & (want < 0))
    finite = np.isfinite(want)
    np.testing.assert_allclose(got[finite], want[finite], rtol=RTOL, atol=0)


def _names(g, prefix, suffix):
    return sorted(k[:-len(suffix)] for k in g if k.startswith(prefix) and k.endswith(suffix))


def test_np_sum_is_numpy_summation_order():
    rng = np.random.default_rng(0)
    for n in range(0, 40):
        v = rng.random(n) * 10.0 ** rng.integers(-8, 8, n)
        assert O.np_sum(v) == np.sum(v)
    for K in range(1, 10):
        for D in range(1, 30):
            a = rng.random((K, D)) * 10.0 ** rng.integers(-8, 8, (K, D))
            np.testing.assert_array_equal(O._mean_rows(a), np.mean(a, axis=0))
            np.testing.assert_array_equal([O.np_sum(r) / D for r in a], np.mean(a, axis=-1))


def test_si_sdr_doctest_cases(golden):
    g = golden('metrics')
    cases = _names(g, 'sisdr_', '_value')
    assert len(cases) == 8
    for c in cases:
        _same(O.si_sdr(g[c + '_reference'], g[c + '_estimation']), g[c + '_value'])
    assert g['sisdr_0_value'] == np.inf and g['sisdr_1_value'] == np.inf and np.isnan(g['sisdr_6_value'])


def test_input_sxr(golden):
    g = golden('metrics')
    cases = _names(g, 'sxr_in_', '_images')
    assert len(cases) >= 14
    for c in cases:
        S, N = O.power(g[c + '_images'], axis=-1), O.power(g[c + '_noise'], axis=-1)
        _same(S, g[c + '_S'])
        _same(N, g[c + '_N'])
        for avg_s, avg_c in itertools.product((0, 1), repeat=2):
            got = O.input_sxr_from_powers(g[c + '_S'], g[c + '_N'], avg_s, avg_c)
            for key, v in zip(('sdr', 'sir', 'snr'), got):
                _same(v, g[f'{c}_{key}_{avg_s}{avg_c}'])


def test_output_sxr(golden):
    g = golden('metrics')
    cases = _names(g, 'sxr_out_', '_contribution')
    assert len(cases) >= 20
    for c in cases:
        _same(O.power(g[c + '_contribution'], axis=-1), g[c + '_S'])
        for avg in (0, 1):
            *values, selection = O.output_sxr_from_powers(g[c + '_S'], g[c + '_N'], avg)
            np.testing.assert_array_equal(selection, g[c + '_selection'])
            for key, v in zip(('sdr', 'sir', 'snr'), values):
                _same(v, g[f'{c}_{key}_{avg}'])


def test_output_sxr_more_sources_than_targets_raises():
    with pytest.raises(ValueError, match='empty sequence'):
        O.output_sxr_from_powers(np.ones((3, 2)), np.ones(2))


def test_get_snr(golden):
    g = golden('metrics')
    for i, (axis, keepdims) in enumerate(SNR_AXES):
        got = 10 * np.log10(O.power(g['snr_X'], axis, keepdims) / O.power(g['snr_N'], axis, keepdims))
        _same(got, g[f'snr_{i}_value'])


def test_wrapper_anchors_are_stored(golden):
    g, b = golden('metrics'), golden('bss_eval')
    for prefix in ('input', 'output'):
        for key in ('invasive_sdr', 'invasive_sir', 'invasive_snr', 'srmr'):
            assert f'anchor_{prefix}_{key}' in g and f'anchor_{prefix}_{key}_rtol' in g
    images, noise = wrapper_images(b['input_source'], b['input_observation'], g['wrapper_taps'])
    assert images.shape == (2, 3, 10000) and noise.shape == (3, 10000)
    # the restatement meets the published invasive anchors of test_input_metrics on the rebuilt images
    S, N = O.power(images, axis=-1), O.power(noise, axis=-1)
    for key, v in zip(('sdr', 'sir', 'snr'), O.input_sxr_from_powers(S, N, False, False)):
        np.testing.assert_allclose(v, g[f'anchor_input_invasive_{key}'], rtol=g[f'anchor_input_invasive_{key}_rtol'])
