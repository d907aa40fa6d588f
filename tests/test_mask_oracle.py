"""CPU checks of oracle/mask_oracle.py (the selection form of the Lorenz threshold, percentiles from explicit order
statistics) against the fixture of the unmodified reference (oracle/make_golden_mask.py) and against np.percentile,
and of the host-side percentile terms the device's quantile_mask is given."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import mask_oracle as MO


@pytest.fixture(scope='module')
def g():
    return load_golden('mask')


def test_lorenz_selection_form_matches_reference(g):
    sig = g['sig']
    np.testing.assert_array_equal(MO.lorenz_mask(sig), g['lorenz'])
    np.testing.assert_array_equal(MO.lorenz_mask(sig, sensor_axis=1), g['lorenz_sens'])
    np.testing.assert_array_equal(MO.lorenz_mask(sig, sensor_axis=1, keepdims=True), g['lorenz_sens_keep'])
    for frac, w in ((0.1, 0.5), (0.4, 0.999), (0.8, 0), (0.89, 1)):
        np.testing.assert_array_equal(MO.lorenz_mask(sig, sensor_axis=0, lorenz_fraction=frac, weight=w),
                                      g[f'lorenz_f{frac}_w{w}'])
    np.testing.assert_array_equal(MO.lorenz_mask(sig, axis=-1, lorenz_fraction=0.7), g['lorenz_axis_t'])
    np.testing.assert_array_equal(MO.lorenz_mask(sig, axis=-2, lorenz_fraction=0.7), g['lorenz_axis_f'])
    np.testing.assert_array_equal(MO.lorenz_mask(g['ties'], lorenz_fraction=0.6), g['lorenz_ties'])
    np.testing.assert_array_equal(MO.lorenz_mask(g['arange33'], weight=1), g['lorenz_arange33'])
    np.testing.assert_array_equal(MO.lorenz_mask(g['arange233'], weight=1), g['lorenz_arange233'])


def test_lorenz_threshold_empty_selection():
    assert MO.lorenz_threshold(np.zeros(5), 0.9) is None                    # 0 / 0: nothing qualifies
    assert MO.lorenz_threshold(np.array([10.0, 0.1, 0.1]), 0.9) is None      # the largest value holds > 90 %
    assert MO.lorenz_threshold(np.array([1.0, 1.0, 1.0, 1.0]), 0.5) == 1.0   # ties: the first of the group qualifies


def test_quantile_order_statistics_match_reference(g):
    sig = g['sig']
    np.testing.assert_array_equal(MO.quantile_mask(sig), g['quantile'])
    np.testing.assert_array_equal(MO.quantile_mask(sig, axis=(-2, -1)), g['quantile_ft'])
    np.testing.assert_array_equal(MO.quantile_mask(sig, 0.3, axis=-1, weight=0.5), g['quantile_t_03'])
    np.testing.assert_array_equal(MO.quantile_mask(sig, -0.25), g['quantile_neg'])
    np.testing.assert_array_equal(MO.quantile_mask(sig.astype(np.complex64)), g['quantile_c64'])
    np.testing.assert_array_equal(MO.quantile_mask(g['ties'], (0.5, -0.5, 0.0, 1.0)), g['quantile_f32'])


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
@pytest.mark.parametrize('n', [1, 2, 7, 12, 513, 4097])
def test_percentile_from_order_statistics_is_bitwise_numpy(dtype, n):
    """The rule the device uses -- q, the virtual index (n - 1) q and gamma in the dtype of the values, then NumPy's
    _lerp in that dtype -- reproduces np.percentile bit for bit, float32 included."""
    rng = np.random.RandomState(n)
    rows = np.abs(rng.randn(6, n)).astype(dtype)
    for quantile in (0.1, -0.9, 0.0, 1.0, -1.0, 0.3, -0.25, 0.5, 0.999, 1 / 3):
        pct = (1 - quantile) * 100 if quantile >= 0 else abs(quantile) * 100
        ref = np.percentile(rows, pct, axis=-1)
        got = MO.percentile_rows(rows, pct)
        assert ref.dtype == got.dtype == dtype
        np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_device_percentile_terms_match_oracle(dtype):
    from pb_bss_b200.extraction.mask_module import _percentile_terms
    for n in (1, 2, 9, 12, 513, 256500):
        for pct in (90.00000000000001, 90.0, 10.0, 0.0, 100.0, 75.0, 25.0, 70.0, 33.3):
            lo, hi, gam, omg = _percentile_terms(n, pct, dtype)
            olo, ohi, ogam, oomg = MO.percentile_terms(n, pct, dtype)
            assert (lo, hi) == (olo, ohi)
            if lo != hi:
                assert gam == float(ogam) and omg == float(oomg)
