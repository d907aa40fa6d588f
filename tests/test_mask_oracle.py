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


# ---- exact forms: hypot, NaN-aware percentile, Lorenz threshold and its rounding interval ------------------------

DBL_MAX = np.finfo(np.float64).max
DBL_TRUE_MIN = 5e-324
EDGE_COMPONENTS = [0.0, -0.0, DBL_TRUE_MIN, -DBL_TRUE_MIN, 2.0 ** -1022, 1e-300, -1e-300, 1.0, -1.0, 1e300, -1e300,
                   DBL_MAX, -DBL_MAX, np.inf, -np.inf, np.nan]


def _pythagorean_midpoint():
    """(a, b, m): doubles a, b whose exact hypot m = p^2 + q^2 is an odd 54-bit integer, a midpoint of two doubles."""
    p = 2 ** 26 + 1235
    while True:
        q = p - 2 ** 24 - 7
        m = p * p + q * q
        if m % 2 == 1 and 2 ** 53 <= m < 2 ** 54 and (p - q) % 2 == 1:
            return float(2 * p * q), float(p * p - q * q), m
        p += 1


def test_exact_hypot_special_cases_and_ties():
    assert MO.exact_hypot(3.0, 4.0) == 5.0
    assert MO.exact_hypot(np.nan, np.inf) == np.inf and MO.exact_hypot(-np.inf, np.nan) == np.inf
    assert np.isnan(MO.exact_hypot(np.nan, 1.0)) and np.isnan(MO.exact_hypot(0.0, np.nan))
    assert MO.exact_hypot(DBL_MAX, DBL_MAX) == np.inf
    assert MO.exact_hypot(DBL_TRUE_MIN, DBL_TRUE_MIN) == DBL_TRUE_MIN      # sqrt(2) 2^-1074 -> 1 * 2^-1074
    assert MO.exact_hypot(3 * DBL_TRUE_MIN, 4 * DBL_TRUE_MIN) == 5 * DBL_TRUE_MIN
    a, b, m = _pythagorean_midpoint()
    assert a < 2 ** 53 and b < 2 ** 53 and int(a) ** 2 + int(b) ** 2 == m ** 2
    assert MO.exact_hypot(a, b) == float(m)                                # int -> float rounds ties to even
    for s in (2.0 ** -600, 2.0 ** 500):
        assert MO.exact_hypot(a * s, b * s) == float(m) * s


def _np_abs(re, im):
    with np.errstate(over='ignore', invalid='ignore'):
        return float(np.abs(np.complex128(complex(re, im))))


def test_numpy_abs_against_exact_hypot():
    """np.abs of complex128 (NumPy's own complex-abs loop, not C's hypot) against the correctly rounded value: the
    special cases (zero, infinite and NaN parts) exactly; finite inputs over the whole exponent range are compared and
    the differing ones named."""
    comps = EDGE_COMPONENTS
    finite = []
    for re in comps:
        for im in comps:
            got, exact = _np_abs(re, im), MO.exact_hypot(re, im)
            if np.isfinite(re) and np.isfinite(im) and re != 0 and im != 0:
                finite.append((re, im))
                continue
            assert (np.isnan(got) and np.isnan(exact)) or got == exact, (re, im, got, exact)
    rng = np.random.default_rng(7)
    e = rng.integers(-1074, 1024, size=(4000, 2))
    d = rng.integers(-60, 61, size=4000)
    e[:, 1] = np.clip(e[:, 0] + d, -1074, 1023)                          # half the pairs within 2^60 of each other
    vals = np.ldexp(rng.uniform(1, 2, size=(4000, 2)), e) * rng.choice([-1, 1], size=(4000, 2))
    tested = finite + vals.tolist()
    differ = [(re, im) for re, im in tested if _np_abs(re, im) != MO.exact_hypot(re, im)]
    print('np.abs differs from the correctly rounded |s| at %d of %d inputs: %s' % (len(differ), len(tested),
                                                                                    differ[:10]))
    # NumPy does not promise a correctly rounded complex abs: the finite differences are recorded, not failed; the
    # device's |s| is held to the correctly rounded value (tests/test_mask_kernels_gpu.py)
    assert all(np.isfinite(_np_abs(re, im)) == np.isfinite(MO.exact_hypot(re, im)) for re, im in differ)


RAW_EDGE_ROWS = [
    [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0, 10.0, 11.0, np.nan],
    [np.nan, 0.0, 1.0],
    [np.inf, 1.0, 2.0, 3.0],
    [np.inf, np.inf, 1.0, 0.0],
    [-np.inf, 0.0, np.inf, 5.0],
    [0.0, 5e-324, 1e-310, DBL_MAX, DBL_MAX, 2.0],
    [DBL_MAX, -DBL_MAX, 1.0, 0.0],
    [-3.0, -1.0, 0.0, 2.5, 7.0, -0.5],
]


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_percentile_rows_nan_aware_bitwise_numpy(dtype):
    """percentile_rows against np.percentile itself on rows with NaN, +-inf, +0, subnormals and the largest finite
    value: bit for bit, NaN where the row holds a NaN."""
    with np.errstate(over='ignore'):
        rows = [np.asarray(r, dtype=dtype) for r in RAW_EDGE_ROWS]
    rng = np.random.default_rng(11)
    for n in (1, 2, 5, 12, 513):
        block = rng.standard_normal((4, n)).astype(dtype)
        block[0, rng.integers(n)] = np.nan
        block[1, rng.integers(n)] = np.inf
        block[2, :] = np.finfo(dtype).tiny / 4
        rows += list(block)
    for r in rows:
        for pct in (0.0, 10.0, 50.0, 90.0, 90.00000000000001, 99.9, 100.0, 100.0 / 3):
            with np.errstate(invalid='ignore'):
                ref = np.percentile(r[None], pct, axis=-1)
            got = MO.percentile_rows(r[None], pct)
            assert got.dtype == ref.dtype == dtype
            np.testing.assert_array_equal(got, ref, err_msg=f'{r} {pct}')
            if np.isnan(r).any():
                assert np.isnan(got).all()


def _lorenz_rows(rng):
    for n in (1, 2, 3, 31, 257, 1000, 4097):
        yield rng.random(n)
        yield rng.standard_normal(n) ** 2
        yield np.exp(rng.standard_normal(n) * 8)                               # wide dynamic range
        z = rng.random(n) ** 2
        z[rng.random(n) < 0.7] = 0.0                                          # many zero powers
        yield z
        yield rng.random(n) * 1e-310                                           # subnormal powers
        yield rng.integers(0, 9, n).astype(np.float64)                         # ties
        yield rng.integers(0, 2 ** 20, n).astype(np.float64)


@pytest.mark.parametrize('fraction', [1e-9, 0.1, 0.5, 0.9, 0.98, 1 - 1e-12, 1.0, 1.5])
def test_lorenz_exact_oracle_against_reference_literal(fraction):
    """The reference's own threshold (np.sort / cumsum / sum / min) lies in the oracle's interval; on integer-valued
    powers, where every summation order is exact, it equals the exact threshold.  An empty selection in the reference
    (ValueError) is one the interval allows."""
    rng = np.random.default_rng(int(fraction * 1000))
    for row in _lorenz_rows(rng):
        t, lo, hi = MO.lorenz_exact(row, fraction)
        try:
            ref = MO.reference_lorenz_threshold(row, fraction)
        except ValueError:
            assert hi is None, (row.size, fraction, t, lo, hi)
            continue
        assert lo is not None and lo <= ref and (hi is None or ref <= hi), (row.size, fraction, ref, t, lo, hi)
        if np.array_equal(row, np.round(row)):
            assert ref == t, (row.size, fraction, ref, t)
        if t is not None:
            assert lo <= t and (hi is None or t <= hi)
    for bad in ([1.0, np.inf, 2.0], [np.nan, 1.0], [0.0, 0.0]):
        assert MO.lorenz_exact(bad, 0.9)[0] is None
        with pytest.raises(ValueError):
            MO.reference_lorenz_threshold(np.asarray(bad), 0.9)


def test_lorenz_exact_interval_is_tight_where_sums_are_exact():
    row = np.arange(1, 101, dtype=np.float64)
    t, lo, hi = MO.lorenz_exact(row, 0.5)
    assert t == lo == hi == MO.reference_lorenz_threshold(row, 0.5)
    # a Lorenz value exactly at the fraction does not qualify: 100 / 200 = 0.5
    t, lo, hi = MO.lorenz_exact(np.array([100.0, 50.0, 50.0]), 0.5)
    assert t is None and hi is None and lo == 100.0
