"""The oracle-mask kernels (csrc/mask.cuh) over their whole domain against exact oracles.

quantile_mask: bit for bit against np.percentile written out as the reference uses it, at every tile edge of the
short-row path and on the long-row path, with data built against the radix select's digits.  lorenz_mask: against
the exact Lorenz threshold of oracle/mask_oracle.py, allowed to differ only where a float evaluation in some summation
order can.  The source masks: bit for bit against a float64 restatement summing in the kernel's order, with |s|
correctly rounded (oracle exact_hypot); phase_sensitive_mask within a bound from CUDA's documented ulp limits.  The
cases run through the public functions, most of them on NumPy input, on CUDA tensors and on transposed CUDA views.
"""
import math

import numpy as np
import pytest
import torch

from oracle import mask_oracle as MO
from pb_bss_b200 import extraction as E
from pb_bss_b200.extraction import beamform_utils as BU

pytestmark = pytest.mark.gpu

DTYPES = [np.complex128, np.complex64, np.float64, np.float32]
REAL = {np.complex128: np.float64, np.complex64: np.float32, np.float64: np.float64, np.float32: np.float32}


def inputs(sig):
    """The signal as NumPy input, as a CUDA tensor and as a transposed (non-contiguous) CUDA view of the same values."""
    yield sig
    yield torch.from_numpy(np.ascontiguousarray(sig)).cuda()
    if sig.ndim >= 2:
        v = torch.from_numpy(np.ascontiguousarray(np.swapaxes(sig, 0, -1))).cuda().transpose(0, -1)
        assert not v.is_contiguous() or 1 in sig.shape
        yield v


def host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def dev(fn, sig, **kw):
    """fn on every form of inputs(sig); the results agree bit for bit.  -> the NumPy result."""
    got = None
    for x in inputs(sig):
        r = host(fn(x, **kw))
        if got is None:
            got = r
        else:
            np.testing.assert_array_equal(r, got)
    return got


# ---- quantile ------------------------------------------------------------------------------------------------------

def ref_quantile(mag, quantile, axis, weight=0.999):
    """The reference's quantile_mask on |signal| = mag, written out: rows over `axis`, np.percentile per row, strict
    comparison, 0.5 + weight (mask - 0.5) in the dtype of mag."""
    axes = axis if isinstance(axis, tuple) else (axis,)
    last = tuple(-1 - i for i in range(len(axes)))
    moved = np.moveaxis(mag, axes, last)
    rows = moved.reshape(-1, int(np.prod(moved.shape[moved.ndim - len(axes):])))
    pct = (1 - quantile) * 100 if quantile >= 0 else abs(quantile) * 100
    with np.errstate(invalid='ignore'):
        thr = np.percentile(rows, pct, axis=-1)[:, None]
        hit = rows > thr if quantile >= 0 else rows < thr
    m = 0.5 + weight * (hit.astype(rows.dtype) - 0.5)
    return np.moveaxis(m.reshape(moved.shape), last, axes)


def short_tile_rows(n):
    R = 1
    while R * 2 <= 32 and R * 2 * n <= 8192:
        R *= 2
    return R


PATTERNS = ['gauss', 'low_byte', 'top_byte', 'equal', 'two_value', 'edges', 'inf_one', 'inf_some', 'inf_all']


def magnitudes(kind, rows, n, rng, f32):
    """(rows, n) non-negative values, exact in float32 if f32, built against the digits of the radix select."""
    ft, it, nbits = (np.float32, np.uint32, 32) if f32 else (np.float64, np.uint64, 64)
    top_shift = it(nbits - 8)
    if kind == 'gauss':
        return np.abs(rng.standard_normal((rows, n))).astype(ft)
    if kind == 'low_byte':      # the top 7 bytes shared: every digit decides
        base = np.abs(rng.standard_normal((rows, 1))).astype(ft).view(it) & ~it(0xff)
        return (base | rng.integers(0, 256, (rows, n)).astype(it)).view(ft)
    if kind == 'top_byte':      # only the top byte differs
        low = it(0x012345) if f32 else it(0x0123456789abcd)
        return ((rng.integers(0, 0x7f, (rows, n)).astype(it) << top_shift) | low).view(ft)
    if kind == 'equal':
        return np.full((rows, n), 0.75, ft)
    if kind == 'two_value':     # a tie block straddling the selected ranks
        m = np.full((rows, n), 2.0, ft)
        for r in range(rows):
            m[r, :rng.integers(0, n + 1)] = 3.0
            rng.shuffle(m[r])
        return m
    fin = np.finfo(ft)
    if kind == 'edges':
        choice = np.array([0.0, fin.smallest_subnormal, fin.tiny, fin.max, 1.0, 2.5, fin.eps], ft)
        return choice[rng.integers(0, len(choice), (rows, n))]
    m = np.abs(rng.standard_normal((rows, n))).astype(ft)
    if kind == 'inf_one':
        m[np.arange(rows), rng.integers(0, n, rows)] = np.inf
    elif kind == 'inf_some':
        m[rng.random((rows, n)) < 0.3] = np.inf
    elif kind == 'inf_all':
        m[:] = np.inf
    return m


def signal_of(mag, dtype, rng):
    """A signal of the given dtype whose |s| is exactly mag: a random sign, and for complex dtypes the value in the
    real or the imaginary part with the other part zero."""
    sign = np.where(rng.random(mag.shape) < 0.5, -1, 1).astype(mag.dtype)
    v = mag * sign
    if np.issubdtype(dtype, np.complexfloating):
        im = rng.random(mag.shape) < 0.5
        s = np.zeros(mag.shape, dtype)
        s.real = np.where(im, 0, v)
        s.imag = np.where(im, v, 0)
        return s
    return v.astype(dtype)


def quantiles_for(n):
    """Percents 0 and 100, gamma = 0 at an interior index, gamma = 0.5 exactly, and gamma just below and above 0.5,
    both signs.  The gamma each one gives on the host (float64 terms) is asserted: +-0.5 is percent 50, which is
    integral for odd n and exactly half way for even n; +-0.25 / +-0.75 are integral when 4 divides n - 1."""
    qs = [0.0, 1.0, -1.0, 0.1, -0.9, 0.5, -0.5]
    g50 = MO.percentile_terms(n, 50.0, np.float64)[2]
    assert g50 == (0.5 if n % 2 == 0 else 0.0) or n == 1
    if n > 1 and (n - 1) % 4 == 0:
        qs += [0.25, -0.25, 0.75, -0.75]
        assert MO.percentile_terms(n, 25.0, np.float64)[2] == 0 == MO.percentile_terms(n, 75.0, np.float64)[2]
    if n >= 3:
        k = (n - 1) // 3
        for d in (-1e-6, 1e-6):
            p = (k + 0.5 + d) / (n - 1)
            qs += [1 - p, -p]
            g = MO.percentile_terms(n, p * 100, np.float64)[2]
            assert (g < 0.5) if d < 0 else (g > 0.5), (n, d, g)
    return qs


def check_quantile(sig, mag, axis, quantiles, weight=0.999):
    for q in quantiles:
        got = dev(E.quantile_mask, sig, quantile=q, axis=axis, weight=weight)
        ref = ref_quantile(mag, q, axis, weight)
        assert got.dtype == ref.dtype
        np.testing.assert_array_equal(got, ref, err_msg=f'quantile={q} axis={axis} shape={sig.shape}')


SHORT_N = [1, 2, 3, 31, 32, 33, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096]


@pytest.mark.parametrize('n', SHORT_N)
def test_quantile_short_rows_every_tile_edge(n):
    """Row lengths on both sides of every change of the tile height R, R - 1 / R / R + 1 rows (and 1), rows along
    the last axis and rows along axis -2 of a C-contiguous array (the row-fastest walk)."""
    R = short_tile_rows(n)
    rng = np.random.default_rng(n)
    for count in sorted({1, max(R - 1, 1), R, R + 1}):
        for dtype in DTYPES:
            kind = PATTERNS[(count + n + DTYPES.index(dtype)) % len(PATTERNS)]
            mag = magnitudes(kind, count, n, rng, REAL[dtype] == np.float32)
            sig = signal_of(mag, dtype, rng)
            qs = quantiles_for(n)
            check_quantile(sig, mag, -1, qs)
            check_quantile(np.ascontiguousarray(sig.T), np.ascontiguousarray(mag.T), -2, qs)


@pytest.mark.parametrize('kind', PATTERNS)
@pytest.mark.parametrize('dtype', DTYPES)
def test_quantile_digit_patterns(kind, dtype):
    rng = np.random.default_rng(PATTERNS.index(kind))
    for n, count in ((257, 33), (513, 16), (4096, 3), (4097, 3)):
        mag = magnitudes(kind, count, n, rng, REAL[dtype] == np.float32)
        sig = signal_of(mag, dtype, rng)
        check_quantile(sig, mag, -1, quantiles_for(n))


@pytest.mark.parametrize('n,counts', [(4097, [1, 2, 263, 264, 265]), (8192, [1, 3]), (65537, [1, 15, 16, 17]),
                                      (1 << 20, [1, 2]), (1 << 22, [1])])
def test_quantile_long_rows(n, counts):
    """The multi-CTA path: CTAs per row = min(ceil(264 / rows), ceil(n / 4096)), on both sides of one CTA per row and
    of the chunk cap."""
    rng = np.random.default_rng(n)
    for i, count in enumerate(counts):
        dtype = DTYPES[i % 4]
        kind = ['gauss', 'low_byte', 'two_value', 'top_byte', 'edges'][i % 5]
        mag = magnitudes(kind, count, n, rng, REAL[dtype] == np.float32)
        sig = signal_of(mag, dtype, rng)
        qs = [0.1, -0.9, 0.0, 1.0] if n > 65537 else quantiles_for(n)
        check_quantile(sig, mag, -1, qs)
        if count > 1 and n <= 65537:
            check_quantile(np.ascontiguousarray(sig.T), np.ascontiguousarray(mag.T), -2, qs[:3])


@pytest.mark.parametrize('dtype', DTYPES)
def test_quantile_layouts_random_complex_and_negative(dtype):
    """Two-axis rows, leading dims, rows along an inner axis; random complex data (|s| correctly rounded: the oracle's
    exact hypot, rounded to float for complex64) and negative real values."""
    rng = np.random.default_rng(3)
    shape = (2, 3, 40, 23)
    if np.issubdtype(dtype, np.complexfloating):
        sig = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)
        hyp = np.frompyfunc(MO.exact_hypot, 2, 1)
        mag = hyp(sig.real.astype(np.float64), sig.imag.astype(np.float64)).astype(np.float64).astype(REAL[dtype])
    else:
        sig = rng.standard_normal(shape).astype(dtype)
        mag = np.abs(sig)
    for axis in (-2, -1, (-2, -1), 1, (1, 3), 0):
        check_quantile(sig, mag, axis, [0.1, -0.9, 0.3, 0.0, 1.0])


@pytest.mark.parametrize('n', [5, 513, 4096, 4097, 70000])
@pytest.mark.parametrize('dtype', DTYPES)
def test_quantile_nan_row_gives_mask_low(n, dtype):
    """np.percentile of a row holding a NaN is NaN, so the reference's mask is mask_low over the whole row (> nan and
    < nan are false); the other rows are untouched.  Both paths, every dtype."""
    rng = np.random.default_rng(n)
    mag = np.abs(rng.standard_normal((4, n))).astype(REAL[dtype])
    mag[1, rng.integers(n)] = np.nan
    mag[3, :] = np.nan
    sig = signal_of(mag, dtype, rng)
    for q in (0.1, -0.9, 0.0, 1.0):
        got = dev(E.quantile_mask, sig, quantile=q, axis=-1)
        ref = ref_quantile(mag, q, -1)
        np.testing.assert_array_equal(got, ref)
        lo = 0.5 + 0.999 * (REAL[dtype](0) - 0.5)
        assert (got[1] == lo).all() and (got[3] == lo).all()


# ---- Lorenz ----------------------------------------------------------------------------------------------------------

def check_lorenz(sig, fraction, axis=(-2, -1), sensor_axis=None, integer=False):
    """Device Lorenz mask (weight 1, keepdims) against the exact oracle row by row: equal except at powers in
    (t_lo, t_hi]; on integer-valued powers bit for bit equal to the reference's get_mask.  A row where nothing
    qualifies in exact arithmetic must raise, naming the first such row; one where something qualifies in every order
    must not."""
    power = MO.kernel_power(sig, sensor_axis)
    rows = MO._rows(power, axis)[0]
    exact = [MO.lorenz_exact(r, fraction) for r in rows]
    first_never = next((i for i, (_, lo, _) in enumerate(exact) if lo is None), None)
    may_fail = [hi is None for _, _, hi in exact]
    kw = dict(sensor_axis=sensor_axis, axis=axis, lorenz_fraction=fraction, weight=1, keepdims=True)
    # each input form separately: the bucket sums are float atomics, so calls may differ where the interval allows
    for x in inputs(sig):
        try:
            got = host(E.lorenz_mask(x, **kw))
        except ValueError as err:
            row = int(str(err).split('row ')[1].split(' ')[0])
            assert may_fail[row] and (first_never is None or row <= first_never), (row, first_never)
            assert not any(lo is None for _, lo, _ in exact[:row]), row
            continue
        assert first_never is None, first_never
        check_lorenz_rows(MO._rows(got, axis)[0], rows, exact, fraction, integer)


def check_lorenz_rows(g, rows, exact, fraction, integer):
    for i, (r, (t, lo, hi)) in enumerate(zip(rows, exact)):
        want = r > t if t is not None else np.zeros_like(r, bool)
        diff = (g[i] == 1) != want
        allowed = (r > lo) & ((r <= hi) if hi is not None else True)
        assert not (diff & ~allowed).any(), (i, r[diff & ~allowed][:5], t, lo, hi)
        if integer:
            assert (g[i] == 1).tolist() == (r > MO.reference_lorenz_threshold(r, fraction)).tolist(), i


FRACTIONS = [0.98, 0.5, 1e-3, 1 - 1e-12, 1.0, 1.5]


@pytest.mark.parametrize('n', [1, 2, 3, 33, 257, 513, 1025, 2049, 4096, 4097, 8192, 65537])
def test_lorenz_lengths_counts_fractions(n):
    rng = np.random.default_rng(n + 1)
    R = short_tile_rows(n) if n <= 4096 else 264
    counts = sorted({1, max(R - 1, 1), R, R + 1}) if n <= 4097 else [1, 3]   # 4097: both sides of 264 CTAs
    if n == 65537:
        counts = [1, 16, 17]
    for count in counts:
        for j, frac in enumerate(FRACTIONS if count <= 64 else FRACTIONS[:1]):
            dtype = DTYPES[(count + j) % 4]
            shape = (count, n)
            if np.issubdtype(dtype, np.complexfloating):
                sig = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)
            else:
                sig = rng.standard_normal(shape).astype(dtype)
            check_lorenz(sig, frac, axis=-1)
            if count > 1 and j < 2:
                check_lorenz(np.ascontiguousarray(sig.T), frac, axis=-2)


@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_lorenz_integer_powers_bitwise_reference(dtype):
    """Integer-valued powers (every summation order exact): ties at the threshold across bucket boundaries, many
    zeros; bit for bit the reference's get_mask, rows of both paths, several layouts."""
    rng = np.random.default_rng(5)
    for n, count in ((17, 40), (300, 27), (4096, 3), (5000, 3)):
        for vals in ((0, 4), (250, 262), (0, 2 ** 12)):
            sig = rng.integers(vals[0], vals[1], (count, n)).astype(dtype) * np.where(rng.random((count, n)) < .5,
                                                                                        -1, 1).astype(dtype)
            sig[:, :n // 2][rng.random((count, n // 2)) < 0.5] = 0
            for frac in (0.98, 0.5, 0.9, 1.0):
                check_lorenz(sig, frac, axis=-1, integer=True)
        check_lorenz(np.ascontiguousarray(sig.T), 0.7, axis=-2, integer=True)
    sig = rng.integers(0, 30, (3, 4, 18, 19)).astype(dtype)
    for axis in ((-2, -1), -1, 1, (0, 2)):
        check_lorenz(sig, 0.8, axis=axis, integer=True)


@pytest.mark.parametrize('D', [1, 2, 3, 8, 16])
def test_lorenz_sensor_pooling(D):
    """Power summed over the sensors in channel order, any sensor_axis position, against the exact oracle; integer
    powers bit for bit."""
    rng = np.random.default_rng(D)
    base = rng.standard_normal((3, D, 17, 40)) + 1j * rng.standard_normal((3, D, 17, 40))
    for se in range(4):
        sig = np.moveaxis(base, 1, se)
        rows_axes = tuple(a for a in range(4) if a != se)[-2:]
        check_lorenz(sig, 0.9, axis=rows_axes, sensor_axis=se)
        isig = np.round(sig.real * 4)
        check_lorenz(isig, 0.7, axis=rows_axes, sensor_axis=se, integer=True)


@pytest.mark.parametrize('n', [300, 5000])
def test_lorenz_failures_name_the_first_row(n):
    """Dominating values (the largest power alone above the fraction), subnormal powers, all-zero rows, inf and NaN:
    the reference raises (np.min of an empty selection); the device names the first failing row of many, on both
    paths."""
    rng = np.random.default_rng(n)
    sig = rng.standard_normal((40, n))
    sig[17, 3] = 1e6
    sig[29, 0] = 1e7
    check_lorenz(sig, 0.98, axis=-1)
    for bad in (np.inf, np.nan, 0.0):
        s = sig.copy()
        s[17, 3] = 1.0
        s[29, 0] = 1.0
        if bad == 0.0:
            s[11] = 0.0
        else:
            s[11, 5] = bad
            s[35, 1] = bad
        with pytest.raises(ValueError, match='row 11 '):
            E.lorenz_mask(s, axis=-1)
        with pytest.raises(ValueError):
            MO.reference_lorenz_threshold(s[11], 0.98)
    tiny = rng.random((5, n)) * 1e-160                                          # powers below 2^-1022
    check_lorenz(tiny, 0.9, axis=-1)
    check_lorenz(tiny, 1e-9, axis=-1)


# ---- more than 65 535 rows ----------------------------------------------------------------------------------------

def _free_bytes():
    return torch.cuda.mem_get_info()[0]


def test_more_than_65535_long_rows():
    """65 536 rows of 4097 float32 values (the multi-CTA path): each row a rotated permutation of offset + 0..4096, so
    its order statistics, its exact Lorenz threshold (integer powers with sums below 2^53: every order exact) and the
    expected masks follow from the offset alone."""
    if torch.cuda.mem_get_info()[0] < (8 << 30):
        pytest.skip('needs about 8 GB of free device memory (input, mask and selection scratch); the device is shared '
                    'and has less free now')
    rows, n, offsets = 65536, 4097, 300
    gen = torch.Generator(device='cuda')
    gen.manual_seed(0)
    perm = torch.randperm(n, device='cuda', generator=gen)
    r = torch.arange(rows, device='cuda')
    x = (((perm[None, :] + r[:, None]) % n) + ((r % offsets) * n)[:, None]).to(torch.float32)
    one = [np.arange(n, dtype=np.float32) + np.float32(o * n) for o in range(offsets)]
    for q in (0.1, -0.9):
        pct = (1 - q) * 100 if q >= 0 else abs(q) * 100
        thr = torch.tensor([float(np.percentile(v, pct)) for v in one], device='cuda', dtype=torch.float32)
        got = E.quantile_mask(x, quantile=q, axis=-1, weight=1)
        assert got.shape == x.shape
        for c in range(0, rows, 8192):
            xs, t = x[c:c + 8192], thr[r[c:c + 8192] % offsets][:, None]
            assert torch.equal(got[c:c + 8192] == 1, xs > t if q >= 0 else xs < t), (q, c)
        del got
    thr = torch.tensor([MO.reference_lorenz_threshold(v.astype(np.float64) ** 2, 0.98) for v in one], device='cuda',
                       dtype=torch.float64)
    got = E.lorenz_mask(x, axis=-1, weight=1)
    for c in range(0, rows, 8192):
        assert torch.equal(got[c:c + 8192] == 1, x[c:c + 8192].double() ** 2 > thr[r[c:c + 8192] % offsets][:, None]), c


def test_more_than_65535_short_rows():
    rng = np.random.default_rng(9)
    sig = rng.integers(-1000, 1000, (70001, 37)).astype(np.float32)     # integer powers: every order exact
    check_quantile(sig, np.abs(sig), -1, [0.1, -0.9])
    got = E.lorenz_mask(sig, axis=-1, weight=1, lorenz_fraction=0.9)
    np.testing.assert_array_equal(got, MO.lorenz_mask(sig, axis=-1, weight=1, lorenz_fraction=0.9))


# ---- invariants -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [100, 4096, 6000])
def test_batch_independence_and_repeatability(n):
    """A row's mask does not depend on its neighbours or on the call: the same row alone, inside a batch, in another
    position, and twice.  Lorenz bit for bit as well wherever its Lorenz values keep a margin from the fraction larger
    than the atomic-order rounding (random data, fraction 0.9)."""
    rng = np.random.default_rng(n)
    sig = rng.standard_normal((9, n)) + 1j * rng.standard_normal((9, n))
    for fn, kw in ((E.quantile_mask, dict(quantile=0.1, axis=-1)), (E.lorenz_mask, dict(axis=-1, lorenz_fraction=0.9))):
        full = fn(sig, **kw)
        np.testing.assert_array_equal(fn(sig, **kw), full)
        np.testing.assert_array_equal(fn(sig[4:5], **kw), full[4:5])
        np.testing.assert_array_equal(fn(sig[::-1], **kw), full[::-1])


# ---- source masks ---------------------------------------------------------------------------------------------------

_hyp = np.frompyfunc(MO.exact_hypot, 2, 1)


def cr_abs(s):
    s = np.asarray(s, np.complex128)
    return _hyp(s.real, s.imag).astype(np.float64)


def restate_source(name, sig, source_axis, sensor_axis, eps):
    """float64 restatement of a source mask summing in the kernel's order (sources, then sensors, sequentially), with
    |s| correctly rounded; the output dtype of the device."""
    cplx_in = np.iscomplexobj(sig)
    rdt = REAL[sig.dtype.type]
    nd = sig.ndim
    sa, se = source_axis % nd, None if sensor_axis is None else sensor_axis % nd
    if se is None:
        x = np.moveaxis(np.asarray(sig), sa, 0).astype(np.complex128)
    else:
        x = np.moveaxis(np.asarray(sig), (sa, se), (0, 1)).astype(np.complex128)
    K = x.shape[0]
    with np.errstate(all='ignore'):
        if name in ('ideal_binary_mask', 'wiener_like_mask'):
            pw = MO.kernel_power(x, None if se is None else 1)
            if se is not None:
                pw = np.squeeze(pw, 1)
            if name == 'ideal_binary_mask':
                arg = np.argmax(pw, axis=0)                      # the first maximum; the first NaN over anything
                out = (arg[None] == np.arange(K).reshape((K,) + (1,) * (pw.ndim - 1))).astype(np.float64)
            else:
                total = pw[0].copy()
                for k in range(1, K):
                    total = total + pw[k]
                out = pw / (total + eps)
            return np.moveaxis(out, 0, sa if se is None or sa < se else sa - 1).astype(rdt)
        obs = x[0].copy()
        for k in range(1, K):
            obs = obs + x[k]
        mag = cr_abs(x)
        if name == 'ideal_ratio_mask':
            ms = mag[0].copy()
            for k in range(1, K):
                ms = ms + mag[k]
            out = mag / (ms + eps)
        elif name == 'ideal_amplitude_mask':
            out = mag / (cr_abs(obs) + eps)
        elif name == 'ideal_complex_mask':
            out = x / obs if cplx_in else x.real / obs.real
            return np.moveaxis(out, 0, source_axis).astype(sig.dtype if cplx_in else rdt)
        else:
            raise ValueError(name)
        return np.moveaxis(out, 0, source_axis).astype(rdt)


def make_sources(dtype, shape, rng, ties=False):
    if ties:
        v = rng.integers(-2, 3, shape) + 1j * rng.integers(-2, 3, shape)
    else:
        v = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    if not np.issubdtype(dtype, np.complexfloating):
        v = v.real
    return v.astype(dtype)


BITWISE = ['ideal_binary_mask', 'wiener_like_mask', 'ideal_ratio_mask', 'ideal_amplitude_mask', 'ideal_complex_mask']


@pytest.mark.parametrize('K', [1, 2, 3, 7, 8, 9, 17, 40])
@pytest.mark.parametrize('dtype', DTYPES)
def test_source_masks_bitwise_restatement(K, dtype):
    """Every source axis position, eps in {0, default, 1}, exact ties (first argmax) and zero observations (NumPy's
    inf / nan), bit for bit."""
    rng = np.random.default_rng(K)
    for ties in (False, True):
        base = make_sources(dtype, (K, 5, 6), rng, ties)
        if ties and K >= 2:
            base[1, 0] = -base[0, 0] if K == 2 else base[1, 0]             # a zero observation when K = 2
        for sa in range(3):
            sig = np.moveaxis(base, 0, sa)
            for name in BITWISE:
                for eps in ((None,) if name in ('ideal_binary_mask', 'ideal_complex_mask') else (0.0, None, 1.0)):
                    kw = dict(source_axis=sa) if eps is None else dict(source_axis=sa, eps=eps)
                    with np.errstate(all='ignore'):
                        got = dev(getattr(E, name), sig, **kw)
                    want = restate_source(name, sig, sa, None, 1e-18 if eps is None else eps)
                    assert got.dtype == want.dtype, (name, got.dtype, want.dtype)
                    np.testing.assert_array_equal(got, want, err_msg=f'{name} K={K} sa={sa} eps={eps}')


@pytest.mark.parametrize('D', [1, 2, 5, 16])
def test_binary_and_wiener_sensor_pooling_bitwise(D):
    rng = np.random.default_rng(D)
    for dtype in DTYPES:
        for K in (1, 2, 9):
            base = make_sources(dtype, (K, D, 4, 7), rng, ties=D == 2)
            for sa, se in ((0, 1), (1, 0), (0, 3), (3, 2), (2, 0)):
                sig = np.moveaxis(base, (0, 1), (sa, se))
                for name in ('ideal_binary_mask', 'wiener_like_mask'):
                    got = dev(getattr(E, name), sig, source_axis=sa, sensor_axis=se)
                    want = restate_source(name, sig, sa, se, 1e-18)
                    np.testing.assert_array_equal(got, want, err_msg=f'{name} D={D} K={K} sa={sa} se={se}')


SPECIAL = [0.0, 5e-324, -5e-324, 1e300, -1e300, np.inf, -np.inf, np.nan, 1.5 * 2.0 ** 1000, -1.5 * 2.0 ** -1000,
           2.0 ** 1001, 2.0 ** -1001, 1.0, 3.0]


def test_source_masks_special_components():
    """Every (re, im) combination of {0, +-subnormal, +-1e300, +-inf, NaN, 2^+-1000 edges} for two sources: |s| as C's
    hypot gives it correctly rounded (an infinite part gives inf even next to a NaN), bit for bit."""
    comps = np.array([complex(a, b) for a in SPECIAL for b in SPECIAL])
    s0 = np.repeat(comps, len(comps))
    s1 = np.tile(comps, len(comps))
    sig = np.stack([s0, s1])
    for name in BITWISE:
        with np.errstate(all='ignore'):
            got = getattr(E, name)(sig)
            want = restate_source(name, sig, 0, None, 1e-18)
        np.testing.assert_array_equal(got, want, err_msg=name)
    # one source: |s| / (|s| + 0) is 1, or NaN for a zero, infinite or NaN |s|
    mag = cr_abs(comps)
    with np.errstate(all='ignore'):
        got = E.ideal_ratio_mask(comps[None], eps=0.0)
        want = mag / mag
    np.testing.assert_array_equal(got[0], want)


def test_abs_correctly_rounded_except_near_midpoints():
    """The device's |s| read exactly through the quantile mask: the row [s, lo, hi] with lo / hi the doubles next to
    the correctly rounded c = |s| has median |s| iff |s| = c, and the masks |x| < median and |x| > median tell which of
    lo, c, hi the device produced.  Inputs over the whole exponent range (subnormal, 2^+-1000 edges, huge) and exact
    Pythagorean midpoints; |s| must be c, or the other neighbour of a midpoint the exact value lies within 2^-48 ulp
    of."""
    rng = np.random.default_rng(12)
    e = rng.integers(-1074, 1022, size=(3000, 1))
    d = rng.integers(-30, 31, size=(3000, 1))
    ex = np.concatenate([e, np.clip(e + d, -1074, 1021)], 1)
    v = np.ldexp(rng.uniform(1, 2, size=(3000, 2)), ex) * rng.choice([-1, 1], size=(3000, 2))
    mids = []
    p = 2 ** 26 + 1235
    while len(mids) < 40:                       # (2pq, p^2 - q^2): odd 54-bit hypotenuse p^2 + q^2
        q = p - 2 ** 24 - 7
        m = p * p + q * q
        if m % 2 == 1 and 2 ** 53 <= m < 2 ** 54:
            s = 2.0 ** int(rng.integers(-1000, 900))
            mids.append((float(2 * p * q) * s, float(p * p - q * q) * s))
        p += 1
    # the overflow edge: |s| rounds to DBL_MAX below DBL_MAX + ulp / 2 and to inf from there on; with a = DBL_MAX
    # that edge is at b = sqrt(2^971 a)
    dmax = np.finfo(np.float64).max
    b_edge = float(math.isqrt(int(dmax) << 971))
    over = [[dmax, dmax], [dmax, 1.0], [1.5 * 2.0 ** 1023, 1.5 * 2.0 ** 1023], [dmax, b_edge],
            [dmax, b_edge * (1 - 2.0 ** -40)], [dmax, b_edge * (1 + 2.0 ** -40)], [np.nextafter(dmax, 0), b_edge],
            [-dmax, -2.0 ** 1000], [2.0 ** 1023, 2.0 ** 1023]]
    v = np.concatenate([v, np.array(mids), over, [[2.0 ** -1074 * 3, 2.0 ** -1074 * 4], [5e-324, 5e-324],
                                                  [2.0 ** 1000 * 1.5, 2.0 ** 999], [1e-310, 2e-310]]])
    c = np.array([MO.exact_hypot(a, b) for a, b in v])
    assert np.isinf(c).sum() >= 3 and (c == dmax).sum() >= 2        # both sides of the overflow edge are reached
    # |s| = inf or finite: the ratio mask of s alone with eps = 0 is |s| / |s|, NaN for inf and 1 for any finite |s|
    # (the median read below would interpolate inf - inf = NaN, as np.percentile does).  The two may differ only where
    # the exact value is within 2^-48 ulp of DBL_MAX + ulp / 2, the midpoint to 2^1024.
    inf = np.isinf(c)
    ratio = dev(E.ideal_ratio_mask, (v[:, 0] + 1j * v[:, 1])[None], eps=0.0)[0]
    dev_inf = np.isnan(ratio)
    assert (ratio[~dev_inf] == 1).all()
    for k in np.flatnonzero(dev_inf != inf):
        assert MO.hypot_near_midpoint(v[k, 0], v[k, 1], dmax, 2 ** 1024, 2.0 ** -48), v[k]
    keep = ~inf & ~dev_inf
    v, c = v[keep], c[keep]
    # c = DBL_MAX has no finite upper neighbour (an inf in the row would make the median inf - inf = NaN): there the
    # row is [s, lo, c], whose median is c if |s| = c (nothing above it) and lo if |s| = lo; |s| = inf is read above
    top = c == dmax
    lo, hi = np.nextafter(c, 0), np.where(top, c, np.nextafter(np.where(top, 0, c), np.inf))
    row = np.stack([v[:, 0] + 1j * v[:, 1], lo + 0j, hi + 0j], 1)
    below = dev(E.quantile_mask, row, quantile=-0.5, axis=-1, weight=1) == 1     # percent 50: k = 1, gamma = 0
    above = dev(E.quantile_mask, row, quantile=0.5, axis=-1, weight=1) == 1
    FFF, FTF, FFT = [False, False, False], [False, True, False], [False, False, True]
    is_c = np.where(top, (below == FTF).all(1) & (above == FFF).all(1), (below == FTF).all(1) & (above == FFT).all(1))
    is_lo = (below == FFF).all(1) & (above == FFT).all(1)
    is_hi = ~top & (below == FTF).all(1) & (above == FFF).all(1)
    off = np.flatnonzero(~is_c)
    print('device |s| differs from the correctly rounded value at %d of %d inputs' % (len(off), len(v)))
    for k in off:
        a, b = v[k]
        assert is_lo[k] or is_hi[k], (a, b, below[k], above[k])
        assert MO.hypot_near_midpoint(a, b, c[k], lo[k] if is_lo[k] else hi[k], 2.0 ** -48), (a, b)


def test_phase_sensitive_mask_within_cuda_ulp_bound():
    """|s| / (|o| + eps) cos(angle(s) - angle(o)): atan2 and cos have at most 2 ulp error each (CUDA C Programming
    Guide, double-precision mathematical functions); the angle difference carries 2 + 2 ulp of the angles (<= pi,
    ulp 2^-51) plus half an ulp of its own rounding (|theta| <= 2 pi, ulp 2^-50), and cos' = -sin, so with
    r = |s| / (|o| + eps): |got - exact| <= r (|sin theta| 5 2^-51 + 2 ulp(cos theta)) + 3 u |got|.  Exact by mpmath
    at 60 digits."""
    import mpmath
    mpmath.mp.dps = 60
    rng = np.random.default_rng(4)
    for K in (1, 2, 3, 9, 40):
        for dtype in (np.complex128, np.complex64):
            sig = make_sources(dtype, (K, 3, 11), rng)
            got = dev(E.phase_sensitive_mask, sig)
            x = sig.astype(np.complex128)
            obs = x[0].copy()
            for k in range(1, K):
                obs = obs + x[k]
            om = cr_abs(obs)
            for idx in np.ndindex(x.shape):
                s, o = x[idx], obs[idx[1:]]
                r = MO.exact_hypot(s.real, s.imag) / (om[idx[1:]] + 1e-18)
                th = mpmath.atan2(s.imag, s.real) - mpmath.atan2(o.imag, o.real)
                exact = float(mpmath.mpf(MO.exact_hypot(s.real, s.imag)) / (mpmath.mpf(om[idx[1:]]) + mpmath.mpf(
                    1e-18)) * mpmath.cos(th))
                bound = r * (abs(math.sin(float(th))) * 5 * 2.0 ** -51 + 2 * 2.0 ** -52) + 3 * 2.0 ** -53 * abs(exact)
                if dtype == np.complex64:
                    bound += np.spacing(np.float32(abs(exact)))
                assert abs(float(got[idx]) - exact) <= bound, (K, idx, got[idx], exact)


# ---- source masks against the reference expression evaluated by NumPy -------------------------------------------

U = 2.0 ** -53


def numpy_reference(name, sig, source_axis, eps):
    """The reference's expressions for float64 / complex128 input, evaluated by NumPy itself (np.sum, np.abs,
    np.argmax, complex division)."""
    with np.errstate(all='ignore'):
        power = sig.real ** 2 + sig.imag ** 2 if np.iscomplexobj(sig) else sig ** 2
        if name == 'ideal_binary_mask':
            K = sig.shape[source_axis]
            shape = [1] * sig.ndim
            shape[source_axis] = K
            return (np.expand_dims(np.argmax(power, axis=source_axis), source_axis) ==
                    np.arange(K).reshape(shape)).astype(np.float64)
        if name == 'wiener_like_mask':
            return power / (power.sum(source_axis, keepdims=True) + eps)
        if name == 'ideal_ratio_mask':
            a = np.abs(sig)
            return a / (a.sum(source_axis, keepdims=True) + eps)
        if name == 'ideal_amplitude_mask':
            return np.abs(sig) / (np.abs(np.sum(sig, source_axis, keepdims=True)) + eps)
        return sig / np.sum(sig, axis=source_axis, keepdims=True)


@pytest.mark.parametrize('K', [1, 2, 5, 7, 8, 13, 40])
def test_source_masks_against_numpy_reference_expression(K):
    """NumPy's np.sum adds sequentially along a non-innermost axis; along the innermost axis its reduction adds the
    first term to a separate (pairwise from 8 terms on) sum of the others, whatever K.  Where it is sequential the
    device equals the reference expression bit for bit
    (real input for the masks that take |s|: NumPy's complex abs is not correctly rounded, see test_mask_oracle);
    elsewhere each of the two sums of K terms is within (K - 1) u S of the exact one (S the sum of the magnitudes),
    so with o the observation and NumPy's |s| within 2 ulp = 4 u:
      wiener (non-negative terms):  |got - ref| <= 4 (K - 1) u |ref| + 2 ulp(ref),
      ratio:                        |got - ref| <= (4 (K - 1) + 16) u |ref| + 2 ulp(ref),
      amplitude:                    |got - ref| <= 2 |ref| (2 (K - 1) u S / |o| + 8 u) + 2 ulp(ref),
      complex:                      |got - ref| <= |s| 2 (K - 1) u S / |o|^2 + 4 u |ref|."""
    rng = np.random.default_rng(K + 100)
    for dtype in (np.complex128, np.float64):
        base = make_sources(dtype, (K, 6, 9), rng)
        for sa in range(3):
            sig = np.ascontiguousarray(np.moveaxis(base, 0, sa))
            sequential = sa != 2
            for name in BITWISE:
                got = getattr(E, name)(sig, source_axis=sa)
                ref = numpy_reference(name, sig, sa, 1e-18)
                if name == 'ideal_complex_mask' and dtype == np.float64:
                    ref = ref.real
                takes_abs = name in ('ideal_ratio_mask', 'ideal_amplitude_mask')
                if sequential and not (takes_abs and dtype == np.complex128):
                    np.testing.assert_array_equal(got, ref, err_msg=f'{name} K={K} sa={sa} {dtype}')
                    continue
                if name == 'ideal_binary_mask':
                    continue                            # argmax of pairwise sums: no bound, checked where sequential
                mag = np.abs(sig)
                S = mag.sum(sa, keepdims=True)
                o = np.abs(np.sum(sig, axis=sa, keepdims=True))
                if name == 'ideal_complex_mask':
                    bound = mag * 2 * (K - 1) * U * S / o ** 2 + 4 * U * np.abs(ref)
                elif name == 'ideal_amplitude_mask':
                    bound = np.abs(ref) * (2 * (K - 1) * U * S / o + 8 * U) * 2 + 2 * np.spacing(np.abs(ref))
                elif name == 'wiener_like_mask':
                    bound = 4 * (K - 1) * U * np.abs(ref) + 2 * np.spacing(np.abs(ref))
                else:
                    bound = (4 * (K - 1) * U + 16 * U) * np.abs(ref) + 2 * np.spacing(np.abs(ref))
                assert (np.abs(got - ref) <= bound).all(), (name, K, sa, dtype, np.abs(got - ref).max())


# ---- biased binary mask and the array geometry ---------------------------------------------------------------------

def restate_biased_binary(sig, low_cut=5, high_cut=500):
    """The reference's decisions in fp64 for a (2, ..., F) signal: power = re^2 + im^2, thresholds 10^(dB / 10) of the
    voiced / unvoiced weighting over the last axis, strict comparisons, the 0.005 floors and the forced cut bins."""
    F = sig.shape[-1]
    v, u = E.voiced_unvoiced_split_characteristic(F)
    ts_db, tn_db = 0 * v + 5 * u, -10 * v + -10 * u
    x = sig.astype(np.complex128)
    p = x.real * x.real + x.imag * x.imag
    ps, pn = p[:1], p[1:]
    a, b = ps / 10 ** (ts_db / 10), ps / 10 ** (tn_db / 10)
    speech = (a > pn) & (a > 0.005)
    noise = (b < pn) | (b < 0.005)
    speech[..., 0:low_cut - 1] = False
    speech[..., high_cut:speech.shape[1] if speech.ndim > 1 else F] = False
    noise[..., 0:low_cut - 1] = True
    noise[..., high_cut:noise.shape[1] if noise.ndim > 1 else F] = True
    return np.concatenate([speech, noise], 0)


@pytest.mark.parametrize('F', [12, 64, 257, 513, 600])     # F >= 10: the voiced / unvoiced ramp needs width 2
def test_biased_binary_mask_decisions(F):
    """Exact decisions against the restatement, every dtype, including powers placed exactly on the thresholds
    (a decision that rounds the other way would show) and the cut bins forced at both ends."""
    rng = np.random.default_rng(F)
    for dtype in DTYPES:
        sig = make_sources(dtype, (2, 3, F), rng) * 0.3
        sig[:, 0] = 0                                                 # zero powers: the 0.005 floors decide
        sig[0, 1] = 1.0
        sig[1, 1] = np.sqrt(0.5)                                      # power 0.5 against the thresholds
        for lc, hc in ((5, 500), (1, F), (3, max(F // 2, 1)), (0, 2)):
            got = dev(E.biased_binary_mask, sig, low_cut=lc, high_cut=hc)
            assert got.dtype == np.bool_
            np.testing.assert_array_equal(got, restate_biased_binary(sig, lc, hc), err_msg=f'{dtype} {lc} {hc}')


def _mp():
    import mpmath
    mpmath.mp.dps = 50
    return mpmath


def test_steering_vector_within_cuda_ulp_bound():
    """exp(-2j pi f tdoa): the argument rounded as NumPy and the kernel round it, w = fl(-2 pi f) and fl(w tdoa),
    arguments up to about 300 rad; sin and cos within 2 ulp (CUDA's documented bound for sincos).  Normalised over
    the M sensors: scale 1 / sqrt(sum of cs^2 + sn^2), whose relative error is at most (7 + M / 2) u (each term
    within 9 u of exact, M terms summed, a correctly rounded sqrt and division), so
    |got - c / sqrt(M)| <= 2 ulp(c) / sqrt(M) + |c| / sqrt(M) (7 + M / 2) u + ulp(got)."""
    mp = _mp()
    rng = np.random.default_rng(21)
    for M in (1, 2, 7):
        tdoa = rng.uniform(-0.006, 0.006, (3, M))
        tdoa[0, 0] = 0.0
        freq = np.arange(0, 64 / 2 + 1) * 16000 / 64
        w = -2.0 * np.pi * freq
        for normalize in (False, True):
            got = dev(BU.get_steering_vector, tdoa, stft_size=64, normalize=normalize)
            assert got.shape == (3, M, 33) and got.dtype == np.complex128
            for idx in np.ndindex(got.shape):
                arg = w[idx[2]] * tdoa[idx[:2]]                      # both products rounded, as in the kernel
                c, s_ = mp.cos(arg), mp.sin(arg)
                for g, e in ((got[idx].real, c), (got[idx].imag, s_)):
                    e = float(e)
                    if not normalize:
                        assert abs(g - e) <= 2 * np.spacing(abs(e)), (idx, g, e)
                    else:
                        r = math.sqrt(M)
                        bound = 2 * np.spacing(abs(e)) / r + abs(e) / r * (7 + M / 2) * U + np.spacing(abs(g))
                        assert abs(g - e / r) <= bound, (idx, g, e / r)
    assert abs(float(np.abs(BU.get_steering_vector(np.array([0.0]), stft_size=64)).max()) - 1) == 0


def test_diffuse_noise_psd_within_cuda_ulp_bound():
    """np.sinc(2 f d / c) with x = fl(fl(fl(2 f) d) / c) and y = fl(pi x) as NumPy and the kernel round them,
    arguments up to about 300 rad: sin within 2 ulp and a correctly rounded division, so
    |got - sin(y) / y| <= 2 ulp(sin y) / |y| + ulp(got); x = 0 gives 1 exactly."""
    mp = _mp()
    rng = np.random.default_rng(22)
    d = rng.uniform(0, 6.5, (5, 5))
    d = (d + d.T) / 2
    np.fill_diagonal(d, 0)
    got = dev(BU.get_diffuse_noise_psd, d, fft_size=64)
    assert got.shape == (33, 5, 5)
    freq = np.arange(0, 64 / 2 + 1) * 16000 / 64
    for f, i, j in np.ndindex(got.shape):
        x = 2.0 * freq[f] * d[i, j] / 343
        if x == 0:
            assert got[f, i, j] == 1.0
            continue
        y = np.pi * x
        e = float(mp.sin(y) / y)
        bound = 2 * np.spacing(abs(float(mp.sin(y)))) / abs(y) + np.spacing(abs(got[f, i, j]))
        assert abs(got[f, i, j] - e) <= bound, (f, i, j, got[f, i, j], e)


def test_time_of_flight_and_farfield_tdoa():
    """Near field: |source - sensor| / c with the squares summed in coordinate order, a correctly rounded sqrt and
    division: bit for bit the reference's np.linalg.norm expression (it sums the 3 coordinates in the same order).
    Far field: the direction (-cos(-el) cos(az), -sin(az), sin(-el) cos(az)) from angles up to a few hundred rad, dotted
    with the sensor offsets by FMAs: against mpmath within 2 ulp per sin / cos, one rounding per product and per FMA
    and a correctly rounded division."""
    mp = _mp()
    rng = np.random.default_rng(23)
    src, sen = rng.uniform(-5, 5, (3, 7)), rng.uniform(-0.3, 0.3, (3, 6))
    got = dev(lambda s: BU.get_nearfield_time_of_flight(s, sen), src)
    ref = np.linalg.norm(src[:, :, None] - sen[:, None, :], axis=0) / 343
    np.testing.assert_array_equal(got, ref)
    ang = rng.uniform(-300, 300, (2, 9))
    ang[:, 0] = 0.0
    for refc in (1, 0, 5):
        got = dev(lambda a: BU.get_farfield_time_difference_of_arrival(a, sen, reference_channel=refc), ang)
        assert got.shape == (6, 9)
        for m, k in np.ndindex(got.shape):
            az, el = mp.mpf(ang[0, k]), mp.mpf(ang[1, k])
            u = [-mp.cos(-el) * mp.cos(az), -mp.sin(az), mp.sin(-el) * mp.cos(az)]
            dvec = [sen[i, m] - sen[i, refc] for i in range(3)]           # rounded as the kernel rounds them
            e = float(sum(mp.mpf(dvec[i]) * u[i] for i in range(3)) / 343)
            ca, sa = abs(float(mp.cos(az))), abs(float(mp.sin(az)))
            ce, se = abs(float(mp.cos(el))), abs(float(mp.sin(el)))
            eu = [2 * np.spacing(ce) * ca + 2 * np.spacing(ca) * ce + np.spacing(ce * ca),
                  2 * np.spacing(sa),
                  2 * np.spacing(se) * ca + 2 * np.spacing(ca) * se + np.spacing(se * ca)]
            mag = sum(abs(dvec[i]) * abs(float(u[i])) for i in range(3))
            bound = (sum(abs(dvec[i]) * eu[i] for i in range(3)) + 3 * U * mag) / 343 * 1.01 + np.spacing(abs(e))
            assert abs(got[m, k] - e) <= bound, (m, k, got[m, k], e, bound)
