"""NumPy restatement of the selection algorithms behind the device's lorenz_mask and quantile_mask (csrc/mask.cuh).

Lorenz: the reference sorts each row and takes the minimum over the prefix whose cumsum / sum is below the fraction.
Here the threshold is found the way the kernel finds it, without a sort of the row: over the distinct values v in
descending order, v qualifies when (sum of the elements above v + v) / sum < fraction, which is the Lorenz value of
the first element of v's group; the qualifying values form a prefix and the threshold is the smallest of them.

Quantile: np.percentile's linear method from two explicit order statistics, selected with np.partition, and NumPy's
_lerp in the dtype of the values; a row holding a NaN gives NaN, as np.percentile does.  Checked against the
reference's fixture and against np.percentile by tests/test_mask_oracle.py.

Exact forms, for checking the device bit for bit: exact_hypot (|a + ib| correctly rounded, in integers) and
lorenz_exact (the Lorenz threshold from exact rational Lorenz values, with the interval of thresholds that a float
evaluation in any summation order can give).
"""
import bisect
import itertools
import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -53  # unit roundoff of float64


def exact_hypot(re, im):
    """|re + i im| rounded to the nearest double (ties to even), from the exact sum of squares in integers.  C's
    special cases: an infinite part gives +inf even next to a NaN; otherwise a NaN part gives NaN."""
    re, im = float(re), float(im)
    if math.isinf(re) or math.isinf(im):
        return math.inf
    if math.isnan(re) or math.isnan(im):
        return math.nan
    if re == 0.0 and im == 0.0:
        return 0.0
    # a = A / 2^m, b = B / 2^m with a common power-of-two denominator; |s| = sqrt(N) / 2^m, N = A^2 + B^2
    m = 1074
    A, B = ((lambda pq: pq[0] << (m + 1 - pq[1].bit_length()))(abs(v).as_integer_ratio()) for v in (re, im))
    N = A * A + B * B
    e = (N.bit_length() - 1 - 2 * m) // 2           # floor(log2 |s|)
    q = max(e - 52, -1074)                          # exponent of the ulp of the result
    t = m + q                                        # |s| / 2^q = sqrt(N / 4^t)
    num, den = (N, 1 << (2 * t)) if t >= 0 else (N << (-2 * t), 1)
    k = math.isqrt(num // den)                       # floor(sqrt(N / 4^t))
    # round: compare N / 4^t with (k + 1/2)^2, i.e. 4 num with (2k + 1)^2 den
    c = 4 * num - (2 * k + 1) ** 2 * den
    if c > 0 or (c == 0 and k % 2 == 1):
        k += 1
    try:
        return float(Fraction(k) * Fraction(2) ** q)
    except OverflowError:
        return math.inf


def hypot_near_midpoint(re, im, x, y, tol):
    """True if the exact |re + i im| lies within tol ulp of the midpoint of the neighbouring doubles x and y (exact:
    the comparison is made on squares of rationals; x or y may be an int or Fraction, e.g. 2^1024 for the overflow
    edge)."""
    x, y = (v if isinstance(v, (int, Fraction)) else Fraction(float(v)) for v in (x, y))
    mid, d = (x + y) / 2, Fraction(tol) * abs(y - x)
    s = Fraction(float(re)) ** 2 + Fraction(float(im)) ** 2
    return max(mid - d, 0) ** 2 <= s <= (mid + d) ** 2


def lorenz_threshold(row, fraction):
    """-> threshold of one row of non-negative powers, or None if no value qualifies."""
    row = np.asarray(row, dtype=np.float64).ravel()
    values, counts = np.unique(row, return_counts=True)
    values, counts = values[::-1], counts[::-1]
    total = row.sum()
    above = np.concatenate(([0.0], np.cumsum(values * counts)[:-1]))
    with np.errstate(invalid='ignore', divide='ignore'):
        qualifies = (above + values) / total < fraction
    if not qualifies.any():
        return None
    return values[np.flatnonzero(qualifies)[-1]]


def kernel_power(signal, sensor_axis=None):
    """|s|^2 as the device forms it: re*re + im*im with every product and sum rounded (no FMA), then summed over
    sensor_axis sequentially in channel order (keepdims)."""
    signal = np.asarray(signal)
    re, im = signal.real.astype(np.float64), signal.imag.astype(np.float64)
    power = re * re + im * im
    if sensor_axis is None:
        return power
    parts = np.moveaxis(power, sensor_axis, 0)
    acc = parts[0].copy()
    for p in parts[1:]:
        acc = acc + p
    return np.expand_dims(acc, sensor_axis)


def lorenz_exact(row, fraction):
    """Exact Lorenz threshold of one row of non-negative powers, and the interval a float evaluation can give.

    -> (t, t_lo, t_hi).  t is the smallest value v whose exact Lorenz value L(v) = (S_above(v) + v) / S_total is below
    `fraction` (S_above: the sum of the elements larger than v; v's first occurrence in the descending order), or
    None when none is.  t_lo <= t <= t_hi bound every threshold a float evaluation can produce, in any summation order:

    A float sum of m non-negative terms, in any order or tree, is s (1 + theta) with |theta| <= gamma_{m-1},
    gamma_k = k u / (1 - k u) (Higham, Accuracy and Stability, Lemma 3.1 / 3.4): every partial sum is a sum of
    non-negative terms, so each rounding's error is at most u times a number no larger than s.  The numerator and the
    denominator are sums of at most n terms of the row, and the division rounds once, so the computed Lorenz value is
    L(v) (1 + theta_1)(1 + theta_2) / (1 + theta_3), which is L(v) (1 + theta) with |theta| <= gamma_{2n-1} <=
    gamma_{2n} =: g (Higham, Lemma 3.3).  A value with L(v) (1 + g) < fraction qualifies in every order, one with
    L(v) (1 - g) >= fraction in none.  L is non-decreasing down the descending order, so
      t_hi = smallest v with L(v) (1 + g) < fraction (None: possibly nothing qualifies, the caller may raise),
      t_lo = smallest v with L(v) (1 - g) < fraction.
    A mask power > t' with t' in [t_lo, t_hi] differs from power > t only at powers p with t_lo < p <= t_hi.
    A row with an infinite or NaN power has no threshold (the reference's np.min of an empty selection):
    (None, None, None).
    """
    row = np.asarray(row, dtype=np.float64).ravel()
    if not np.isfinite(row).all():
        return None, None, None
    values, counts = np.unique(row, return_counts=True)
    values, counts = values[::-1], counts[::-1]
    ratios = [v.as_integer_ratio() for v in values.tolist()]
    den = max(q for _, q in ratios)
    ints = [p * (den // q) for p, q in ratios]       # values * den, exact integers
    tops = list(itertools.accumulate(i * c for i, c in zip(ints, counts.tolist())))
    total = tops[-1]
    if total == 0:
        return None, None, None
    # L(v_j) = (tops[j - 1] + ints[j]) / total, non-decreasing in j: each condition holds on a prefix of j
    lv = [(tops[j - 1] if j else 0) + ints[j] for j in range(len(ints))]
    fn, fd = Fraction(float(fraction)).as_integer_ratio()
    n = row.size
    gn, gd = (Fraction(2 * n * U) / (1 - Fraction(2 * n * U))).as_integer_ratio()

    def last(scale_num, scale_den):
        # largest j with lv[j] scale_num / scale_den * fd < fn * total, or -1
        rhs = fn * total * scale_den
        k = bisect.bisect_left(lv, rhs, key=lambda x: x * scale_num * fd) - 1
        return float(values[k]) if k >= 0 else None

    return last(1, 1), last(gd - gn, gd), last(gd + gn, gd)


def reference_lorenz_threshold(power, lorenz_fraction):
    """The reference's get_mask (mask_module.py), written out: np.sort, [::-1], np.cumsum / np.sum, np.min over the
    qualifying prefix.  Raises ValueError for an empty selection, as the reference does."""
    sorted_power = np.sort(power, axis=None)[::-1]
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        lorenz_function = np.cumsum(sorted_power) / np.sum(sorted_power)
    return np.min(sorted_power[lorenz_function < lorenz_fraction])


def _rows(power, axis):
    if not isinstance(axis, (tuple, list)):
        axis = (axis,)
    last = tuple(-i - 1 for i in range(len(axis)))
    moved = np.moveaxis(power, axis, last)
    shape = moved.shape
    n = int(np.prod(shape[len(shape) - len(axis):]))
    return moved.reshape(-1, n), shape, last, axis


def lorenz_mask(signal, *, sensor_axis=None, axis=(-2, -1), lorenz_fraction=0.98, weight=0.999, keepdims=False):
    signal = np.asarray(signal)
    rdt = np.float32 if signal.dtype in (np.complex64, np.float32) else np.float64
    power = signal.real.astype(np.float64) ** 2 + signal.imag.astype(np.float64) ** 2
    if sensor_axis is not None:
        power = power.sum(axis=sensor_axis, keepdims=True)
    rows, shape, last, axis = _rows(power, axis)
    mask = np.zeros(rows.shape, dtype=rdt)
    for i, row in enumerate(rows):
        t = lorenz_threshold(row, lorenz_fraction)
        if t is None:
            raise ValueError(f'row {i}: no value has a Lorenz value below {lorenz_fraction}')
        mask[i] = row > t
    mask = 0.5 + weight * (mask - 0.5)
    mask = np.moveaxis(mask.reshape(shape), last, axis)
    if sensor_axis is not None and not keepdims:
        mask = np.squeeze(mask, sensor_axis)
    return mask


def percentile_terms(n, percent, dtype):
    """(k_lower, k_upper, gamma, 1 - gamma) of np.percentile's linear method in the given dtype."""
    q = np.true_divide(percent, dtype(100))
    virtual = np.asarray((n - 1) * q)
    if virtual >= n - 1:
        return n - 1, n - 1, virtual.dtype.type(0), virtual.dtype.type(1)
    if virtual < 0:
        return 0, 0, virtual.dtype.type(0), virtual.dtype.type(1)
    k = int(np.floor(virtual))
    gamma = np.asarray(virtual - k, dtype=virtual.dtype)
    return k, k + 1, gamma[()], np.asarray(1 - gamma)[()]


def percentile_rows(rows, percent):
    """np.percentile(rows, percent, axis=-1) from the order statistics k_lower / k_upper; NaN for a row that holds a
    NaN, whatever the rank (np.percentile sorts NaN last and propagates it)."""
    rows = np.asarray(rows)
    n = rows.shape[-1]
    k_lo, k_hi, g, omg = percentile_terms(n, percent, rows.dtype.type)
    part = np.partition(rows, sorted({k_lo, k_hi}), axis=-1)
    x, y = part[:, k_lo], part[:, k_hi]
    with np.errstate(invalid='ignore'):
        diff = y - x
        out = np.where(g >= 0.5, y - diff * omg, x + diff * g).astype(rows.dtype)
    return np.where(np.isnan(rows).any(axis=-1), rows.dtype.type(np.nan), out)


def quantile_mask(signal, quantile=(0.1, -0.9), *, axis=-2, weight=0.999):
    signal = np.abs(np.asarray(signal))
    if isinstance(quantile, (tuple, list)):
        return np.array([quantile_mask(signal, q, axis=axis, weight=weight) for q in quantile])
    rows, shape, last, axis = _rows(signal, axis)
    if quantile >= 0:
        thr = percentile_rows(rows, (1 - quantile) * 100)
        mask = (rows > thr[:, None]).astype(rows.dtype)
    else:
        thr = percentile_rows(rows, abs(quantile) * 100)
        mask = (rows < thr[:, None]).astype(rows.dtype)
    mask = 0.5 + weight * (mask - 0.5)
    return np.moveaxis(mask.reshape(shape), last, axis)
