"""NumPy restatement of the selection algorithms behind the device's lorenz_mask and quantile_mask (csrc/mask.cuh).

Lorenz: the reference sorts each row and takes the minimum over the prefix whose cumsum / sum is below the fraction.
Here the threshold is found the way the kernel finds it, without a sort of the row: over the distinct values v in
descending order, v qualifies when (sum of the elements above v + v) / sum < fraction, which is the Lorenz value of
the first element of v's group; the qualifying values form a prefix and the threshold is the smallest of them.

Quantile: np.percentile's linear method from two explicit order statistics, selected with np.partition, and NumPy's
_lerp in the dtype of the values.  Checked against the reference's fixture by tests/test_mask_oracle.py.
"""
import numpy as np


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
    """np.percentile(rows, percent, axis=-1) from the order statistics k_lower / k_upper."""
    rows = np.asarray(rows)
    n = rows.shape[-1]
    k_lo, k_hi, g, omg = percentile_terms(n, percent, rows.dtype.type)
    part = np.partition(rows, sorted({k_lo, k_hi}), axis=-1)
    x, y = part[:, k_lo], part[:, k_hi]
    diff = y - x
    return np.where(g >= 0.5, y - diff * omg, x + diff * g).astype(rows.dtype)


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
