"""Oracle masks on the device, signatures of pb_bss/extraction/mask_module.py.

Every mask takes the (complex or real) STFT images of the sources and reads them on the device in their own layout:
any source / sensor axis, any number of independent dims, no transposed copy.  The arithmetic is fp64; the output
dtype follows the reference (the real dtype of the signal, the complex dtype for ideal_complex_mask, bool for
biased_binary_mask).  numpy in -> numpy out, CUDA tensors in -> CUDA tensors out; lists are taken like np.asarray
takes them.
"""
from typing import Optional

import numpy as np
import torch
from numpy.lib.array_utils import normalize_axis_index, normalize_axis_tuple

from .. import _device, _lib

EPS = 1e-18

__all__ = [
    'voiced_unvoiced_split_characteristic',
    'ideal_binary_mask',
    'wiener_like_mask',
    'ideal_ratio_mask',
    'ideal_amplitude_mask',
    'phase_sensitive_mask',
    'ideal_complex_mask',
    'lorenz_mask',
    'quantile_mask',
    'biased_binary_mask',
]

_SENSOR_AXIS_UNDEFINED = ('sensor_axis is not defined for this mask: pooling |s| or s over the sensors would '
                          'not keep the complex signal the mask is defined on')

_CODES = {torch.complex128: _lib.PBB_C128, torch.complex64: _lib.PBB_C64,
          torch.float64: _lib.PBB_F64, torch.float32: _lib.PBB_F32}
_REAL = {torch.complex128: torch.float64, torch.complex64: torch.float32,
         torch.float64: torch.float64, torch.float32: torch.float32}


def _signal(signal):
    """-> (CUDA tensor in its own strides, like_numpy).  Other dtypes than complex64/128 and float32/64 are taken
    as float64."""
    like_numpy = not _device.is_tensor(signal)
    if like_numpy:
        x = np.asarray(signal)
        if x.dtype not in (np.complex128, np.complex64, np.float64, np.float32):
            x = x.astype(np.float64)
        x = _device.to_device(x)
    else:
        x = signal
        if x.dtype not in _CODES:
            x = x.to(torch.float64)
        if x.device != _device.device():
            x = x.to(_device.device())
    return x, like_numpy


def _contiguous_strides(shape):
    strides, s = [], 1
    for n in reversed(shape):
        strides.append(s)
        s *= n
    return strides[::-1]


def _layout(dims):
    """[(size, in_stride, out_stride)] in row-major order -> pbb_mask_layout, dims of size 1 dropped and neighbours
    that are contiguous in both input and output merged."""
    merged = []
    for size, si, so in dims:
        if size == 1:
            continue
        if merged and merged[-1][1] == si * size and merged[-1][2] == so * size:
            merged[-1] = (merged[-1][0] * size, si, so)
        else:
            merged.append((size, si, so))
    if len(merged) > _lib.MASK_MAX_DIMS:
        raise NotImplementedError(f'more than {_lib.MASK_MAX_DIMS} non-mergeable dims')
    lay = _lib.MaskLayout()
    lay.nd = len(merged)
    for a, (size, si, so) in enumerate(merged):
        lay.shape[a], lay.in_stride[a], lay.out_stride[a] = size, si, so
    return lay


def _mask_values(dtype, weight):
    """The two values of 0.5 + weight * (mask - 0.5) in the reference's output dtype."""
    lo, hi = 0.5 + weight * (np.array([0.0, 1.0], dtype=dtype) - 0.5)
    return float(lo), float(hi)


def _source_mask(kind, signal, source_axis, sensor_axis, keepdims, eps):
    x, like_numpy = _signal(signal)
    nd = x.dim()
    sa = normalize_axis_index(source_axis, nd)
    se = None if sensor_axis is None else normalize_axis_index(sensor_axis, nd)
    if se == sa:
        raise ValueError('source_axis and sensor_axis must differ')
    shape = list(x.shape)
    keep_shape = list(shape)
    if se is not None:
        keep_shape[se] = 1
    complex_out = kind == _lib.MASK_IDEAL_COMPLEX and x.is_complex()
    out = _device.empty(keep_shape, x.dtype if complex_out else _REAL[x.dtype])
    if out.numel():
        ostr = _contiguous_strides(keep_shape)
        rest = _layout([(shape[a], x.stride(a), ostr[a]) for a in range(nd) if a not in (sa, se)])
        _device.call('pbb_source_mask', x, _CODES[x.dtype], kind, shape[sa], 1 if se is None else shape[se],
                     x.stride(sa), 0 if se is None else x.stride(se), ostr[sa], rest, eps, out)
    if se is not None and not keepdims:
        out = out.squeeze(se)
    return _device.to_host(out, like_numpy)


def voiced_unvoiced_split_characteristic(
        frequency_bins: int,
        split_bin: Optional[int] = None,
        width: Optional[int] = None
):
    """Voiced and unvoiced frequency weightings (mask_module.py:53-87): 1 below the split, a raised-cosine
    transition of `width` bins starting one bin before int(split_bin - width / 2), 0 above; unvoiced = 1 - voiced.
    A function of integers, computed on the host like the reference."""
    split_bin = frequency_bins // 2 if split_bin is None else split_bin
    width = frequency_bins // 5 if width is None else width
    ramp = 0.5 * (1 + np.cos(np.pi / (width - 1) * np.arange(0, width)))
    first = int(split_bin - width / 2) - 1
    voiced = np.ones(frequency_bins)
    voiced[first:first + width] = ramp
    voiced[first + width:] = 0
    return voiced, 1 - voiced


def ideal_binary_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
        keepdims: bool = False
) -> np.ndarray:
    """1 for the source of largest power (summed over sensor_axis if given; the first on ties), else 0
    (mask_module.py:90-136).  dtype: the real dtype of the signal."""
    return _source_mask(_lib.MASK_IDEAL_BINARY, signal, source_axis, sensor_axis, keepdims, 0.0)


def wiener_like_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
        eps: float = EPS,
        keepdims: bool = False
) -> np.ndarray:
    """Source power / (total power + eps), power summed over sensor_axis if given (mask_module.py:139-179)."""
    return _source_mask(_lib.MASK_WIENER_LIKE, signal, source_axis, sensor_axis, keepdims, eps)


def ideal_ratio_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
        eps: float = EPS,
) -> np.ndarray:
    """|s| / (sum over sources of |s| + eps) (mask_module.py:182-232)."""
    assert sensor_axis is None, _SENSOR_AXIS_UNDEFINED
    return _source_mask(_lib.MASK_IDEAL_RATIO, signal, source_axis, None, False, eps)


def ideal_amplitude_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
        eps: float = EPS,
) -> np.ndarray:
    """|s| / (|sum over sources of s| + eps) (mask_module.py:235-287)."""
    assert sensor_axis is None, _SENSOR_AXIS_UNDEFINED
    return _source_mask(_lib.MASK_IDEAL_AMPLITUDE, signal, source_axis, None, False, eps)


def phase_sensitive_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
        eps: float = EPS,
) -> np.ndarray:
    """|s| / (|o| + eps) * cos(angle(s) - angle(o)) with o the sum over sources (mask_module.py:290-322)."""
    assert sensor_axis is None, _SENSOR_AXIS_UNDEFINED
    return _source_mask(_lib.MASK_PHASE_SENSITIVE, signal, source_axis, None, False, eps)


def ideal_complex_mask(
        signal: np.ndarray,
        source_axis: int = 0,
        sensor_axis: Optional[int] = None,
) -> np.ndarray:
    """s / (sum over sources of s), no eps: a zero observation gives NumPy's inf / nan (mask_module.py:325-347)."""
    assert sensor_axis is None, _SENSOR_AXIS_UNDEFINED
    return _source_mask(_lib.MASK_IDEAL_COMPLEX, signal, source_axis, None, False, 0.0)


def _row_geometry(x, elem_axes, pooled_axis, out_shape):
    """Row / element layouts for the selection masks: the elements of a row are the dims in elem_axes, the rows all
    other dims except the pooled sensor axis."""
    nd = x.dim()
    ostr = _contiguous_strides(out_shape)
    rows = _layout([(x.shape[a], x.stride(a), ostr[a]) for a in range(nd) if a not in elem_axes and a != pooled_axis])
    elems = _layout([(x.shape[a], x.stride(a), ostr[a]) for a in range(nd) if a in elem_axes and a != pooled_axis])
    n_rows = int(np.prod([x.shape[a] for a in range(nd) if a not in elem_axes and a != pooled_axis]))
    n = int(np.prod([x.shape[a] for a in elem_axes if a != pooled_axis]))
    return rows, elems, n_rows, n


def _scratch(n_rows, n):
    if n <= _lib.ROW_SELECT_SHORT_MAX:
        return None, 0
    nbytes = _lib.load().pbb_row_select_scratch_bytes(n_rows, n)
    return _device.workspace(nbytes), nbytes


def lorenz_mask(
        signal: np.ndarray,
        *,
        sensor_axis=None,
        axis=(-2, -1),
        lorenz_fraction: float = 0.98,
        weight: float = 0.999,
        keepdims: bool = False,
) -> np.ndarray:
    """Softened mask by the Lorenz-function criterion (mask_module.py:350-417).

    Per row (the power |s|^2, summed over sensor_axis if given, flattened over `axis`): the threshold is the
    smallest value among the descending-sorted ones whose cumsum / sum is below lorenz_fraction; the mask is
    0.5 + weight * ((power > threshold) - 0.5).  A row where no value qualifies raises ValueError, as np.min of the
    empty selection does in the reference."""
    x, like_numpy = _signal(signal)
    nd = x.dim()
    if not isinstance(axis, (tuple, list)):
        axis = (axis,)
    elem_axes = normalize_axis_tuple(tuple(axis), nd)
    se = None if sensor_axis is None else normalize_axis_index(sensor_axis, nd)
    out_shape = list(x.shape)
    if se is not None:
        out_shape[se] = 1
    rdt = _REAL[x.dtype]
    lo, hi = _mask_values(np.float32 if rdt == torch.float32 else np.float64, weight)
    out = _device.empty(out_shape, rdt)
    if out.numel():
        rows, elems, n_rows, n = _row_geometry(x, elem_axes, se, out_shape)
        scratch, nbytes = _scratch(n_rows, n)
        status = torch.zeros(1, dtype=torch.int32, device=x.device)
        _device.call('pbb_lorenz_mask', x, _CODES[x.dtype], 1 if se is None else x.shape[se],
                     0 if se is None else x.stride(se), rows, elems, float(lorenz_fraction), lo, hi, out, scratch,
                     nbytes, status)

        def on_error(s):
            raise ValueError(f'lorenz_mask: no value of row {s - 1} has a Lorenz value below lorenz_fraction='
                             f'{lorenz_fraction} (zero-size array to reduction operation minimum which has no '
                             'identity)')
        _device.check_status(status, on_error)
    if se is not None and not keepdims:
        out = out.squeeze(se)
    return _device.to_host(out, like_numpy)


def _percentile_terms(n, percent, np_dtype):
    """np.percentile's linear method (numpy/lib/_function_base_impl.py: percentile, _quantile, _get_indexes,
    _get_gamma) for a row of n values: (k_lower, k_upper, gamma, 1 - gamma), with q, the virtual index and gamma in
    the dtype of the values."""
    q = np.true_divide(percent, np_dtype(100))
    if not (0 <= q <= 1):
        raise ValueError('Percentiles must be in the range [0, 100]')
    virtual = np.asanyarray((n - 1) * q)
    previous = np.floor(virtual)
    if virtual >= n - 1:
        k_lower = k_upper = n - 1
        previous = np.asanyarray(-1.0)
    elif virtual < 0:
        k_lower = k_upper = 0
        previous = np.asanyarray(0.0)
    else:
        k_lower, k_upper = int(previous), int(previous) + 1
    gamma = np.asanyarray(virtual - previous.astype(np.intp), dtype=virtual.dtype)
    return k_lower, k_upper, float(gamma), float(np.asanyarray(1 - gamma))


def quantile_mask(
        signal: np.ndarray,
        quantile=(0.1, -0.9),
        *,
        sensor_axis=None,
        axis=-2,
        weight: float = 0.999,
) -> np.ndarray:
    """Mask from a per-row percentile of |signal| (mask_module.py:420-493): q >= 0 marks |s| above the
    (1 - q) * 100 percentile, q < 0 |s| below the |q| * 100 percentile, softened by weight.  A tuple / list of
    quantiles stacks the masks into (len(quantile), *signal.shape)."""
    x, like_numpy = _signal(signal)
    assert sensor_axis is None, _SENSOR_AXIS_UNDEFINED
    if isinstance(quantile, (tuple, list)):
        masks = [quantile_mask(x, quantile=q, axis=axis, weight=weight) for q in quantile]
        out = torch.stack(masks) if masks else _device.empty((0, *x.shape), _REAL[x.dtype])
        return _device.to_host(out, like_numpy)
    nd = x.dim()
    if not isinstance(axis, (tuple, list)):
        axis = (axis,)
    elem_axes = normalize_axis_tuple(tuple(axis), nd)
    rdt = _REAL[x.dtype]
    np_dtype = np.float32 if rdt == torch.float32 else np.float64
    lo, hi = _mask_values(np_dtype, weight)
    out = _device.empty(list(x.shape), rdt)
    if out.numel():
        rows, elems, n_rows, n = _row_geometry(x, elem_axes, None, list(x.shape))
        percent = (1 - quantile) * 100 if quantile >= 0 else abs(quantile) * 100
        k_lower, k_upper, gamma, one_minus_gamma = _percentile_terms(n, percent, np_dtype)
        scratch, nbytes = _scratch(n_rows, n)
        _device.call('pbb_quantile_mask', x, _CODES[x.dtype], rows, elems, k_lower, k_upper, gamma, one_minus_gamma,
                     int(quantile < 0), lo, hi, out, scratch, nbytes)
    return _device.to_host(out, like_numpy)


def biased_binary_mask(
        signal: np.ndarray,
        component_axis: int = 0,
        sensor_axis: Optional[int] = None,
        frequency_axis: int = -1,
        threshold_unvoiced_speech: int = 5,
        threshold_voiced_speech: int = 0,
        threshold_unvoiced_noise: int = -10,
        threshold_voiced_noise: int = -10,
        low_cut: int = 5,
        high_cut: int = 500,
) -> np.ndarray:
    """Speech / noise binary masks with frequency-dependent dB thresholds (mask_module.py:496-550), concatenated
    along component_axis, dtype bool.  As in the reference the thresholds (length signal.shape[frequency_axis])
    broadcast over the LAST axis, the cuts are [..., 0:low_cut - 1] and [..., high_cut:shape[1]] of the half array,
    and 0.005 floors both power thresholds."""
    x, like_numpy = _signal(signal)
    nd = x.dim()
    ca = normalize_axis_index(component_axis, nd)
    assert x.shape[ca] == 2, 'Only works for one speaker and noise.'
    voiced, unvoiced = voiced_unvoiced_split_characteristic(x.shape[frequency_axis])
    threshold_speech = threshold_voiced_speech * voiced + threshold_unvoiced_speech * unvoiced
    threshold_noise = threshold_unvoiced_noise * voiced + threshold_voiced_noise * unvoiced
    if sensor_axis is not None:
        raise NotImplementedError()
    half = list(x.shape)
    half[ca] = 1
    if tuple(np.broadcast_shapes(tuple(half), threshold_speech.shape)) != tuple(half):
        raise ValueError(f'thresholds of shape {threshold_speech.shape} do not broadcast to {tuple(half)}')
    L = half[-1]
    speech_div = np.ascontiguousarray(np.broadcast_to(10 ** (threshold_speech / 10), (L,)))
    noise_div = np.ascontiguousarray(np.broadcast_to(10 ** (threshold_noise / 10), (L,)))
    force = np.zeros(L, dtype=np.uint8)
    force[0:low_cut - 1] = 1
    force[high_cut:half[1] if nd > 1 else L] = 1
    out = _device.empty(list(x.shape), torch.bool)
    if out.numel():
        ostr = _contiguous_strides(list(x.shape))
        rest = _layout([(x.shape[a], x.stride(a), ostr[a]) for a in range(nd) if a != ca])
        sd, nd_, fc = (_device.to_device(a) for a in (speech_div, noise_div, force))
        _device.call('pbb_biased_binary_mask', x, _CODES[x.dtype], x.stride(ca), ostr[ca], rest, L, sd, nd_, fc, out)
    return _device.to_host(out, like_numpy)
