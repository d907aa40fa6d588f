"""The invasive SxR of pb_bss/evaluation/sxr_module.py on the device, with the reference's names, signatures,
asserts and return types: ``get_variance_for_zero_mean_signal``, ``get_snr``, ``input_sxr`` and ``output_sxr``.

The powers are one pass over the signals (include/pbb.h, pbb_mean_square): the mean of |x|^2 along the reduced axes,
fp64, and a row's value does not depend on the rest of the batch.  From the powers S and N, one small kernel each
(pbb_input_sxr, pbb_output_sxr) computes SDR / SIR / SNR in the reference's order of operations, with np.sum's
summation order; output_sxr searches every selection of itertools.permutations(range(K_target), K_source) and keeps
the first maximiser of the mutual power, as np.argmax does.

NumPy in gives NumPy out (an np.float64 for a single value); a CUDA tensor in gives float64 CUDA tensors out, and the
call only enqueues work on the current stream.

Documented differences from the reference:
  - integer and float32 input are computed in fp64 (the reference squares int16 in int16, where it wraps, and
    returns float32 powers for float32 input);
  - NumPy's divide-by-zero and invalid-value RuntimeWarnings are not emitted; the inf / nan values are the same;
  - as in the reference, ``output_sxr`` returns the tuple, not a dict, for a string ``return_dict``: it tests
    ``return_dict is True`` (sxr_module.py:264).
"""
import collections
import math

import numpy as np
import torch

from numpy.lib.array_utils import normalize_axis_tuple

from .. import _device, _lib, _nd

__all__ = ['get_snr', 'input_sxr', 'output_sxr']

ResultTuple = collections.namedtuple('SXR', ['sdr', 'sir', 'snr'])

MAX_K = 9    # PBB_SXR_MAX_K
MAX_D = 29   # PBB_SXR_MAX_D

_DTYPES = {torch.float32: _lib.PBB_F32, torch.float64: _lib.PBB_F64, torch.int16: _lib.PBB_I16,
           torch.int32: _lib.PBB_I32, torch.int64: _lib.PBB_I64, torch.complex64: _lib.PBB_C64,
           torch.complex128: _lib.PBB_C128}


def _like_numpy(*xs):
    return not any(_device.is_tensor(x) for x in xs)


def _out(t, like_numpy):
    """A device result as the caller gets it: the tensor, or NumPy (np.float64 for a single value)."""
    if not like_numpy:
        return t
    v = t.cpu().numpy()
    return np.float64(v) if v.ndim == 0 else v


def mean_square(x):
    """mean |x|^2 of every row of x (rows, n) on the device: float64 (rows,)."""
    lib = _lib.load()
    x = x.contiguous()
    rows, n = x.shape
    nbytes = lib.pbb_mean_square_workspace_bytes(rows, n)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x.device)
    out = torch.empty(rows, dtype=torch.float64, device=x.device)
    _device.call('pbb_mean_square', x if x.numel() else None, _DTYPES[x.dtype], rows, n, ws, nbytes, out)
    return out


def _variance(X, axis=None, keepdims=False):
    """get_variance_for_zero_mean_signal on the device: a float64 CUDA tensor of the reference's shape."""
    x = _device.to_device(X if _device.is_tensor(X) else np.array(X))
    if x.dtype not in _DTYPES:
        x = x.to(torch.float64)
    nd = x.dim()
    axes = tuple(range(nd)) if axis is None else (axis if isinstance(axis, tuple) else (axis,))
    for a in axes:
        if not -nd <= a < nd:
            raise np.exceptions.AxisError(a, nd)
    axes = tuple(sorted(a % nd for a in axes))
    if len(set(axes)) != len(axes):
        raise ValueError('duplicate value in axis')
    kept = [a for a in range(nd) if a not in axes]
    x = x.permute(*kept, *axes)
    lead = tuple(x.shape[:len(kept)])
    n = math.prod(x.shape[len(kept):])
    out = mean_square(x.reshape(math.prod(lead), n))
    if keepdims:
        return out.reshape(tuple(1 if a in axes else s for a, s in enumerate(X.shape if _device.is_tensor(X)
                                                                                else np.shape(X))))
    return out.reshape(lead)


def get_energy(x, axis=None, keepdims=False):
    """sum |x * conj(x)| over ``axis`` (sxr_module.py:13-14): re*re + im*im per element (no FMA), summed on the device
    in a fixed order (pbb_axis_sum; a long sum is split over chunks).  fp64, rounded once to the real dtype of x;
    integer input gives float64 (the reference's integer sum is int64)."""
    like = _like_numpy(x)
    t = _nd.device_view(x)
    nd = t.dim()
    axes = tuple(range(nd)) if axis is None else tuple(sorted(normalize_axis_tuple(axis, nd)))
    return _out(_nd.axis_sum(t, axes, keepdims, square=True), like)


def get_variance_for_zero_mean_signal(X, axis=None, keepdims=False):
    """np.mean(|X|^2, axis, keepdims) (sxr_module.py:17-23): re^2 + im^2 for complex X, X^2 otherwise, in fp64."""
    return _out(_variance(X, axis, keepdims), _like_numpy(X))


def get_snr(X, N, *, axis=None, keepdims=False):
    """10 log10(power of X / power of N) in dB (sxr_module.py:26-48); the powers as get_variance_for_zero_mean_signal.

    >>> print(get_snr([1, 2, 3], [1, 2, 3]))
    0.0
    """
    pX, pN = _variance(X, axis, keepdims), _variance(N, axis, keepdims)
    if _like_numpy(X, N):
        pX, pN = _out(pX, True), _out(pN, True)
        with np.errstate(divide='ignore', invalid='ignore'):
            return 10 * np.log10(pX / pN)
    return 10 * torch.log10(pX / pN)


def set_snr(X, N, snr, current_snr=None, *, axis=None, inplace=True):
    """Rescales the noise N to the SNR ``snr`` (dB) against X (sxr_module.py:51-78): factor =
    10 ** (-(snr - current_snr) / 20), current_snr = get_snr(X, N, axis=axis, keepdims=True) by default.  The few
    factors are host math; the scaling is one device pass (pbb_scale_nd).  inplace=True scales the caller's NumPy array
    or CUDA tensor N and returns None (an integer N raises NumPy's casting error, as the reference's ``N *= factor``);
    inplace=False returns (X, N * factor) in NumPy's result dtype."""
    if current_snr is None:
        current_snr = get_snr(X, N, axis=axis, keepdims=True)
    if _device.is_tensor(current_snr):
        current_snr = current_snr.cpu().numpy()
    factor = 10 ** (-(snr - current_snr) / 20)
    n_tensor = _device.is_tensor(N)
    n_dtype = np.dtype(str(N.dtype).replace('torch.', '')) if n_tensor else np.asarray(N).dtype
    if inplace:
        # NumPy's own casting check of ``N *= factor`` (UFuncTypeError for integer N)
        np.multiply(np.zeros(1, n_dtype), factor if np.ndim(factor) == 0 else np.zeros((1,) * np.ndim(factor)),
                    out=np.zeros((1,) * max(1, np.ndim(factor)), n_dtype), casting='same_kind')
        out_dtype = n_dtype
    else:
        out_dtype = np.result_type(n_dtype, factor)
    torch_out = getattr(torch, out_dtype.name)
    if inplace and n_tensor:
        x = N if N.device == _device.device() else None
        if x is None:
            raise ValueError('set_snr(inplace=True) scales a CUDA tensor or a NumPy array in place')
    else:
        x = _nd.device_view(N)
        if x.dtype != torch_out:
            x = x.to(torch_out)
    if x.dtype not in _nd.CODES:
        raise TypeError(f'set_snr: N of dtype {x.dtype} is not supported')
    f = _device.to_device(np.asarray(factor, dtype=np.float64))
    shape = tuple(np.broadcast_shapes(tuple(x.shape), tuple(f.shape)))
    if shape != tuple(x.shape):
        raise ValueError(f'non-broadcastable output operand with shape {tuple(x.shape)} doesn\'t match the broadcast '
                         f'shape {shape}')
    out = x if inplace and n_tensor else _device.empty(shape, x.dtype)
    lay = _nd.layout(shape, x.stride(), _nd.broadcast_strides(f, shape), out.stride())
    _device.call('pbb_scale_nd', x if x.numel() else None, _nd.CODES[x.dtype], f, lay, out if out.numel() else None)
    if inplace:
        if not n_tensor:
            N[...] = out.cpu().numpy()
        return None
    return X, _device.to_host(out, not n_tensor)


def _result(values, return_dict, strict):
    if return_dict is True:
        return dict(zip(('sdr', 'sir', 'snr'), values))
    if return_dict and not strict:
        if isinstance(return_dict, str):
            return dict(zip((return_dict + 'sdr', return_dict + 'sir', return_dict + 'snr'), values))
        raise TypeError(return_dict)
    return ResultTuple(*values)


def input_sxr_from_powers(S, N, average_sources=True, average_channels=True):
    """SDR, SIR, SNR (float64 CUDA tensors) of input_sxr from the powers S (K, D) and N (D), float64 CUDA tensors."""
    K, D = S.shape
    shape = {(True, True): (), (False, True): (K,), (True, False): (D,), (False, False): (K, D)}[
        (bool(average_sources), bool(average_channels))]
    out = [_device.empty(shape, torch.float64) for _ in range(3)]
    S, N = S.contiguous(), N.contiguous()
    _device.call('pbb_input_sxr', S, N, K, D, int(bool(average_sources)), int(bool(average_channels)), *out)
    return out


def input_sxr(images, noise, average_sources=True, average_channels=True, *, return_dict=False):
    """Input SDR, SIR and SNR (sxr_module.py:94-165) of images (K, D, T) and noise (D, T): the power of each image
    against the sum of the other images' powers (I) and the noise power (N), per source and channel, averaged over
    the channels and / or the sources on request.  Returns ``ResultTuple(sdr, sir, snr)``, or a dict with the keys
    sdr, sir, snr (prefixed with ``return_dict`` when it is a string)."""
    K, D, T = images.shape
    assert (D, T) == tuple(noise.shape), ((D, T), images.shape, noise.shape)
    assert K < 10, images.shape
    assert D < 30, images.shape
    S = _variance(images, axis=-1)
    N = _variance(noise, axis=-1)
    values = input_sxr_from_powers(S, N, average_sources, average_channels)
    like_numpy = _like_numpy(images, noise)
    return _result([_out(v, like_numpy) for v in values], return_dict, strict=False)


def output_sxr_from_powers(S, N, average_sources=True):
    """SDR, SIR, SNR and the selection (int64 (K_source,)) of output_sxr from the powers S (K_source, K_target) and N
    (K_target), float64 CUDA tensors.  K_source > K_target raises the ValueError of np.argmax of nothing."""
    lib = _lib.load()
    K_source, K_target = S.shape
    if K_source > K_target:
        raise ValueError('attempt to get argmax of an empty sequence')
    shape = () if average_sources else (K_source,)
    out = [_device.empty(shape, torch.float64) for _ in range(3)]
    selection = _device.empty((K_source,), torch.int64)
    nbytes = lib.pbb_output_sxr_workspace_bytes(K_source, K_target)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=S.device)
    S, N = S.contiguous(), N.contiguous()
    _device.call('pbb_output_sxr', S, N, K_source, K_target, int(bool(average_sources)), ws, nbytes, *out, selection)
    return out + [selection]


def output_sxr(image_contribution, noise_contribution, average_sources=True, return_dict=False):
    """Output SDR, SIR and SNR (sxr_module.py:168-274) of image_contribution (K_source, K_target, T) and
    noise_contribution (K_target, T): the selection of one output per source with the largest summed power, then per
    source its power on the selected output against the other sources' powers there (I) and the noise power there (N).
    Returns ``ResultTuple(sdr, sir, snr)``, or a dict with the keys sdr, sir, snr for ``return_dict=True``.  A string
    ``return_dict`` returns the tuple, as in the reference."""
    K_source, K_target, samples = image_contribution.shape
    assert tuple(noise_contribution.shape) == (K_target, samples), (image_contribution.shape,
                                                                     noise_contribution.shape)
    assert K_source < 10, (image_contribution.shape, noise_contribution.shape)
    assert K_target < 10, (image_contribution.shape, noise_contribution.shape)
    S = _variance(image_contribution, axis=-1)
    N = _variance(noise_contribution, axis=-1)
    values = output_sxr_from_powers(S, N, average_sources)[:3]
    like_numpy = _like_numpy(image_contribution, noise_contribution)
    return _result([_out(v, like_numpy) for v in values], return_dict, strict=True)
