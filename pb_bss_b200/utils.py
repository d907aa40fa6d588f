"""pb_bss/utils.py: labels_to_one_hot, get_pca and abs_square on the device; the shape helpers (reshape, unsqueeze,
is_broadcast_compatible), get_stft_center_frequencies and the ``deprecated`` decorator on the host.

NumPy in gives NumPy out, CUDA tensors in give CUDA tensors out."""
import functools
import inspect
import math
import warnings

import numpy as np
import torch

from . import _device, _lib, _nd
from .extraction.beamform_utils import get_stft_center_frequencies  # noqa: F401
from .extraction.linalg import eigh


class DeprecatedWarning(UserWarning):
    pass


def deprecated(instructions):
    """Flags a function as deprecated (utils.py:12-43): every call warns with a DeprecatedWarning at the caller."""
    def decorator(func):
        @functools.wraps(func)
        def wrapper(*args, **kwargs):
            message = 'Call to deprecated function {} ({}). {}'.format(
                func.__qualname__, inspect.getfile(func), instructions)
            frame = inspect.currentframe().f_back
            warnings.warn_explicit(message, category=DeprecatedWarning, filename=inspect.getfile(frame.f_code),
                                   lineno=frame.f_lineno)
            return func(*args, **kwargs)
        return wrapper
    return decorator


def _normalize(op):
    op = op.replace(',', '').replace(' ', '')
    op = ' '.join(c for c in op)
    return op.replace(' * ', '*').replace('- >', '->')


def reshape(array, operation):
    """The generalised reshape of utils.py:46-116, e.g. ``reshape(x, 'a b c -> c a*b')``: squeeze the '1' dims,
    transpose, merge the '*' groups.  Only views and permutes; a tensor whose permuted dims cannot be merged as a
    view is copied once (.reshape)."""
    operation = _normalize(operation)
    if '*' in operation.split('->')[0]:
        raise NotImplementedError(
            'Unflatten operation not supported by design. '
            'Actual values for dimensions are not available to this function.')
    lhs, rhs = operation.split('->')
    tensor = _device.is_tensor(array)
    for axis, op in reversed(list(enumerate(lhs.split()))):
        if op == '1':
            array = array.squeeze(axis) if tensor else np.squeeze(array, axis=axis)
    source = [c for c in lhs.split() if c != '1']
    order = [c for c in rhs.replace('1', ' ').replace('*', ' ').split()]
    if sorted(source) != sorted(order) or len(set(source)) != len(source):
        raise ValueError(f'op: {operation}, shape: {tuple(np.shape(array))}')
    perm = [source.index(c) for c in order]
    array = array.permute(*perm) if tensor else np.transpose(array, perm)
    size = dict(zip(order, array.shape))
    shape = [1 if t == '1' else math.prod(size[c] for c in t.split('*')) for t in rhs.replace(' * ', '*').split()]
    return array.reshape(shape)


def get_pca(target_psd_matrix, use_scipy=False):
    """The principal eigenvector (..., D) and its eigenvalue (...) of every Hermitian matrix (utils.py:119-178),
    through the device eigensolver of extraction.beamformer.get_pca (pbb_heig_batched).  use_scipy=True returns what
    the reference's scipy branch returns: it decomposes ``target_psd_matrix[-1]`` (the last matrix) for every
    index, so every row of the result is that matrix's principal pair.  The eigensolver is complex, so real input gives
    complex eigenvectors (the reference's are real; the eigenvalues are the same)."""
    tensor = _device.is_tensor(target_psd_matrix)
    x = target_psd_matrix if tensor else np.asarray(target_psd_matrix)
    shape = tuple(x.shape)
    flat = x.reshape((-1,) + shape[-2:])
    if use_scipy:
        last = flat[-1:]
        flat = last.expand(flat.shape) if tensor else np.broadcast_to(last, flat.shape)
    w, v = eigh(flat)
    vec, val = v[..., -1], w[..., -1]
    if tensor:
        vec, val = vec.contiguous(), val.contiguous()
    return vec.reshape(shape[:-1]), val.reshape(shape[:-2])


def is_broadcast_compatible(*shapes):
    """True if the shapes broadcast against each other (utils.py:193-202)."""
    if len(shapes) < 2:
        return True
    for dim in zip(*[shape[::-1] for shape in shapes]):
        if len(set(dim).union({1})) > 2:
            return False
    return True


_TORCH_DTYPES = {np.dtype(k): v for k, v in [
    (np.bool_, torch.bool), (np.uint8, torch.uint8), (np.int8, torch.int8), (np.int16, torch.int16),
    (np.int32, torch.int32), (np.int64, torch.int64), (np.float16, torch.float16), (np.float32, torch.float32),
    (np.float64, torch.float64), (np.complex64, torch.complex64), (np.complex128, torch.complex128)]}


def labels_to_one_hot(labels, categories: int, axis: int = 0, keepdims=False, dtype=bool):
    """One-hot coding of integer labels along ``axis`` (utils.py:205-311), written by one device pass in its final
    layout (pbb_labels_to_one_hot), with no moveaxis copy.  Any NumPy dtype (the output holds that dtype's 1 and
    0); negative labels wrap as NumPy indexing does; a label outside [-categories, categories) raises IndexError.
    keepdims=True replaces the singleton ``axis`` of labels by the categories."""
    like = _nd.like_numpy(labels)
    if not like:
        lab = labels.to(_device.device())
        if lab.dtype.is_floating_point or lab.dtype.is_complex:
            raise IndexError('arrays used as indices must be of integer (or boolean) type')
    else:
        lab = np.asarray(labels)
        if lab.dtype.kind not in 'iub':
            raise IndexError('arrays used as indices must be of integer (or boolean) type')
    shape = tuple(lab.shape)
    if keepdims:
        assert shape[axis] == 1
        result_ndim = len(shape)
    else:
        result_ndim = len(shape) + 1
    if axis < 0:
        axis += result_ndim
    if not 0 <= axis < result_ndim:
        raise np.exceptions.AxisError(axis, result_ndim)
    rest = shape[axis + 1:] if keepdims else shape[axis:]
    out_shape = shape[:axis] + (categories,) + rest
    outer, inner = math.prod(shape[:axis]), math.prod(rest)
    np_dtype = np.dtype(dtype)
    one = np.ones(1, np_dtype).tobytes()
    if like:
        lab = _device.to_device(lab.astype(np.int64, copy=False))
        out = torch.empty(math.prod(out_shape) * np_dtype.itemsize, dtype=torch.uint8, device=_device.device())
    else:
        lab = lab.to(torch.int64).contiguous()
        out = torch.empty(out_shape, dtype=_TORCH_DTYPES[np_dtype], device=_device.device())
    status = torch.zeros((), dtype=torch.int32, device=_device.device())
    _device.call('pbb_labels_to_one_hot', lab if lab.numel() else None, outer, inner, int(categories),
                 np_dtype.itemsize, one, out if out.numel() else None, status)

    def on_error(s):
        raise IndexError(f'index {int(lab.reshape(-1)[s - 1])} is out of bounds for axis 0 with size {categories}')
    _device.check_status(status, on_error)
    if like:
        return out.cpu().numpy().view(np_dtype).reshape(out_shape)
    return out


_ABS_SQUARE_CODES = {torch.float32: _lib.PBB_F32, torch.float64: _lib.PBB_F64, torch.complex64: _lib.PBB_C64,
                     torch.complex128: _lib.PBB_C128, torch.int32: _lib.PBB_I32, torch.int64: _lib.PBB_I64}


def abs_square(x):
    """re*re + im*im for complex x, x*x for real x (utils.py:314-336), one device pass in the precision of the input
    (no FMA, as NumPy), with NumPy's result dtype.  int8 / int16 / uint8 / uint16 / uint32 are squared in int64 and
    wrapped back to their type, which gives NumPy's bits; bool is squared as int8 (NumPy's True ** 2 is int8 1);
    float16 is squared in float32 and rounded once to float16, which is exact.  uint64 is taken as float64 (NumPy
    keeps uint64)."""
    like = _nd.like_numpy(x)
    t = _nd.device_view(x, floating=False)
    dtype = t.dtype
    if dtype == torch.bool:
        dtype = torch.int8
    if dtype in (torch.int8, torch.int16, torch.uint8, torch.uint16, torch.uint32):
        t = t.to(torch.int64)
    elif dtype == torch.float16:
        t = t.to(torch.float32)
    elif dtype not in _ABS_SQUARE_CODES:
        t = t.to(torch.float64)
        dtype = torch.float64
    t = t.contiguous()
    out = _device.empty(tuple(t.shape), _nd.REAL.get(t.dtype, t.dtype))
    _device.call('pbb_abs_square', t if t.numel() else None, _ABS_SQUARE_CODES[t.dtype], t.numel(),
                 out if out.numel() else None)
    if out.dtype != _nd.REAL.get(dtype, dtype):
        out = out.to(_nd.REAL.get(dtype, dtype))
    return _device.to_host(out, like)


def unsqueeze(array, axis):
    """Inserts singleton dims at ``axis`` (a tuple) of the result (utils.py:339-366)."""
    tensor = _device.is_tensor(array)
    if not tensor:
        array = np.array(array)
    shape = list(array.shape)
    future_ndim = len(shape) + len(axis)
    try:
        np.empty((future_ndim,))[list(axis)]
    except IndexError as e:
        raise IndexError(tuple(array.shape), shape, axis) from e
    axis = [a % future_ndim for a in axis]
    for p in sorted(axis):
        shape.insert(p, 1)
    return array.reshape(shape)
