"""Host bookkeeping of the strided building-block kernels (include/pbb.h, pbb_nd_layout): operands on the device in
their own strides, and the index-space descriptors the kernels walk.  Nothing here computes."""
import numpy as np
import torch

from . import _device, _lib

CODES = {torch.float32: _lib.PBB_F32, torch.float64: _lib.PBB_F64,
         torch.complex64: _lib.PBB_C64, torch.complex128: _lib.PBB_C128}
REAL = {torch.float32: torch.float32, torch.float64: torch.float64,
        torch.complex64: torch.float32, torch.complex128: torch.float64}


def like_numpy(*xs):
    """NumPy out unless one of the operands is a torch tensor."""
    return not any(_device.is_tensor(x) for x in xs)


def device_view(x, floating=True):
    """x (array-like / tensor) -> CUDA tensor in its own strides (a host array is uploaded as it is laid out).
    floating: dtypes other than float32 / float64 / complex64 / complex128 become float64, as NumPy's float
    arithmetic takes integers and booleans."""
    if _device.is_tensor(x):
        t = x if x.device == _device.device() else x.to(_device.device())
    else:
        a = np.asarray(x)
        if not (a.flags.c_contiguous or a.flags.f_contiguous) or not a.flags.writeable or a.dtype.byteorder == '>':
            a = np.ascontiguousarray(a)
        t = torch.from_numpy(a).to(_device.device())
    if floating and t.dtype not in CODES:
        t = t.to(torch.float64)
    return t


def layout(shape, *strides):
    """The index space ``shape`` with one stride tuple per operand -> pbb_nd_layout; dims of size 1 are dropped and
    neighbours that are contiguous for every operand are merged."""
    merged = []
    for a, n in enumerate(shape):
        if n == 1:
            continue
        st = [s[a] for s in strides]
        if merged and all(ps == s * n for ps, s in zip(merged[-1][1], st)):
            merged[-1] = (merged[-1][0] * n, st)
        else:
            merged.append((n, st))
    if len(merged) > _lib.ND_MAX_DIMS:
        raise NotImplementedError(f'more than {_lib.ND_MAX_DIMS} non-mergeable dims')
    lay = _lib.NdLayout()
    lay.nd = len(merged)
    for a, (n, st) in enumerate(merged):
        lay.shape[a] = n
        for o, s in enumerate(st):
            lay.stride[o][a] = s
    return lay


def broadcast_strides(t, shape):
    """Strides of tensor t read as ``shape`` (0 along broadcast dims)."""
    return t.expand(shape).stride()


def axis_sum(x, axes, keepdims, multiplier=None, square=False, divide_by_count=False, out_dtype=None):
    """Sum over ``axes`` (normalised, sorted) of x * multiplier (real x) or |x|^2 (square) on the device
    (pbb_axis_sum, long reductions split over chunks), optionally divided by the number of summed elements
    (np.mean).  x and multiplier are read as their broadcast shape.  -> float tensor of the reduced shape."""
    shape = tuple(x.shape) if multiplier is None else tuple(torch.broadcast_shapes(x.shape, multiplier.shape))
    kept = [a for a in range(len(shape)) if a not in axes]
    out_shape = tuple(1 if a in axes else n for a, n in enumerate(shape))
    out_dtype = out_dtype or REAL[x.dtype]
    out = _device.empty(out_shape, out_dtype)
    xs = broadcast_strides(x, shape)
    ms = broadcast_strides(multiplier, shape) if multiplier is not None else (0,) * len(shape)
    os_ = out.stride()
    outer = layout([shape[a] for a in kept], [xs[a] for a in kept], [ms[a] for a in kept], [os_[a] for a in kept])
    red = layout([shape[a] for a in axes], [xs[a] for a in axes], [ms[a] for a in axes])
    count = int(np.prod([shape[a] for a in axes])) if axes else 1
    lib = _lib.load()
    outs = int(np.prod(out_shape))
    nbytes = lib.pbb_reduce_workspace_bytes(outs, count)
    ws = _device.workspace(max(nbytes, 1))
    _device.call('pbb_axis_sum', x if x.numel() else None, CODES[x.dtype], multiplier, outer, red, int(square),
                 float(count) if divide_by_count else 1.0, out if out.numel() else None, CODES[out_dtype], ws, nbytes)
    if not keepdims:
        out = out.reshape(tuple(shape[a] for a in kept))
    return out
