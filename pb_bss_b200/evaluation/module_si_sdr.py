"""SI-SDR, the scale-invariant signal-to-distortion ratio of pb_bss/evaluation/module_si_sdr.py, on the device, with
the reference's signature, broadcasting, assert and return types: ``si_sdr(reference, estimation)``.

Le Roux, Wisdom, Erdogan and Hershey, "SDR - half-baked or well done?", ICASSP 2019: per pair of the broadcast leading
dims, alpha = <r, e> / <r, r> (pass 1), then 10 log10(sum (alpha r)^2 / sum (e - alpha r)^2) from the rounded
projection and residual (pass 2), as the reference computes them (include/pbb.h, pbb_si_sdr).  The one-pass closed
form is not used: it cancels at high SI-SDR.  Every sum has the same fixed tree, so si_sdr(r, 2 r) is exactly inf.
A broadcast operand is read in place through a row-offset table, never materialised.  fp64, bitwise reproducible,
and a pair's value does not depend on the rest of the batch.

NumPy in gives NumPy out (an np.float64 for 1-D input); a CUDA tensor in gives a float64 CUDA tensor out, and the
call only enqueues work on the current stream.  Documented difference: NumPy's divide-by-zero and invalid-value
RuntimeWarnings are not emitted; the inf / nan values are the same.
"""
import math

import numpy as np
import torch

from .. import _device, _lib


def _operand(x, shape):
    """(data, offsets): x as a contiguous float64 CUDA tensor in its own (unbroadcast) shape, and the int64 element
    offset of each of the broadcast shape's rows in it."""
    lead, n = shape[:-1], shape[-1]
    x = x.reshape((1,) * (len(shape) - x.dim()) + tuple(x.shape))
    if x.shape[-1] != n:                      # a broadcast last axis is materialised (one sample per row)
        x = x.expand(*x.shape[:-1], n)
    x = x.contiguous()
    own = tuple(x.shape[:-1])
    offsets = np.broadcast_to(np.arange(math.prod(own), dtype=np.int64).reshape(own) * n, lead).reshape(-1)
    return x, _device.to_device(np.ascontiguousarray(offsets))


def _is_float64(x):
    return x.dtype == torch.float64 if _device.is_tensor(x) else x.dtype == np.float64


def si_sdr(reference, estimation):
    """Scale-invariant SDR in dB of estimation against reference along the last axis, after broadcasting the two
    (module_si_sdr.py:4-56).  Both must be float64 (AssertionError otherwise, as in the reference).

    >>> np.random.seed(0)
    >>> reference = np.random.randn(100)
    >>> print(si_sdr(reference, reference * 2))
    inf
    >>> print(si_sdr([1., 0], [0., 0]))  # never predict only zeros
    nan
    """
    like_numpy = not (_device.is_tensor(reference) or _device.is_tensor(estimation))
    r = reference if _device.is_tensor(reference) else np.asarray(reference)
    e = estimation if _device.is_tensor(estimation) else np.asarray(estimation)
    shape = tuple(np.broadcast_shapes(tuple(e.shape), tuple(r.shape)))
    assert _is_float64(r), r.dtype
    assert _is_float64(e), e.dtype
    if len(shape) == 0:
        raise np.exceptions.AxisError(-1, 0)
    lib = _lib.load()
    lead, n = shape[:-1], shape[-1]
    rows = math.prod(lead)
    out = _device.empty(lead, torch.float64)
    if rows:
        rd, ro = _operand(_device.to_device(r), shape)
        ed, eo = _operand(_device.to_device(e), shape)
        nbytes = lib.pbb_si_sdr_workspace_bytes(rows, n)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
        _lib.check(lib.pbb_si_sdr(_device.ptr(rd) if n else None, _device.ptr(ed) if n else None, _device.ptr(ro),
                                  _device.ptr(eo), rows, n, _device.ptr(ws), nbytes, _device.ptr(out),
                                  _device.stream_ptr()), 'pbb_si_sdr')
    if not like_numpy:
        return out
    v = out.cpu().numpy()
    return np.float64(v) if v.ndim == 0 else v
