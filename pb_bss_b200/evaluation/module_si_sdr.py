"""SI-SDR, the scale-invariant signal-to-distortion ratio of pb_bss/evaluation/module_si_sdr.py, on the device, with
the reference's signature, broadcasting, assert and return types: ``si_sdr(reference, estimation)``.

Le Roux, Wisdom, Erdogan and Hershey, "SDR - half-baked or well done?", ICASSP 2019: per pair of the broadcast leading
dims, alpha = <r, e> / <r, r> (pass 1), then 10 log10(sum (alpha r)^2 / sum (e - alpha r)^2) from the rounded
projection and residual (pass 2), as the reference computes them (include/pbb.h, pbb_si_sdr).  The one-pass closed
form is not used: it cancels at high SI-SDR.  Every sum has the same fixed tree, so si_sdr(r, 2 r) is exactly inf.
A broadcast operand is read in place through a row-offset table, never materialised.  fp64, bitwise reproducible,
and a pair's value does not depend on the rest of the batch.

NumPy in gives NumPy out (an np.float64 for 1-D input); a CUDA tensor in gives a float64 CUDA tensor out, and the
call only enqueues work on the current stream.  CUDA tensors that require grad get a graph: the backward runs
pbb_si_sdr_backward, ds/de = (20 / ln 10)(p / P - q / Q) and ds/dr = (20 alpha / ln 10)(1 / P + 1 / Q) q with
p = alpha r, q = e - p, P = |p|^2, Q = |q|^2; a broadcast operand's gradient sums the rows that share it.  Rows whose
value is inf or nan (r = 0, e = 2 r, ...) give non-finite gradients.  Double backward raises.  Documented difference: NumPy's divide-by-zero and invalid-value
RuntimeWarnings are not emitted; the inf / nan values are the same.
"""
import math

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _device, _lib


def _operand(x, shape):
    """(data, offsets, host offsets): x as a contiguous float64 CUDA tensor in its own (unbroadcast) shape, and the
    int64 element offset of each of the broadcast shape's rows in it (on the device and as a NumPy array)."""
    lead, n = shape[:-1], shape[-1]
    x = x.reshape((1,) * (len(shape) - x.dim()) + tuple(x.shape))
    if x.shape[-1] != n:                      # a broadcast last axis is materialised (one sample per row)
        x = x.expand(*x.shape[:-1], n)
    x = x.contiguous()
    own = tuple(x.shape[:-1])
    offsets = np.broadcast_to(np.arange(math.prod(own), dtype=np.int64).reshape(own) * n, lead).reshape(-1)
    offsets = np.ascontiguousarray(offsets)
    return x, _device.to_device(offsets), offsets


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
    _lib.load()
    lead, n = shape[:-1], shape[-1]
    rows = math.prod(lead)
    if rows:
        rd, ro, ro_host = _operand(_device.to_device(r), shape)
        ed, eo, eo_host = _operand(_device.to_device(e), shape)
        out = _SiSdr.apply(rd, ed, ro, eo, ro_host, eo_host, lead, n)
    else:
        out = _device.empty(lead, torch.float64)
    if not like_numpy:
        return out
    v = out.cpu().numpy()
    return np.float64(v) if v.ndim == 0 else v


def _row_table(offsets, n, own_rows):
    """(start, index) on the device: the rows that read own row u of an operand are index[start[u]:start[u + 1]], in
    increasing row order."""
    own = offsets // n
    index = np.argsort(own, kind='stable').astype(np.int64)
    start = np.concatenate([[0], np.cumsum(np.bincount(own, minlength=own_rows))]).astype(np.int64)
    return _device.to_device(start), _device.to_device(index)


class _SiSdr(torch.autograd.Function):
    """reference / estimation in their own shapes (float64 CUDA tensors) and their row offsets -> SI-SDR (lead) by
    pbb_si_sdr; backward pbb_si_sdr_backward."""

    @staticmethod
    def forward(ctx, rd, ed, ro, eo, ro_host, eo_host, lead, n):
        lib = _lib.load()
        rows = math.prod(lead)
        out = _device.empty(lead, torch.float64)
        nbytes = lib.pbb_si_sdr_workspace_bytes(rows, n)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
        _device.call('pbb_si_sdr', rd if n else None, ed if n else None, ro, eo, rows, n, ws, nbytes, out)
        # the row tables of the backward are built here, where a host-to-device copy may synchronise
        tables = [_row_table(off, n, x.numel() // n) if need and n else (None, None)
                  for need, off, x in zip(ctx.needs_input_grad[:2], (ro_host, eo_host), (rd, ed))]
        ctx.save_for_backward(rd, ed, ro, eo)
        ctx.args = (rows, n, tables)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        rd, ed, ro, eo = ctx.saved_tensors
        rows, n, ((rs, ri), (es, ei)) = ctx.args
        need_r, need_e = ctx.needs_input_grad[:2]
        gr = torch.zeros_like(rd) if need_r else None
        ge = torch.zeros_like(ed) if need_e else None
        if n and (need_r or need_e):
            lib = _lib.load()
            g = grad.to(torch.float64).contiguous()
            nbytes = lib.pbb_si_sdr_backward_workspace_bytes(rows, n)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=rd.device)
            _device.call('pbb_si_sdr_backward', rd, ed, ro, eo, rows, n, g, rd.numel() // n, rs, ri, ed.numel() // n,
                         es, ei, ws, nbytes, gr, ge)
        return gr, ge, None, None, None, None, None, None
