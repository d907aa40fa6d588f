"""BSS Eval, ``mir_eval_sources`` of pb_bss/evaluation/module_mir_eval.py, on the device, with the reference's
signature, return tuple / dict, shapes and errors.

The reference wraps mir_eval.separation.bss_eval_sources (BSS Eval v3: 512-tap time-invariant distortion filters;
Vincent, Gribonval and Fevotte, IEEE TASLP 14(4), 2006) and, for K + 1 estimates, its own
``_bss_eval_sources_and_noise``.  Here every item of a batch runs through one pass per step (include/pbb.h,
pbb_bss_eval): fp64 lag correlations on the tensor cores, one LU with partial pivoting of the order-512 K system per
item (and one per diagonal block), the projections as 512-tap convolutions, and the energy ratios of the explicit
residual signals.  Results are bitwise reproducible and an item's values do not depend on the rest of the batch.

Documented differences from the reference:
  - an all-zero reference or estimate raises ValueError on every path (the reference's K + 1 path would fall
    through to lstsq instead);
  - K <= 8 (N = 512 K <= 4096) and 1 <= T <= 2^22; larger inputs raise ValueError;
  - an exactly zero LU pivot (mir_eval would switch to lstsq) or a non-finite sample raises ValueError naming the
    batch item.
"""
import numpy as np
import torch

from .. import _device, _lib

FILTER_LENGTH = 512           # PBB_BSS_EVAL_FILTER
MAX_SOURCES = 8               # PBB_BSS_EVAL_MAX_SOURCES
MAX_SAMPLES = 1 << 22         # PBB_BSS_EVAL_MAX_SAMPLES
MAX_GROUP = 65535             # PBB_BSS_EVAL_MAX_GROUP
WORKSPACE_BYTES = 1 << 30     # items run in groups whose workspace stays under this (one item at least)

_FLAGS = ((1, 'an all-zero reference or estimate'), (2, 'a non-finite sample'),
          (4, 'an exactly singular system (zero LU pivot)'))


def _status_error(s):
    what = ' and '.join(text for bit, text in _FLAGS if s & bit)
    raise ValueError(f'mir_eval_sources: batch item {(s >> 3) - 1}: {what}')


def _is_complex(x):
    return x.is_complex() if _device.is_tensor(x) else np.iscomplexobj(x)


def _check(reference, estimation, compute_permutation):
    """(K, E, middle shape, T) after the reference's and mir_eval's shape checks."""
    rs, es = tuple(reference.shape), tuple(estimation.shape)
    if len(rs) == 2:
        assert len(es) == 2, es
        assert rs[1] == es[1], (rs, es)
    elif len(rs) >= 3:
        assert rs[1:] == es[1:], (rs, es)
    else:
        raise ValueError(f'Strange input shape: {rs}')
    K, E, T = rs[0], es[0], rs[-1]
    if E == K + 1:
        if not compute_permutation:
            raise NotImplementedError(compute_permutation, 'with K + 1')
    elif E != K:
        raise ValueError(f'Shapes do not fit: {rs} vs. {es}')
    if _is_complex(reference) or _is_complex(estimation):
        raise TypeError('mir_eval_sources of real signals, got complex input')
    if not 1 <= K <= MAX_SOURCES:
        raise ValueError(f'mir_eval_sources supports 1 to {MAX_SOURCES} references, got {K}')
    if not 1 <= T <= MAX_SAMPLES:
        raise ValueError(f'mir_eval_sources supports 1 to {MAX_SAMPLES} samples, got {T}')
    middle = rs[1:-1]
    if int(np.prod(middle, dtype=np.int64)) == 0:
        raise ValueError(f'mir_eval_sources of an empty batch: {rs}')
    return K, E, middle, T


def _stack(reference, estimation, K, E, T):
    """(items, K + E, T) float64 CUDA tensor: per item the references, then the estimates."""
    parts = []
    for x, n in ((reference, K), (estimation, E)):
        x = _device.to_device(x)
        x = x if x.dtype == torch.float64 else x.to(torch.float64)
        parts.append(x.reshape(n, -1, T).transpose(0, 1))
    return torch.cat(parts, dim=1).contiguous()


def _evaluate(x, K, E, T, compute_permutation, pairs=False):
    """sdr, sir, sar (items, K), selection (items, K) int64 or None, pairs (items, 3, E, K) or None, on the device;
    the status is checked (deferred inside ``deferred_status``)."""
    lib = _lib.load()
    items = x.shape[0]
    per_item = lib.pbb_bss_eval_workspace_bytes(1, K, E, T)
    group = int(max(1, min(items, MAX_GROUP, WORKSPACE_BYTES // per_item)))
    nbytes = lib.pbb_bss_eval_workspace_bytes(group, K, E, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    sdr, sir, sar = (_device.empty((items, K), torch.float64) for _ in range(3))
    selection = _device.empty((items, K), torch.int64) if compute_permutation else None
    pm = _device.empty((items, 3, E, K), torch.float64) if pairs else None
    status = torch.zeros(1, dtype=torch.int64, device=x.device)
    _device.call('pbb_bss_eval', x, items, K, E, T, int(bool(compute_permutation)), group, ws, nbytes, sdr, sir, sar,
                 selection, pm, status)
    _device.check_status(status, _status_error)
    return sdr, sir, sar, selection, pm


def mir_eval_sources(reference, estimation, return_dict=False, compute_permutation=True):
    """pb_bss.evaluation.mir_eval_sources: SDR, SIR, SAR (and the selection) of the estimates against the references.

    reference (K, T) or (K, ..., T); estimation (K, ...) or (K + 1, ...) with the same trailing shape.  Returns
    ``sdr, sir, sar, selection`` (or without the selection when compute_permutation is False), or a dict with those
    keys when return_dict; each of shape (K, ...).  selection[k] is the estimate picked for reference k: the first
    maximiser of the mean SIR in itertools.permutations order (int64).  E = K + 1 needs compute_permutation
    (NotImplementedError otherwise).

    NumPy in gives NumPy out; a CUDA tensor in gives float64 (selection int64) CUDA tensors out, enqueued on the
    current stream -- the only host synchronisation is the read of the status word, which ``deferred_status()``
    postpones to the end of its block.  float32 and integer input are computed in fp64; complex input raises
    TypeError.  Shape errors follow the reference (AssertionError / ValueError); an all-zero reference or estimate,
    a non-finite sample or an exactly singular system raises ValueError naming the batch item."""
    K, E, middle, T = _check(reference, estimation, compute_permutation)
    like_numpy = not (_device.is_tensor(reference) or _device.is_tensor(estimation))
    x = _stack(reference, estimation, K, E, T)
    sdr, sir, sar, selection, _ = _evaluate(x, K, E, T, compute_permutation)
    out = [v.reshape(*middle, K).movedim(-1, 0) for v in (sdr, sir, sar)]
    if compute_permutation:
        out.append(selection.reshape(*middle, K).movedim(-1, 0))
    if like_numpy:
        out = [np.ascontiguousarray(v.cpu().numpy()) for v in out]
    if return_dict:
        return dict(zip(('sdr', 'sir', 'sar', 'selection'), out))
    return tuple(out)
