"""WPE dereverberation with the interface of nara_wpe.wpe on the device: ``from pb_bss_b200.wpe import wpe`` in place
of ``from nara_wpe.wpe import wpe``.

Weighted prediction error (T. Nakatani et al., IEEE TASLP 18(7), 2010; T. Yoshioka and T. Nakatani, IEEE TASLP
20(10), 2012) with nara_wpe's defaults and ``wpe_v8`` semantics; the contract is restated in
``oracle/wpe_oracle.py``.  Every leading index of Y (..., D, T) -- normally the frequency bin -- is an independent
problem.  Per bin and iteration the weighted correlations R (taps D x taps D) and P (taps D x D) are accumulated on
the FP64 tensor cores straight from Y (the delayed stack Yt is never stored), R G = P is solved by LU with partial
pivoting (np.linalg.solve's pivots; an exactly zero pivot takes np.linalg.lstsq's minimum-norm solution), and the
filter X = Y - G^H Yt is fused with the next iteration's power.  All arithmetic is fp64; sums run in a fixed order,
so repeated calls are bitwise identical.

NumPy in gives NumPy out; a CUDA tensor in gives a CUDA tensor out (in the input's strides where they are dense).
Any strides are accepted: a view whose leading dims do not collapse to one stride is copied once on the device.

Documented differences from nara_wpe:
  - real input raises TypeError (nara_wpe would compute in the real domain);
  - taps * D > 96 or D > 30 raises NotImplementedError (wpe, get_power, get_power_inverse);
  - sums over frames run in a fixed order, not NumPy's pairwise order.
"""
import math

import numpy as np
import torch

from . import _device, _lib

MAX_N = 96                      # PBB_WPE_MAX_N: taps * D
MAX_D = 30                      # PBB_WPE_MAX_D: channels
MAX_GROUP = 65535               # PBB_WPE_MAX_GROUP
WORKSPACE_BYTES = 1 << 30       # bins run in groups whose workspace stays under this (one bin at least)
NONFINITE, LSTSQ = 1, 2         # PBB_WPE_NONFINITE, PBB_WPE_LSTSQ

__all__ = ['wpe', 'get_power', 'get_power_inverse', 'build_y_tilde']


def _is_complex(x):
    return x.is_complex() if _device.is_tensor(x) else np.iscomplexobj(x)


def _context(psd_context):
    """psd_context -> the ABI's value: an integer >= 0, or -1 for inf."""
    c = float(psd_context)
    if math.isinf(c) and c > 0:
        return -1
    if not c >= 0:
        raise ValueError(f'psd_context must be >= 0 or inf, got {psd_context}')
    if c != int(c):
        raise ValueError(f'psd_context must be an integer or inf, got {psd_context}')
    return int(c)


def _prepare(Y, what):
    """(device tensor (..., D, T), like_numpy) for complex Y with at least two dims."""
    if not _is_complex(Y):
        raise TypeError(f'{what} needs a complex STFT, got {getattr(Y, "dtype", type(Y))}')
    if len(Y.shape) < 2:
        raise ValueError(f'{what} needs shape (..., D, T), got {tuple(Y.shape)}')
    like_numpy = not _device.is_tensor(Y)
    if like_numpy:
        Y = np.asarray(Y)
        if Y.dtype not in (np.complex64, np.complex128):
            Y = Y.astype(np.complex128)
        return _device.to_device(Y), True
    if Y.dtype not in (torch.complex64, torch.complex128):
        Y = Y.to(torch.complex128)
    if Y.device.type != 'cuda':
        Y = Y.to(_device.device())
    return Y, False


def _strides(t):
    """(bin, d, t) element strides of t (..., D, T), or None if the leading dims do not collapse to one stride."""
    shape, stride = t.shape[:-2], t.stride()[:-2]
    dims = [(n, s) for n, s in zip(shape, stride) if n != 1]
    for (n0, s0), (n1, s1) in zip(dims, dims[1:]):
        if s0 != s1 * n1:
            return None
    sb = dims[-1][1] if dims else 0
    return sb, t.stride(-2), t.stride(-1)


def _layout(t):
    """t and its (bin, d, t) strides, after at most one device-side copy."""
    s = _strides(t)
    if s is None:
        t = t.contiguous()
        s = _strides(t)
    return t, s


def _run(Y, taps, delay, iterations, psd_context, statistics_mode, inplace):
    """(X, status) for a device tensor Y; status is the PBB_WPE_* bits, read once after the last iteration."""
    D, T = Y.shape[-2], Y.shape[-1]
    bins = int(np.prod(Y.shape[:-2], dtype=np.int64))
    lib = _lib.load()
    y, ys = _layout(Y)
    if inplace:
        out, os_ = y, ys
    else:
        out = torch.empty_like(y)
        out, os_ = _layout(out)
    if bins == 0 or T == 0:
        if not inplace:
            out.copy_(y)
        return (Y if inplace else out), 0
    valid = int(statistics_mode == 'valid')
    per_bin = lib.pbb_wpe_workspace_bytes(1, D, T, taps, delay, valid)
    group = int(max(1, min(bins, MAX_GROUP, WORKSPACE_BYTES // per_bin)))
    nbytes = lib.pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
    status = torch.zeros(1, dtype=torch.int32, device=y.device)
    _lib.check(lib.pbb_wpe(_device.ptr(y), _device.complex_dtype_code(y), bins, D, T, *ys, _device.ptr(out), *os_,
                           taps, delay, iterations, _context(psd_context), valid, group, _device.ptr(ws), nbytes,
                           _device.ptr(status), _device.stream_ptr()), 'pbb_wpe')
    if inplace and out.data_ptr() != Y.data_ptr():
        Y.copy_(out)
        out = Y
    return out, int(status.item())


def _check_args(Y, taps, delay, iterations, psd_context, statistics_mode):
    if statistics_mode not in ('full', 'valid'):
        raise ValueError(f"statistics_mode must be 'full' or 'valid', got {statistics_mode!r}")
    if taps < 1:
        raise ValueError(f'taps must be >= 1, got {taps}')
    if delay < 0:
        raise ValueError(f'delay must be >= 0, got {delay}')
    if iterations < 0:
        raise ValueError(f'iterations must be >= 0, got {iterations}')
    _context(psd_context)
    if len(Y.shape) >= 2 and (taps * Y.shape[-2] > MAX_N or Y.shape[-2] > MAX_D):
        raise NotImplementedError(f'wpe supports taps * D <= {MAX_N} and D <= {MAX_D}, got taps = {taps}, '
                                  f'D = {Y.shape[-2]}')


def wpe(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode='full', inplace=False):
    """nara_wpe.wpe.wpe (wpe_v8): the dereverberated (..., D, T) STFT of Y (..., D, T).

    taps: filter length in frames, delay: prediction delay, iterations: re-estimations of the power,
    psd_context: frames on each side of the power's moving mean (inf: the mean over all frames),
    statistics_mode: 'full' (every frame) or 'valid' (frames t >= delay + taps - 1) for the correlations,
    inplace: write X into Y and return Y."""
    _check_args(Y, taps, delay, iterations, psd_context, statistics_mode)
    Yd, like_numpy = _prepare(Y, 'wpe')
    if like_numpy:
        X, _ = _run(Yd, taps, delay, iterations, psd_context, statistics_mode, False)
        X = X.cpu().numpy()
        if inplace:
            Y[...] = X
            return Y
        return X
    X, _ = _run(Yd, taps, delay, iterations, psd_context, statistics_mode, inplace and Yd is Y)
    if inplace and Yd is not Y:
        Y.copy_(X)
        return Y
    return X


def _power(signal, psd_context, inverse):
    x, like_numpy = _prepare(signal, 'get_power_inverse' if inverse else 'get_power')
    c = _context(psd_context)
    D, T = x.shape[-2], x.shape[-1]
    if D > MAX_D:
        raise NotImplementedError(f'get_power supports D <= {MAX_D}, got D = {D}')
    lead = tuple(x.shape[:-2])
    bins = int(np.prod(lead, dtype=np.int64))
    out = _device.empty(lead + (T,), torch.float64)
    if bins and T:
        lib = _lib.load()
        x, xs = _layout(x)
        nbytes = lib.pbb_wpe_power_workspace_bytes(bins, T)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        _lib.check(lib.pbb_wpe_power(_device.ptr(x), _device.complex_dtype_code(x), bins, D, T, *xs, c, int(inverse),
                                     _device.ptr(out), _device.ptr(ws), nbytes, _device.stream_ptr()), 'pbb_wpe_power')
    return _device.to_host(out, like_numpy)


def get_power(signal, psd_context=0):
    """nara_wpe.wpe.get_power: (..., T) float64, the mean over D of |signal|^2 per frame, averaged over the frames
    t - psd_context .. t + psd_context that exist (psd_context = inf: the mean over all frames).  Any number of
    leading indices; D <= 30."""
    return _power(signal, psd_context, False)


def get_power_inverse(signal, psd_context=0):
    """nara_wpe.wpe.get_power_inverse: 1 / maximum(get_power(signal), 1e-10 max), the max over the whole array."""
    return _power(signal, psd_context, True)


def build_y_tilde(Y, taps, delay):
    """nara_wpe.wpe.build_y_tilde: (..., taps D, T), row k D + d at frame t is Y[..., d, t - delay - k] (0 before the
    first frame), in Y's complex dtype."""
    if taps < 1:
        raise ValueError(f'taps must be >= 1, got {taps}')
    if delay < 0:
        raise ValueError(f'delay must be >= 0, got {delay}')
    y, like_numpy = _prepare(Y, 'build_y_tilde')
    D, T = y.shape[-2], y.shape[-1]
    lead = tuple(y.shape[:-2])
    bins = int(np.prod(lead, dtype=np.int64))
    out = _device.empty(lead + (taps * D, T), y.dtype)
    if bins and T:
        y, ys = _layout(y)
        _lib.check(_lib.load().pbb_wpe_build_y_tilde(_device.ptr(y), _device.complex_dtype_code(y), bins, D, T, *ys,
                                                     taps, delay, _device.ptr(out), _device.stream_ptr()),
                   'pbb_wpe_build_y_tilde')
    return _device.to_host(out, like_numpy)
