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

``wpe_step`` is one WPE iteration with the caller's inverse power (nara_wpe's TensorFlow ``wpe_step`` and ESPnet's
``wpe_one_iteration`` compute the same; the contract is restated in ``oracle/wpe_autograd_oracle.py``), the building
block of DNN-WPE, where a network estimates the power.  ``wpe`` (through every iteration and its weights),
``wpe_step`` (Y and the inverse power), ``get_power`` and ``get_power_inverse`` are differentiable for CUDA tensors
that require grad: the forward runs the same kernels, so outputs are bitwise those of a call without grad, and the
backward passes are the fp64 device kernels of pbb_wpe_backward and pbb_wpe_power_backward (closed forms in
include/pbb.h; fixed-order sums, no atomics, no host synchronisation).  Gradients come back in the input's dtype,
repeated backward calls are bitwise identical and double backward raises.  A bin whose R has an exactly zero pivot
(the forward took lstsq) or holds a non-finite value gets NaN gradients in that bin only.  NumPy input and the online
functions return results without a graph.

Documented differences from nara_wpe:
  - real input raises TypeError (nara_wpe would compute in the real domain);
  - taps * D > 96 or D > 30 raises NotImplementedError (wpe, get_power, get_power_inverse);
  - sums over frames run in a fixed order, not NumPy's pairwise order.

Frame-online WPE: ``online_wpe_step`` and ``get_power_online`` keep nara_wpe's signatures; ``online_wpe`` (not in
nara_wpe) runs the step over a whole stream (T, ..., D) in one launch and returns the state to continue it, so a
one-frame chunk is a streaming step.  The contract is restated in ``oracle/wpe_online_oracle.py``.  One CTA per bin
keeps the inverse correlation Q in registers over all frames.  nara_wpe's ``OnlineWPE`` class is not provided: its
power smoothing and buffer handling are not part of the restated contract, and ``online_wpe`` with ``state`` covers
streaming.  Differences from nara_wpe: alpha outside (0, 1] raises ValueError (nara_wpe does not check it); the
division by alpha is a multiplication by 1 / alpha; the taps + delay + 1 frames of the buffer must fit the shared
memory of a CTA (about 1500 frames at D = 8, 350 at D = 30), else NotImplementedError.
"""
import collections
import math

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _device, _lib

MAX_N = 96                      # PBB_WPE_MAX_N: taps * D
MAX_D = 30                      # PBB_WPE_MAX_D: channels
MAX_GROUP = 65535               # PBB_WPE_MAX_GROUP
WORKSPACE_BYTES = 1 << 30       # bins run in groups whose workspace stays under this (one bin at least)
NONFINITE, LSTSQ = 1, 2         # PBB_WPE_NONFINITE, PBB_WPE_LSTSQ

GRAD_INVERSE, GRAD_PLAIN, GRAD_INVERSE_ALL = 0, 1, 2   # PBB_WPE_GRAD_*

__all__ = ['wpe', 'wpe_step', 'get_power', 'get_power_inverse', 'build_y_tilde', 'online_wpe_step',
           'get_power_online', 'online_wpe', 'OnlineWPEState']


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
    group = _group(lib.pbb_wpe_workspace_bytes(1, D, T, taps, delay, valid), bins)
    nbytes = lib.pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
    status = torch.zeros(1, dtype=torch.int32, device=y.device)
    _device.call('pbb_wpe', y, _device.complex_dtype_code(y), bins, D, T, *ys, out, *os_, taps, delay, iterations,
                 _context(psd_context), valid, group, ws, nbytes, status)
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


def _needs_graph(*ts):
    return torch.is_grad_enabled() and any(_device.is_tensor(t) and t.requires_grad for t in ts)


def _group(per_bin, bins):
    return int(max(1, min(bins, MAX_GROUP, WORKSPACE_BYTES // per_bin)))


def _backward_workspace(bins, D, T, taps, delay, valid):
    """(group, workspace) of pbb_wpe_backward"""
    lib = _lib.load()
    group = _group(lib.pbb_wpe_backward_workspace_bytes(1, D, T, taps, delay, valid), bins)
    nbytes = lib.pbb_wpe_backward_workspace_bytes(group, D, T, taps, delay, valid)
    return group, torch.empty(nbytes, dtype=torch.uint8, device=_device.device())


def _power_backward(y, ys, G, taps, delay, c, mode, gin, xbar):
    """pbb_wpe_power_backward: xbar (bins, D, T) complex128 += the power chain's gradient of y (G: x = y - G^H Yt)"""
    bins, D, T = xbar.shape
    lib = _lib.load()
    nbytes = lib.pbb_wpe_power_backward_workspace_bytes(bins, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xbar.device)
    _device.call('pbb_wpe_power_backward', y, _device.complex_dtype_code(y), bins, D, T, *ys, G, taps, delay, c, mode,
                 gin, xbar, ws, nbytes)


def _step_backward(y, ys, w, G, xbar, ybar, taps, delay, valid):
    """pbb_wpe_backward: ybar += Y's gradient of one step; returns the weights' gradient (bins, T) float64"""
    bins, D, T = xbar.shape
    group, ws = _backward_workspace(bins, D, T, taps, delay, valid)
    wbar = torch.empty((bins, T), dtype=torch.float64, device=xbar.device)
    _device.call('pbb_wpe_backward', y, _device.complex_dtype_code(y), bins, D, T, *ys, w, G, xbar, taps, delay, valid,
                 ybar, wbar, group, ws, ws.numel())
    return wbar


def _grad_in(grad, bins, D, T):
    return grad.to(torch.complex128).contiguous().reshape(bins, D, T)


class _Wpe(torch.autograd.Function):
    """Y (..., D, T) complex on the device -> X by pbb_wpe_forward, which also keeps every iteration's G_i and w_i;
    backward: pbb_wpe_backward per stage from the last to the first, each stage's weight gradient through
    pbb_wpe_power_backward into the previous stage's output (into Y for the first stage)."""

    @staticmethod
    def forward(ctx, Y, taps, delay, iterations, c, valid):
        D, T = Y.shape[-2], Y.shape[-1]
        bins = int(np.prod(Y.shape[:-2], dtype=np.int64))
        lib = _lib.load()
        y, ys = _layout(Y)
        out, os_ = _layout(torch.empty_like(y))
        group = _group(lib.pbb_wpe_workspace_bytes(1, D, T, taps, delay, valid), bins)
        nbytes = lib.pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
        status = torch.zeros(1, dtype=torch.int32, device=y.device)
        G = torch.empty((iterations, bins, taps * D, D), dtype=torch.complex128, device=y.device)
        w = torch.empty((iterations, bins, T), dtype=torch.float64, device=y.device)
        _device.call('pbb_wpe_forward', y, _device.complex_dtype_code(y), bins, D, T, *ys, out, *os_, taps, delay,
                     iterations, c, valid, group, ws, nbytes, status, G if iterations else None,
                     w if iterations else None)
        ctx.save_for_backward(y, G, w)
        ctx.args = (ys, taps, delay, iterations, c, valid, Y.shape, Y.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        y, G, w = ctx.saved_tensors
        ys, taps, delay, iterations, c, valid, shape, dtype = ctx.args
        D, T = shape[-2], shape[-1]
        bins = int(np.prod(shape[:-2], dtype=np.int64))
        xbar = _grad_in(grad, bins, D, T)
        if iterations == 0:
            return xbar.reshape(shape).to(dtype), None, None, None, None, None
        ybar = torch.zeros((bins, D, T), dtype=torch.complex128, device=y.device)
        for i in range(iterations - 1, -1, -1):
            wbar = _step_backward(y, ys, w[i], G[i], xbar, ybar, taps, delay, valid)
            xprev = ybar if i == 0 else torch.zeros_like(ybar)
            _power_backward(y, ys, G[i - 1] if i else None, taps, delay, c, GRAD_INVERSE, wbar, xprev)
            xbar = xprev
        return ybar.reshape(shape).to(dtype), None, None, None, None, None


def wpe(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode='full', inplace=False):
    """nara_wpe.wpe.wpe (wpe_v8): the dereverberated (..., D, T) STFT of Y (..., D, T).

    taps: filter length in frames, delay: prediction delay, iterations: re-estimations of the power,
    psd_context: frames on each side of the power's moving mean (inf: the mean over all frames),
    statistics_mode: 'full' (every frame) or 'valid' (frames t >= delay + taps - 1) for the correlations,
    inplace: write X into Y and return Y (raises for a tensor that requires grad).
    Differentiable with respect to a CUDA tensor Y that requires grad (see the module's docstring)."""
    _check_args(Y, taps, delay, iterations, psd_context, statistics_mode)
    if _needs_graph(Y):
        if inplace:
            raise RuntimeError('wpe(inplace=True) on a tensor that requires grad: an in-place operation would '
                               'overwrite the input its gradient needs')
        Yd, _ = _prepare(Y, 'wpe')
        if Yd.numel() == 0:
            return Yd.clone()
        return _Wpe.apply(Yd, taps, delay, iterations, _context(psd_context), int(statistics_mode == 'valid'))
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


def _power_launch(x, c, inverse):
    """(out (..., T) float64, x after _layout, its strides) by pbb_wpe_power"""
    D, T = x.shape[-2], x.shape[-1]
    lead = tuple(x.shape[:-2])
    bins = int(np.prod(lead, dtype=np.int64))
    out = _device.empty(lead + (T,), torch.float64)
    xs = None
    if bins and T:
        lib = _lib.load()
        x, xs = _layout(x)
        nbytes = lib.pbb_wpe_power_workspace_bytes(bins, T)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        _device.call('pbb_wpe_power', x, _device.complex_dtype_code(x), bins, D, T, *xs, c, int(inverse), out, ws,
                     nbytes)
    return out, x, xs


class _Power(torch.autograd.Function):
    """get_power / get_power_inverse of x (..., D, T) on the device by pbb_wpe_power; backward
    pbb_wpe_power_backward (GRAD_PLAIN / GRAD_INVERSE_ALL)."""

    @staticmethod
    def forward(ctx, x, c, inverse):
        out, xl, xs = _power_launch(x, c, inverse)
        ctx.save_for_backward(xl)
        ctx.args = (xs, c, inverse, x.shape, x.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        xl, = ctx.saved_tensors
        xs, c, inverse, shape, dtype = ctx.args
        D, T = shape[-2], shape[-1]
        bins = int(np.prod(shape[:-2], dtype=np.int64))
        xbar = torch.zeros((bins, D, T), dtype=torch.complex128, device=xl.device)
        if bins and T:
            g = grad.to(torch.float64).contiguous().reshape(bins, T)
            _power_backward(xl, xs, None, 1, 0, c, GRAD_INVERSE_ALL if inverse else GRAD_PLAIN, g, xbar)
        return xbar.reshape(shape).to(dtype), None, None


class _WpeStep(torch.autograd.Function):
    """Y (..., D, T) complex and w (bins, T) float64 on the device -> X by pbb_wpe_step, which also keeps G;
    backward pbb_wpe_backward."""

    @staticmethod
    def forward(ctx, Y, w, taps, delay, valid):
        D, T = Y.shape[-2], Y.shape[-1]
        bins = w.shape[0]
        lib = _lib.load()
        y, ys = _layout(Y)
        out, os_ = _layout(torch.empty_like(y))
        group = _group(lib.pbb_wpe_workspace_bytes(1, D, T, taps, delay, valid), bins)
        nbytes = lib.pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
        status = torch.zeros(1, dtype=torch.int32, device=y.device)
        G = torch.empty((bins, taps * D, D), dtype=torch.complex128, device=y.device)
        _device.call('pbb_wpe_step', y, _device.complex_dtype_code(y), bins, D, T, *ys, w, w.stride(0), w.stride(1),
                     out, *os_, taps, delay, valid, group, ws, nbytes, status, G)
        ctx.save_for_backward(y, w, G)
        ctx.args = (ys, taps, delay, valid, Y.shape, Y.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        y, w, G = ctx.saved_tensors
        ys, taps, delay, valid, shape, dtype = ctx.args
        D, T = shape[-2], shape[-1]
        bins = w.shape[0]
        ybar = torch.zeros((bins, D, T), dtype=torch.complex128, device=y.device)
        wc = w.contiguous()
        wbar = _step_backward(y, ys, wc, G, _grad_in(grad, bins, D, T), ybar, taps, delay, valid)
        return ybar.reshape(shape).to(dtype), wbar, None, None, None


def wpe_step(Y, inverse_power, taps=10, delay=3, statistics_mode='full'):
    """One WPE iteration with the caller's weights: X (..., D, T) for Y (..., D, T) complex and inverse_power
    (..., T) real (float32 or float64, exactly Y's leading shape):
        R = sum_S w_t Yt_t Yt_t^H, P = sum_S w_t Yt_t Y_t^H, G = stable_solve(R, P), X = Y - G^H Yt
    with Yt = build_y_tilde(Y, taps, delay) and S as in ``wpe`` (the same limits and errors).  This is the step of
    DNN-WPE, where a network estimates the power; differentiable with respect to Y and inverse_power for CUDA
    tensors that require grad."""
    _check_args(Y, taps, delay, 1, 0, statistics_mode)
    if len(Y.shape) < 2:
        raise ValueError(f'wpe_step needs shape (..., D, T), got {tuple(Y.shape)}')
    want = tuple(Y.shape[:-2]) + (Y.shape[-1],)
    if tuple(inverse_power.shape) != want:
        raise ValueError(f'inverse_power must have shape {want}, got {tuple(inverse_power.shape)}')
    if _device.is_tensor(inverse_power):
        ok = inverse_power.dtype in (torch.float32, torch.float64)
    else:
        ok = np.asarray(inverse_power).dtype in (np.float32, np.float64)
    if not ok:
        raise ValueError(f'inverse_power must be float32 or float64, got {inverse_power.dtype}')
    Yd, like_numpy = _prepare(Y, 'wpe_step')
    w = inverse_power if _device.is_tensor(inverse_power) else torch.from_numpy(np.asarray(inverse_power))
    w = w.to(device=Yd.device, dtype=torch.float64)
    if Yd.numel() == 0:
        X = Yd.clone()
    else:
        bins, T = int(np.prod(Yd.shape[:-2], dtype=np.int64)), Yd.shape[-1]
        X = _WpeStep.apply(Yd, w.reshape(bins, T), taps, delay, int(statistics_mode == 'valid'))
    return _device.to_host(X, like_numpy)


def _power(signal, psd_context, inverse, graph=True):
    x, like_numpy = _prepare(signal, 'get_power_inverse' if inverse else 'get_power')
    c = _context(psd_context)
    D = x.shape[-2]
    if D > MAX_D:
        raise NotImplementedError(f'get_power supports D <= {MAX_D}, got D = {D}')
    if graph and _needs_graph(x):
        return _Power.apply(x, c, inverse)
    return _device.to_host(_power_launch(x, c, inverse)[0], like_numpy)


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
        _device.call('pbb_wpe_build_y_tilde', y, _device.complex_dtype_code(y), bins, D, T, *ys, taps, delay, out)
    return _device.to_host(out, like_numpy)


OnlineWPEState = collections.namedtuple('OnlineWPEState', ['history', 'inv_cov', 'filter_taps'])
OnlineWPEState.__doc__ = """State of ``online_wpe`` in nara_wpe's layouts: history (taps + delay, ..., D) in Y's dtype, the last
frames of the stream; inv_cov (..., n, n) and filter_taps (..., n, D) complex128, n = taps D, window index d taps + k."""

ONLINE_MAX_SMEM = 232448        # PBB_WPE_ONLINE_MAX_SMEM


def get_power_online(signal):
    """nara_wpe.wpe.get_power_online: (...,) float64, the mean over D and T of |signal (..., D, T)|^2, i.e.
    get_power(signal, psd_context=inf)[..., 0]."""
    if signal.shape[-1] == 0:
        raise ValueError('get_power_online needs at least one frame')
    return _power(signal, math.inf, False, graph=False)[..., 0]


def _check_online(taps, delay, alpha, D):
    if taps < 1:
        raise ValueError(f'taps must be >= 1, got {taps}')
    if delay < 0:
        raise ValueError(f'delay must be >= 0, got {delay}')
    if not 0.0 < float(alpha) <= 1.0:
        raise ValueError(f'alpha must be in (0, 1], got {alpha}')
    if taps * D > MAX_N or D > MAX_D:
        raise NotImplementedError(f'online WPE supports taps * D <= {MAX_N} and D <= {MAX_D}, got taps = {taps}, '
                                  f'D = {D}')
    if _lib.load().pbb_wpe_online_smem_bytes(D, taps, delay) > ONLINE_MAX_SMEM:
        raise NotImplementedError(f'online WPE keeps taps + delay + 1 frames of D channels in shared memory; '
                                  f'taps = {taps}, delay = {delay}, D = {D} do not fit')


def _frames(t):
    """(frames, ..., D) device tensor -> (..., D, frames) view, or one copy, and its (bin, d, t) element strides."""
    return _layout(t.movedim(0, -1))


def _state_tensor(x, shape, what):
    x = x if _device.is_tensor(x) else torch.from_numpy(np.asarray(x))
    if tuple(x.shape) != tuple(shape):
        raise ValueError(f'{what} must have shape {tuple(shape)}, got {tuple(x.shape)}')
    return x.to(device=_device.device(), dtype=torch.complex128).contiguous()


def _online(y, hist, power, Q, G, taps, delay, alpha):
    """Launch pbb_wpe_online.  y (T, ..., D) and hist (taps + delay, ..., D) device tensors of one complex dtype (hist
    None: zeros), power (...) float64 or None, Q, G contiguous complex128 or None.  -> (Z like y, Q', G')."""
    T, lead, D = y.shape[0], tuple(y.shape[1:-1]), y.shape[-1]
    bins = int(np.prod(lead, dtype=np.int64))
    n = taps * D
    Z = torch.empty_like(y, memory_format=torch.contiguous_format)
    Qo = _device.empty(lead + (n, n), torch.complex128)
    Go = _device.empty(lead + (n, D), torch.complex128)
    if bins == 0:
        return Z, Qo, Go
    yv, ys = _frames(y) if T else (y, (0, 0, 0))
    zv, zs = _frames(Z) if T else (Z, (0, 0, 0))
    hv, hs = _frames(hist) if hist is not None else (None, (0, 0, 0))
    _device.call('pbb_wpe_online', yv if T else None, _device.complex_dtype_code(y), bins, D, T, *ys, hv, *hs, power, Q,
                 G, zv if T else None, *zs, Qo, Go, taps, delay, float(alpha))
    return Z, Qo, Go


def _complex_dtype(x):
    """torch complex dtype of a real or complex array: complex64 for single precision, else complex128."""
    single = (x.dtype in (torch.float32, torch.complex64) if _device.is_tensor(x)
              else np.asarray(x).dtype in (np.float32, np.complex64))
    return torch.complex64 if single else torch.complex128


def online_wpe_step(input_buffer, power_estimate, inv_cov, filter_taps, alpha, taps, delay):
    """nara_wpe.wpe.online_wpe_step: one frame of recursive least-squares WPE per bin.

    input_buffer (taps + delay + 1, ..., D) complex, the last frame the current one; power_estimate (...) lambda;
    inv_cov (..., n, n) Q and filter_taps (..., n, D) G, n = taps D, window index d taps + k (real Q, G are promoted
    to complex).  Returns (prediction (..., D) in input_buffer's dtype, inv_cov_k, filter_taps_k) with
        pred = y_t - G^H w,  k = Q w / (alpha lambda + w^H Q w),  Q' = (Q - k w^H Q) / alpha,  G' = G + k pred^H;
    Q' and G' are complex64 where Q, G are single precision, else complex128."""
    if len(input_buffer.shape) < 3:
        raise ValueError(f'input_buffer needs shape (taps + delay + 1, ..., D), got {tuple(input_buffer.shape)}')
    L, lead, D = input_buffer.shape[0], tuple(input_buffer.shape[1:-1]), input_buffer.shape[-1]
    _check_online(taps, delay, alpha, D)
    if L != taps + delay + 1:
        raise ValueError(f'input_buffer needs taps + delay + 1 = {taps + delay + 1} frames, got {L}')
    n = taps * D
    if tuple(power_estimate.shape) != lead:
        raise ValueError(f'power_estimate must have shape {lead}, got {tuple(power_estimate.shape)}')
    qdt, gdt = _complex_dtype(inv_cov), _complex_dtype(filter_taps)
    buf, like_numpy = _prepare(input_buffer, 'online_wpe_step')
    Q = _state_tensor(inv_cov, lead + (n, n), 'inv_cov')
    G = _state_tensor(filter_taps, lead + (n, D), 'filter_taps')
    p = power_estimate if _device.is_tensor(power_estimate) else torch.from_numpy(np.asarray(power_estimate))
    p = p.to(device=buf.device, dtype=torch.float64).contiguous()
    Z, Qo, Go = _online(buf[L - 1:], buf[:L - 1], p, Q, G, taps, delay, alpha)
    return (_device.to_host(Z[0], like_numpy), _device.to_host(Qo.to(qdt), like_numpy),
            _device.to_host(Go.to(gdt), like_numpy))


def online_wpe(Y, taps=10, delay=2, alpha=0.9999, state=None):
    """Frame-online WPE over a whole stream: ``online_wpe_step`` for every frame of Y (T, ..., D) (frames first;
    an STFT X (D, T, F) passes as ``X.transpose(1, 2, 0)``), with lambda = the mean of |.|^2 over the D channels and
    the taps + delay + 1 frames of the step's buffer.  Returns (Z (T, ..., D) in Y's dtype, OnlineWPEState).
    state None starts from taps + delay zero frames, Q = I and G = 0; passing the returned state continues the
    stream, and any split of a stream gives bitwise the same Z and state as one call."""
    if len(Y.shape) < 2:
        raise ValueError(f'online_wpe needs Y of shape (T, ..., D), got {tuple(Y.shape)}')
    T, lead, D = Y.shape[0], tuple(Y.shape[1:-1]), Y.shape[-1]
    _check_online(taps, delay, alpha, D)
    n, H = taps * D, taps + delay
    y, like_numpy = _prepare(Y, 'online_wpe')
    if state is None:
        hist, Q, G = None, None, None
    else:
        h = state.history if _device.is_tensor(state.history) else torch.from_numpy(np.asarray(state.history))
        if tuple(h.shape) != (H,) + lead + (D,):
            raise ValueError(f'state.history must have shape {(H,) + lead + (D,)}, got {tuple(h.shape)}')
        hist = h.to(device=y.device, dtype=y.dtype)
        Q = _state_tensor(state.inv_cov, lead + (n, n), 'state.inv_cov')
        G = _state_tensor(state.filter_taps, lead + (n, D), 'state.filter_taps')
    Z, Qo, Go = _online(y, hist, None, Q, G, taps, delay, alpha)
    if hist is None:
        hist = torch.zeros((H,) + lead + (D,), dtype=y.dtype, device=y.device)
    history = torch.cat([hist, y])[T:].clone()
    return (_device.to_host(Z, like_numpy),
            OnlineWPEState(*(_device.to_host(t, like_numpy) for t in (history, Qo, Go))))
