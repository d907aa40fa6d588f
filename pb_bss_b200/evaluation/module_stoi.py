"""STOI, the short-time objective intelligibility of pb_bss/evaluation/module_stoi.py, on the device, with the
reference's signature, broadcasting and return types, and ESTOI, its extended form:
``stoi(reference, estimation, sample_rate, extended=False)``.

The reference calls pystoi.stoi(x, y, fs_sig) (extended=False; Taal, Hendriks, Heusdens and Jensen, IEEE TASLP 19(7),
2011) on every pair of the broadcast leading dims.  Here every pair runs in one pass per step (include/pbb.h,
pbb_stoi): resample_poly to 10 kHz with Octave's Kaiser filter, silent-frame removal 40 dB below the loudest frame
of the reference, the 512-point STFT of the overlap-added kept frames, 15 one-third octave bands from 150 Hz, and
the clipped correlations of 30-frame segments.  fp64, bitwise reproducible, and a pair's value does not depend on
the rest of the batch.

``extended=True`` gives ESTOI (Jensen and Taal, IEEE/ACM TASLP 24(11), 2016), pystoi's stoi(x, y, fs,
extended=True), the measure designed for modulated maskers such as competing talkers (pbb_estoi).  It shares every
step up to the band envelopes bit for bit, and the 1e-5 rule below 30 frames; each 15 x 30 segment is then
normalised per band over the frames and per frame over the bands, without clipping, and the value is the mean over
the segments of the normalised inner product / 30.

Documented differences from the reference:
  - integer and float32 input are computed in fp64 (at 10 kHz pystoi would frame float32 input in float32);
  - at most 2^22 samples per signal and 2^23 after resampling to 10 kHz; larger inputs raise ValueError, as does a
    signal with no 256-sample frame at 10 kHz (where NumPy raises an AxisError inside pystoi);
  - ESTOI: pystoi adds N(0, eps^2) noise before each normalisation step, this does not; a band or frame whose centred
    sum of squares is zero up to rounding (at most 2^-92 of its sum of squares) normalises to zeros, the expected
    value of pystoi's random term there.  Digital silence in the estimate reaches this: its all-zero bands, and the
    segments with one non-zero frame at either end of a silent stretch, whose frames are constant over the bands
    after the first step in exact arithmetic.

Gradients: STOI and ESTOI of CUDA tensors that require grad are differentiable with respect to both signals
(pbb_stoi_backward, which runs the forward's stages again and then one fp64 kernel per adjoint step; fixed-order sums,
no atomics, no host synchronisation).  The value is bitwise the same with or without a graph, gradients come back in
the input's dtype, repeated backward calls are bitwise identical, and double backward raises.  A broadcast operand's
gradient is torch's reduction of the broadcast.  The derivative's conventions:
  - the silent-frame selection is a constant of the graph (it depends on the reference only through a threshold): the
    gradient flows through the kept frames into both signals; a dropped frame's samples get only the contributions of
    the kept frames that overlap them;
  - the clipping min(c y, C x) passes the gradient to the operand the forward selected (x on a tie);
  - a zero norm (a band energy, ||y|| in the scale c, a centred norm in the correlation) has a zero subgradient, as
    torch.linalg.vector_norm: digital silence in the estimate gives finite, possibly very large, gradients;
  - ESTOI's rows and columns that the 2^-92 rule normalises to zeros pass no gradient;
  - rows on the 1e-5 path (fewer than 30 frames, including a non-finite reference) get zero gradients;
  - a non-finite estimate sample with a finite reference gives NaN gradients in its row only.
"""
import math
import warnings

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _device, _lib

FS = 10000                    # PBB_STOI_FS
FRAME = 256                   # PBB_STOI_FRAME
NFFT = 512                    # PBB_STOI_NFFT
BANDS = 15                    # PBB_STOI_BANDS
MIN_FREQ = 150
MAX_SAMPLES = 1 << 22         # PBB_STOI_MAX_SAMPLES
MAX_RESAMPLED = 1 << 23       # PBB_STOI_MAX_RESAMPLED
MAX_GROUP = 65535             # PBB_STOI_MAX_GROUP
WORKSPACE_BYTES = 1 << 30     # rows run in groups whose workspace stays under this (one row at least)
WARNING = ('Not enough STFT frames to compute intermediate intelligibility measure after removing silent frames. '
           'Returning 1e-5. Please check you wav files')

_tables = {}


def rates(sample_rate):
    """(up, down): 10000 / sample_rate in lowest terms."""
    g = math.gcd(FS, sample_rate)
    return FS // g, sample_rate // g


def resampled_length(n, sample_rate):
    up, down = rates(sample_rate)
    return -(-n * up // down)


def resample_filter(sample_rate):
    """The window pystoi passes to scipy.signal.resample_poly: Octave's Kaiser-windowed sinc for 10000 / sample_rate
    at 60 dB rejection, normalised to unit sum (pystoi.utils._resample_window_oct, the same NumPy calls)."""
    g = np.gcd(FS, sample_rate)
    p, q = FS / g, sample_rate / g
    stopband_cutoff_f = 1. / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = 60.0
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off_width))
    t = np.arange(-L, L + 1)
    ideal_filter = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    beta = 0.1102 * (rejection_db - 8.7)
    h = np.kaiser(2 * L + 1, beta) * ideal_filter
    return h / np.sum(h)


def polyphase_taps(sample_rate):
    """(taps (up, taps_per_phase), pre_remove): resample_poly's filter (the window times up after its n_pre_pad
    zeros) laid out per phase, taps[ph][m] = h[ph + m up], and its n_pre_remove."""
    up, down = rates(sample_rate)
    h = resample_filter(sample_rate).copy()
    h *= up
    half_len = (h.size - 1) // 2
    n_pre_pad = down - half_len % down
    h = np.concatenate((np.zeros(n_pre_pad), h))
    tpp = -(-h.size // up)
    table = np.zeros(up * tpp)
    table[:h.size] = h
    return np.ascontiguousarray(table.reshape(tpp, up).T), (half_len + n_pre_pad) // down


def window():
    return np.hanning(FRAME + 2)[1:-1]


def band_edges():
    """(15, 2) int32: the [lo, hi) rfft bins of the one-third octave bands (pystoi.utils.thirdoct)."""
    f = np.linspace(0, FS, NFFT + 1)[:NFFT // 2 + 1]
    k = np.arange(BANDS).astype(float)
    fl = MIN_FREQ * 2. ** ((2 * k - 1) / 6)
    fh = MIN_FREQ * 2. ** ((2 * k + 1) / 6)
    return np.array([[np.argmin((f - fl[i]) ** 2), np.argmin((f - fh[i]) ** 2)] for i in range(BANDS)],
                    dtype=np.int32)


def _device_tables(sample_rate):
    key = (sample_rate, _device.device())
    t = _tables.get(key)
    if t is None:
        up, down = rates(sample_rate)
        taps, pre_remove = polyphase_taps(sample_rate) if (up, down) != (1, 1) else (np.zeros((1, 1)), 0)
        k = 2 * np.pi * np.arange(NFFT) / NFFT
        t = _tables[key] = (_device.to_device(taps), taps.shape[1], pre_remove, _device.to_device(window()),
                            _device.to_device(band_edges()),
                            _device.to_device(np.stack([np.cos(k), np.sin(k)], axis=-1)))
    return t


def _is_complex(x):
    return x.is_complex() if _device.is_tensor(x) else np.iscomplexobj(x)


def _check(reference, estimation, sample_rate):
    """The broadcast shape, after the checks that raise before any device work."""
    if _is_complex(reference) or _is_complex(estimation):
        raise TypeError('stoi of real signals, got complex input')
    if isinstance(sample_rate, bool) or not isinstance(sample_rate, (int, np.integer)) or sample_rate < 1:
        raise ValueError(f'stoi needs a positive integer sample_rate, got {sample_rate!r}')
    shape = np.broadcast_shapes(tuple(np.shape(reference)), tuple(np.shape(estimation)))
    if len(shape) == 0:
        raise ValueError('stoi needs signals with at least one axis')
    n = shape[-1]
    if not 1 <= n <= MAX_SAMPLES:
        raise ValueError(f'stoi supports 1 to {MAX_SAMPLES} samples per signal, got {n}')
    L = resampled_length(n, int(sample_rate))
    if L <= FRAME:
        raise ValueError(f'stoi needs more than {FRAME} samples at {FS} Hz (one frame), got {L} from {n} samples '
                         f'at {sample_rate} Hz')
    if L > MAX_RESAMPLED:
        raise ValueError(f'stoi supports up to {MAX_RESAMPLED} samples at {FS} Hz, got {L}')
    return shape


def _operands(reference, estimation, shape):
    """x, y: (rows, n) contiguous CUDA tensors of one dtype, float32 if both are float32, else float64."""
    xs = [_device.to_device(v) for v in (reference, estimation)]
    dtype = torch.float32 if all(v.dtype == torch.float32 for v in xs) else torch.float64
    n = shape[-1]
    return [torch.broadcast_to(v.to(dtype), shape).reshape(-1, n).contiguous() for v in xs]


def _warn(status):
    def on_error(count):
        warnings.warn(f'{WARNING} ({count} signal(s); the first is row {int(status[1])} of the flattened batch)',
                      RuntimeWarning, stacklevel=4)
    return on_error


def _stages(x, y, sample_rate, stages=True, extended=False):
    """Every step on the device for x, y (rows, n): dict of value (rows,), STOI or with ``extended`` ESTOI, and with
    ``stages`` frames (rows, 2) int64 (K_r, M_r), resampled (rows, 2, L) (None at 10 kHz) and energies
    (rows, 2, 15, M_max), zero from M_r on.  The status is checked (deferred inside ``deferred_status``)."""
    lib = _lib.load()
    rows, n = x.shape
    up, down = rates(sample_rate)
    taps, tpp, pre_remove, win, bands, tw = _device_tables(sample_rate)
    L = resampled_length(n, sample_rate)
    m_max = len(range(0, L - FRAME, FRAME // 2)) - 1
    per_row = lib.pbb_stoi_workspace_bytes(1, n, up, down)
    group = int(max(1, min(rows, MAX_GROUP, WORKSPACE_BYTES // per_row)))
    nbytes = lib.pbb_stoi_workspace_bytes(group, n, up, down)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    value = _device.empty((rows,), torch.float64)
    status = torch.empty(2, dtype=torch.int64, device=x.device)
    out = dict(value=value)
    if stages:
        out['frames'] = _device.empty((rows, 2), torch.int64)
        out['resampled'] = _device.empty((rows, 2, L), torch.float64) if (up, down) != (1, 1) else None
        out['energies'] = torch.zeros((rows, 2, BANDS, m_max), dtype=torch.float64, device=x.device)
    name = 'pbb_estoi' if extended else 'pbb_stoi'
    _device.call(name, x, y, _lib.PBB_F32 if x.dtype == torch.float32 else _lib.PBB_F64, rows, n, up, down, taps, tpp,
                 pre_remove, win, bands, tw, group, ws, nbytes, value, out.get('frames'), out.get('resampled'),
                 out.get('energies'), status)
    _device.check_status(status[:1], _warn(status))
    return out


def _backward(x, y, sample_rate, extended, grad, need_x, need_y):
    """(grad_x, grad_y) float64 (rows, n), None where not needed, by pbb_stoi_backward; only enqueues work."""
    lib = _lib.load()
    rows, n = x.shape
    up, down = rates(sample_rate)
    taps, tpp, pre_remove, win, bands, tw = _device_tables(sample_rate)
    per_row = lib.pbb_stoi_backward_workspace_bytes(1, n, up, down, int(extended))
    group = int(max(1, min(rows, MAX_GROUP, WORKSPACE_BYTES // per_row)))
    nbytes = lib.pbb_stoi_backward_workspace_bytes(group, n, up, down, int(extended))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    gx = torch.empty((rows, n), dtype=torch.float64, device=x.device) if need_x else None
    gy = torch.empty((rows, n), dtype=torch.float64, device=x.device) if need_y else None
    g = grad.to(torch.float64).contiguous()
    _device.call('pbb_stoi_backward', x, y, _lib.PBB_F32 if x.dtype == torch.float32 else _lib.PBB_F64, rows, n, up,
                 down, taps, tpp, pre_remove, win, bands, tw, group, ws, nbytes, int(extended), g, gx, gy)
    return gx, gy


class _Stoi(torch.autograd.Function):
    """x, y (rows, n) contiguous CUDA tensors of one dtype -> STOI / ESTOI (rows,) float64 by pbb_stoi / pbb_estoi;
    backward pbb_stoi_backward, which recomputes the forward's stages from x and y."""

    @staticmethod
    def forward(ctx, x, y, sample_rate, extended):
        value = _stages(x, y, sample_rate, stages=False, extended=extended)['value']
        ctx.save_for_backward(x, y)
        ctx.args = (sample_rate, extended)
        return value

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        x, y = ctx.saved_tensors
        sample_rate, extended = ctx.args
        need_x, need_y = ctx.needs_input_grad[:2]
        gx, gy = _backward(x, y, sample_rate, extended, grad, need_x, need_y)
        return (gx.to(x.dtype) if need_x else None, gy.to(y.dtype) if need_y else None, None, None)


def stoi(reference, estimation, sample_rate, extended=False):
    """pb_bss.evaluation.stoi: the STOI of estimation against reference along the last axis, after broadcasting the
    two (NumPy's rules; ValueError if they do not broadcast).  1-D input gives an np.float64, n-D input an ndarray of
    the broadcast leading shape.  A CUDA tensor in (either argument) gives a float64 CUDA tensor of that shape (0-d
    for 1-D input), and the call only enqueues work on the current stream: the one host synchronisation is the read
    of the status word, which ``deferred_status()`` postpones to the end of its block.

    With ``extended`` true the value is ESTOI (pystoi's stoi(x, y, fs, extended=True); Jensen and Taal, 2016), with
    the same types, broadcasting, checks and warning.  Unlike pystoi, no random noise is added before its
    normalisations: a band or frame of a segment whose centred sum of squares is zero up to rounding, such as digital
    silence, normalises to zeros.

    A pair with fewer than 30 STFT frames after the silent-frame removal gives 1e-5 and a RuntimeWarning, as pystoi
    does.  float32 and integer input are computed in fp64; complex input raises TypeError; signals of more than 2^22
    samples, more than 2^23 at 10 kHz, or without one 256-sample frame at 10 kHz raise ValueError.

    CUDA tensors that require grad get a graph: the value is differentiable with respect to both signals (see the
    module's docstring for the conventions at the keep mask, the clip, zero norms and the 1e-5 rows)."""
    shape = _check(reference, estimation, sample_rate)
    sample_rate = int(sample_rate)
    like_numpy = not (_device.is_tensor(reference) or _device.is_tensor(estimation))
    lead = shape[:-1]
    if math.prod(lead) == 0:
        value = _device.empty(lead, torch.float64)
    else:
        x, y = _operands(reference, estimation, shape)
        value = _Stoi.apply(x, y, sample_rate, bool(extended)).reshape(lead)
    if not like_numpy:
        return value
    v = value.cpu().numpy()
    return np.float64(v) if v.ndim == 0 else v
