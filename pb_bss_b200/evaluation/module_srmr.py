"""SRMR, the speech-to-reverberation modulation energy ratio of pb_bss/evaluation/module_srmr.py, on the device, with
the reference's names, defaults, return types and errors: ``srmr(signal, sample_rate, n_cochlear_filters,
low_freq)`` and ``SRMR(signal, sample_rate, n, low_freq)``.

The steps and their quirks follow the reference: a VAD that compares |x| (an amplitude) with max|x|^2 / 1e5 and
removes the samples strictly between two above-threshold samples more than 0.05 sample_rate apart; normalisation to
zero mean and unit population std; the gammatone filterbank (pb_bss_b200.transform.gammatone); the Hilbert envelope
of every band over the row's own length N_r; eight second-order modulation band-pass filters per band from zero
state; the mean over frames (``segment_axis`` with end='pad': frames of int(sr / 1000) * 256 samples every
int(sr / 1000) * 64, zero-padded at the end) of the Hamming-windowed frame energies; then the bandwidth BW, the ERB
of the first band whose cumulative energy share exceeds 90 %, and the ratio of the modulation bands 0-3 to 4, 5 and,
depending on where BW falls among the cutoffs, 6 and 7.

Every row of the input runs in one pass per step (include/pbb.h, pbb_srmr_*): fp64, bitwise reproducible, and a
row's value does not depend on the other rows of the batch.  One documented difference: integer input is cast to
float64 first (the reference squares max|x| in the integer dtype, which overflows).
"""
import math

import numpy as np
import torch

from .. import _device, _lib
from ..transform import gammatone

MAX_SAMPLES = 1 << 22                 # PBB_SRMR_MAX_SAMPLES
HILBERT_WORKSPACE_BYTES = 1 << 31     # FFT buffers of the Hilbert step: sequences are transformed in groups this size
MODULATION_FREQUENCIES = (4.0, 6.5, 10.7, 17.6, 28.9, 47.5, 78.1, 128.0)

_tables = {}


def modulation_coefficients(sample_rate):
    """(8, 3): b0, a1, a2 of the modulation filters b = [b0, 0, -b0], a = [1, a1, a2], in the reference's order of
    operations (module_srmr.py:79-83)."""
    out = np.empty((8, 3))
    for k, f in enumerate(MODULATION_FREQUENCIES):
        W0 = math.tan(2 * math.pi * f / (2 * sample_rate))
        B0 = W0 / 2
        out[k] = [B0 / (1 + B0 + W0 ** 2), (2 * W0 ** 2 - 2) / (1 + B0 + W0 ** 2),
                  (1 - B0 + W0 ** 2) / (1 + B0 + W0 ** 2)]
    return out


def cutoffs(sample_rate):
    """The modulation filters' cutoffs (module_srmr.py:137-142)."""
    out = []
    for f in MODULATION_FREQUENCIES:
        w0 = 2 * math.pi * f / sample_rate
        B0 = math.tan(w0 / 2) / 2
        out.append(f - (B0 * sample_rate / (2 * math.pi)))
    return np.array(out)


def frame_lengths(sample_rate):
    """(W, S): the frame length int(sr / 1000) * 256 and the hop int(sr / 1000) * 64."""
    k = int(sample_rate / 1000)
    return k * 256, k * 64


def _modulation_step(coef, state):
    """One zero-input sample of the modulation filters on states (8, 2, m), (z0, z1) of lfilter's direct form II
    transposed: y = z0, z0 <- z1 - a1 y, z1 <- -a2 y."""
    y = state[:, 0]
    return np.stack([state[:, 1] - coef[:, 1, None] * y, -coef[:, 2, None] * y], axis=1)


def _device_tables(sample_rate, n, low_freq):
    key = (sample_rate, n, low_freq, _device.device())
    t = _tables.get(key)
    if t is None:
        W, S = frame_lengths(sample_rate)
        coef = modulation_coefficients(sample_rate)
        trans = gammatone.chunk_transition(_modulation_step, coef, 2, S).reshape(8, 4)
        erb = gammatone.calculate_cfs(low_freq, sample_rate / 2, n) / 9.26449 + 24.7
        t = _tables[key] = tuple(_device.to_device(np.ascontiguousarray(v, dtype=np.float64)) for v in (
            coef, trans, np.hamming(W), erb, cutoffs(sample_rate)))
    return t


def _check(signal, sample_rate, n, low_freq):
    """The input as a contiguous float32 / float64 CUDA tensor of at least one axis, and whether numpy came in."""
    like_numpy = not _device.is_tensor(signal)
    x = np.asarray(signal) if like_numpy else signal
    if x.ndim == 0:
        raise NotImplementedError(0)
    for i in range(x.ndim - 1):
        assert x.shape[i] < 30, (i, tuple(x.shape))
    gammatone.calculate_cfs(low_freq, sample_rate / 2, n)   # the reference's errors for an invalid n
    if int(sample_rate / 1000) < 1:
        raise ValueError(f'srmr needs int(sample_rate / 1000) >= 1, got sample_rate={sample_rate}')
    N = x.shape[-1]
    if not 1 <= N <= MAX_SAMPLES:
        raise ValueError(f'srmr supports 1 to {MAX_SAMPLES} samples per signal, got {N}')
    if np.iscomplexobj(x) if like_numpy else x.is_complex():
        raise TypeError(f'srmr of a real signal, got {x.dtype}')
    if like_numpy:
        x = x.astype(np.float32 if x.dtype == np.float32 else np.float64, copy=False)
    else:
        x = x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)
    return _device.to_device(x), like_numpy


def _vad(xd, sample_rate, normalise):
    """(rows, N) float64 kept samples (normalised or not) and N_r (rows,) int64 of a (..., N) CUDA tensor."""
    lib = _lib.load()
    N = xd.shape[-1]
    rows = xd.numel() // N
    nbytes = lib.pbb_srmr_vad_workspace_bytes(rows, N)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xd.device)
    out = _device.empty((rows, N), torch.float64)
    nr = _device.empty((rows,), torch.int64)
    stats = _device.empty((rows, 2), torch.float64)
    _device.call('pbb_srmr_vad', xd, _lib.PBB_F32 if xd.dtype == torch.float32 else _lib.PBB_F64, rows, N,
                 0.05 * sample_rate, int(normalise), ws, nbytes, out, nr, stats)
    return out, nr


def _hilbert_envelopes(y, nr):
    """|hilbert| of the first N_r samples of every sequence of y (n, rows, N), in place."""
    lib = _lib.load()
    n, rows, N = y.shape
    P = 1 << (lib.pbb_srmr_fft_log2(N) - 1)
    group = max(1, min(n * rows, HILBERT_WORKSPACE_BYTES // (16 * P)))
    nbytes = lib.pbb_srmr_hilbert_workspace_bytes(rows, N, group)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=y.device)
    _device.call('pbb_srmr_hilbert', y, rows, N, n, nr, group, ws, nbytes)
    return y


def _stages(xd, sample_rate, n, low_freq):
    """Every step on the device: dict of nr, normalised (rows, N), envelopes (n, rows, N; entries past N_r are not
    envelopes), means (rows, n, 8) and value (rows,)."""
    lib = _lib.load()
    coef, trans, window, erb, cut = _device_tables(sample_rate, n, low_freq)
    x, nr = _vad(xd, sample_rate, True)
    rows, N = x.shape
    env = _hilbert_envelopes(gammatone.filterbank_tensor(x, sample_rate, n, low_freq, sample_rate / 2), nr)
    hop = frame_lengths(sample_rate)[1]
    nbytes = lib.pbb_srmr_means_workspace_bytes(rows, N, n, hop)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xd.device)
    means = _device.empty((rows, n, 8), torch.float64)
    _device.call('pbb_srmr_means', env, rows, N, n, nr, hop, coef, trans, window, ws, nbytes, means)
    value = _device.empty((rows,), torch.float64)
    _device.call('pbb_srmr_ratio', means, rows, n, erb, cut, value)
    return dict(nr=nr, normalised=x, envelopes=env, means=means, value=value)


def srmr(signal, sample_rate: int = 16000, n_cochlear_filters: int = 23, low_freq: int = 125):
    """pb_bss.evaluation.srmr: the SRMR of every signal along the last axis.  1-D numpy input gives an np.float64,
    n-D input an ndarray of shape signal.shape[:-1] (every leading dim must be < 30, else AssertionError); 0-d input
    raises NotImplementedError.  A CUDA tensor in gives a float64 CUDA tensor of shape signal.shape[:-1] (0-d for
    1-D input), and the call only enqueues work on the current stream.  Signals of more than 2^22 samples raise
    ValueError."""
    xd, like_numpy = _check(signal, sample_rate, n_cochlear_filters, low_freq)
    value = _stages(xd, sample_rate, n_cochlear_filters, low_freq)['value'].reshape(xd.shape[:-1])
    if not like_numpy:
        return value
    v = value.cpu().numpy()
    return np.float64(v) if v.ndim == 0 else v


def SRMR(signal, sample_rate: int = 16000, n: int = 23, low_freq: int = 125):
    """pb_bss.evaluation.module_srmr.SRMR: the SRMR of one 1-D signal (a float; a 0-d float64 CUDA tensor for a CUDA
    tensor)."""
    if np.ndim(signal) != 1 if not _device.is_tensor(signal) else signal.dim() != 1:
        raise ValueError('SRMR takes one 1-D signal; srmr takes batches')
    return srmr(signal, sample_rate, n, low_freq)
