"""The gammatone filterbank of pb_bss/transform/gammatone.py on the device, with the reference's names, defaults and
return type: ``gammatone_filterbank(signal, sample_rate, n, low_freq, high_freq)`` gives a list of n float64 arrays
(numpy in -> numpy out, CUDA tensor in -> CUDA tensors out, on the current stream, without a host synchronisation),
each ``signal`` filtered along its last axis by one gammatone filter.

The filters follow Slaney, "An Efficient Implementation of the Patterson-Holdsworth Auditory Filter Bank" (Apple
Computer Technical Report #35, 1993): n centre frequencies spaced linearly on the ERB-rate scale 21.4 log10(0.00437 f
+ 1) from ``low_freq`` up to (not including) ``high_freq``, and for each a 4th-order gammatone filter realised as four
second-order sections in cascade.  The sections share the complex-conjugate pole pair exp(-B T +- 2 pi i f_c T),
B = 1.019 * 2 pi ERB(f_c); section k has the zero T cos(2 pi f_c T) +- sqrt(3 -+ 2^1.5) T sin(2 pi f_c T) (scaled by
exp(-B T)), and the first section is divided by the cascade's gain at f_c, so each filter has unit gain at its
centre frequency.  Each section runs in direct form II transposed from zero state, as scipy.signal.lfilter does.

The coefficients are a few hundred scalars, computed here in NumPy and cached on the device; the cascade runs in the
fp64 kernels of csrc/gammatone.cuh as a chunked linear scan over time (include/pbb.h, pbb_gammatone).  Complex input
raises TypeError.
"""
import numpy as np
import torch

from .. import _device, _lib

EAR_Q = 9.26449   # Glasberg and Moore's ERB: f / EAR_Q + MIN_BW (TR #35)
MIN_BW = 24.7
CARRY_GROUP = 32  # chunks per group of the carry kernel (PBB_GAMMATONE_CARRY_GROUP, include/pbb.h)

_tables = {}


def Hz_2_ERBS(f):
    """ERB-rate (in ERBs) of the frequency f (Hz)."""
    return 21.4 * (np.log(0.00437 * f + 1) / np.log(10))


def ERBS_2_Hz(f):
    """Frequency (Hz) of the ERB-rate f, the inverse of Hz_2_ERBS."""
    return (10 ** (f / 21.4) - 1) / 0.00437


def calculate_cfs(low_f, high_f, n):
    """n centre frequencies spaced linearly on the ERB-rate scale from low_f up to, but not including, high_f."""
    cfs = np.empty((n,))                   # ValueError for a negative n, TypeError for a non-integer one
    low, high = float(Hz_2_ERBS(low_f)), float(Hz_2_ERBS(high_f))
    step = (high - low) / n                # ZeroDivisionError for n = 0
    cfs[:] = ERBS_2_Hz(low + np.arange(n) * step)
    return cfs


def filter_coefficients(cfs, sample_rate):
    """Per filter (rows of the returned (n, 10) array): (b0, b1) of the four sections, then (a1, a2) of their shared
    denominator [1, a1, a2].  The sections' b2 is 0.  The first section carries 1 / gain."""
    cf = np.asarray(cfs, dtype=np.float64)
    pi = np.pi
    T = 1 / sample_rate
    B = 1.019 * 2 * pi * (cf / EAR_Q + MIN_BW)
    # TR #35's formulas, written in the paper's order of operations.  The gain's denominator cancels for low centre
    # frequencies, so another arrangement of the same algebra rounds differently there, by up to ~1e-11 relative.
    cos, sin, decay = np.cos(2 * cf * pi * T), np.sin(2 * cf * pi * T), np.exp(B * T)
    a1 = -2 * cos / decay
    a2 = np.exp(-2 * B * T)
    # the four zeros, in the order of the cascade: -(T cos + s T sin) / exp(B T), s = +-sqrt(3 + 2^1.5), +-sqrt(3 - 2^1.5)
    rp, rm = (3 + 2 ** 1.5) ** 0.5, (3 - 2 ** 1.5) ** 0.5
    s = np.array([rp, -rp, rm, -rm])
    b1 = -(T * (cos / decay)[:, None] + s * (T * (sin / decay))[:, None])
    # the cascade's gain at its centre frequency
    z = np.exp(4j * cf * pi * T)
    c1, c2 = -2 * z * T, 2 * np.exp(-1 * B * T + 2j * cf * pi * T) * T
    num = ((c1 + c2 * (cos - rm * sin)) * (c1 + c2 * (cos + rm * sin))
           * (c1 + c2 * (cos - rp * sin)) * (c1 + c2 * (cos + rp * sin)))
    gain = np.abs(num / (-2 / np.exp(2 * B * T) - 2 * z + 2 * (1 + z) / decay) ** 4)
    b0 = np.full((len(cf), 4), T)
    b0[:, 0] /= gain
    b1[:, 0] /= gain
    return np.concatenate([np.stack([b0, b1], axis=-1).reshape(-1, 8), a1[:, None], a2[:, None]], axis=1)


def _cascade_step(coef, state):
    """One zero-input sample of the cascade on states (n, 8, m): the recurrence of the device kernel, with the state
    order (u_0, v_0, ..., u_3, v_3) of the four direct-form-II-transposed sections."""
    out = np.empty_like(state)
    w = np.zeros_like(state[:, 0])
    for k in range(4):
        b0, b1 = coef[:, 2 * k, None], coef[:, 2 * k + 1, None]
        a1, a2 = coef[:, 8, None], coef[:, 9, None]
        y = b0 * w + state[:, 2 * k]
        out[:, 2 * k] = b1 * w + state[:, 2 * k + 1] - a1 * y
        out[:, 2 * k + 1] = -a2 * y
        w = y
    return out


def chunk_transition(step, coef, dim, length):
    """(n, dim, dim): the zero-input state transition of n linear recurrences over `length` samples, the recurrence
    ``step(coef, state)`` (states (n, dim, m)) run from the dim unit states."""
    M = np.broadcast_to(np.eye(dim), (coef.shape[0], dim, dim)).copy()
    for _ in range(length):
        M = step(coef, M)
    return M


def transition_matrices(coef, chunk_length):
    """(n, 2, 8, 8): the cascade's zero-input state transition over chunk_length samples, M, and over CARRY_GROUP
    chunks, M^CARRY_GROUP.  M is the recurrence run from the 8 unit states and M^CARRY_GROUP a chain of products, as
    the device applies them.  Repeated squaring would be faster but cancels in the blocks that map the first section's
    states (about 1e10 times the signal, through 1 / gain) into the later sections': at 48 kHz it costs the output a
    factor of 40 in accuracy."""
    M = chunk_transition(_cascade_step, coef, 8, chunk_length)
    MG = M
    for _ in range(CARRY_GROUP - 1):
        MG = M @ MG
    return np.stack([M, MG], axis=1)


def chunk_length(rows, n, N):
    """The chunk length pbb_gammatone uses for `rows` signals of N samples and n filters (a host-only query)."""
    return int(_lib.load().pbb_gammatone_chunk_length(int(rows), int(n), int(N)))


def _device_tables(sample_rate, n, low_freq, high_freq, L):
    key = (sample_rate, n, low_freq, high_freq, L, _device.device())
    t = _tables.get(key)
    if t is None:
        coef = filter_coefficients(calculate_cfs(low_freq, high_freq, n), sample_rate)
        t = _tables[key] = (_device.to_device(coef), _device.to_device(transition_matrices(coef, L)))
    return t


def gammatone_filterbank(signal, sample_rate=16000, n=23, low_freq=125, high_freq=0):
    """pb_bss.transform.gammatone.gammatone_filterbank: a list of n float64 arrays of the shape of ``signal``, entry
    i the signal filtered along its last axis by the gammatone filter of the i-th centre frequency
    (``calculate_cfs(low_freq, high_freq or sample_rate / 2, n)``).  float32 and integer input give float64, as
    scipy.signal.lfilter does; complex input raises TypeError.  CUDA tensors in give CUDA tensors out (views of one
    (n, *signal.shape) tensor), and the call only enqueues work on the current stream."""
    if high_freq == 0:
        high_freq = sample_rate / 2
    calculate_cfs(low_freq, high_freq, n)      # the reference's errors for an invalid n, before any other check
    like_numpy = not _device.is_tensor(signal)
    x = np.asarray(signal) if like_numpy else signal
    if np.iscomplexobj(x) if like_numpy else x.is_complex():
        raise TypeError(f'gammatone_filterbank of a real signal, got {x.dtype}')
    if like_numpy:
        x = x.astype(np.float32 if x.dtype == np.float32 else np.float64, copy=False)
    else:
        x = x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)
    xd = _device.to_device(x)
    if not xd.shape:
        raise ValueError('gammatone_filterbank needs a signal with at least one axis')
    out = filterbank_tensor(xd, sample_rate, n, low_freq, high_freq)
    return list(out.cpu().numpy()) if like_numpy else list(out.unbind(0))


def filterbank_tensor(xd, sample_rate, n, low_freq, high_freq):
    """The (n, *xd.shape) float64 CUDA tensor of the filter outputs of a contiguous float32 / float64 CUDA tensor xd
    with at least one axis, enqueued on the current stream."""
    shape = tuple(xd.shape)
    N = shape[-1]
    rows = int(np.prod(shape[:-1], dtype=np.int64))
    out = _device.empty((n,) + shape, torch.float64)
    if out.numel():
        lib = _lib.load()
        L = lib.pbb_gammatone_chunk_length(rows, n, N)
        coef, trans = _device_tables(sample_rate, n, low_freq, high_freq, L)
        nbytes = lib.pbb_gammatone_workspace_bytes(rows, n, N)
        ws = _device.workspace(nbytes) if nbytes else None
        _device.call('pbb_gammatone', xd, _lib.PBB_F32 if xd.dtype == torch.float32 else _lib.PBB_F64, rows, N, n, coef,
                     trans, L, ws, nbytes, out)
    return out
