"""NumPy restatement of SRMR, the speech-to-reverberation modulation energy ratio of
pb_bss/evaluation/module_srmr.py, with its intermediates and decision margins.

Steps (the reference's quirks kept): the VAD of ``_preprocessing_vad`` (an amplitude compared with max|x|^2 / 1e5,
gaps of more than 0.05 sr between above-threshold samples removed), normalisation to zero mean and unit population
std, the gammatone filterbank (oracle/gammatone_oracle.py), the Hilbert envelope of every band, eight second-order
modulation band-pass filters per band, Hamming-windowed frame energies (frames of ``segment_axis`` with end='pad'),
their means over frames, the 90 % bandwidth and the ratio of the modulation bands 0-3 to 4..7.  Written from the
contract; tests/test_srmr_oracle.py checks it against tests/golden/srmr.npz, which the unmodified reference produced
(oracle/make_golden_srmr.py)."""
import math

import numpy as np
import scipy.signal

from . import gammatone_oracle as GO

MOD_FREQS = (4.0, 6.5, 10.7, 17.6, 28.9, 47.5, 78.1, 128.0)


def segment_axis(x, length, shift, axis=-1, end='pad'):
    """Frames of length `length` every `shift` samples along the last axis, the contract of paderbox's
    ``segment_axis`` with ``end='pad'`` restated (this is not paderbox): a signal shorter than `length` is one frame
    zero-padded to `length`; otherwise zeros are appended until (N - length) % shift == 0, which gives
    1 + ceil((N - length) / shift) frames."""
    assert axis == -1 and end == 'pad'
    x = np.asarray(x)
    N = x.shape[-1]
    if N < length:
        pad = length - N
    else:
        pad = (-(N - length)) % shift
    x = np.concatenate([x, np.zeros(x.shape[:-1] + (pad,), x.dtype)], axis=-1)
    F = 1 + (x.shape[-1] - length) // shift
    idx = np.arange(F)[:, None] * shift + np.arange(length)
    return x[..., idx]


def frame_count(N, sample_rate):
    W, S = frame_lengths(sample_rate)
    return 1 if N < W else 1 + -(-(N - W) // S)


def frame_lengths(sample_rate):
    """(W, S): frame length and hop, int(sr / 1000) * 256 and * 64."""
    k = int(sample_rate / 1000)
    return k * 256, k * 64


def vad(x, sample_rate=16000):
    """_preprocessing_vad of a 1-D signal: the kept samples, in the input dtype."""
    x = np.asarray(x)
    return x[vad_keep(x, sample_rate)]


def vad_keep(x, sample_rate=16000):
    """The keep mask of _preprocessing_vad for a 1-D signal."""
    x = np.asarray(x)
    a = abs(x)
    threshold = (a.max() ** 2) / (10 ** 5)
    above = a > threshold
    idx = np.arange(len(x))
    prev = np.maximum.accumulate(np.where(above, idx, -1))
    nxt = np.minimum.accumulate(np.where(above, idx, len(x))[::-1])[::-1]
    gap = (prev >= 0) & (nxt < len(x)) & ((nxt - prev) > 0.05 * sample_rate)
    return above | ~gap


def modulation_coefficients(sample_rate):
    """(8, 2, 3): b and a of the eight modulation filters, in the reference's order of operations."""
    out = np.empty((8, 2, 3))
    for k, f in enumerate(MOD_FREQS):
        W0 = math.tan(2 * math.pi * f / (2 * sample_rate))
        B0 = W0 / 2
        d = 1 + B0 + W0 ** 2
        out[k, 0] = [B0 / d, 0, -B0 / d]
        out[k, 1] = [1, (2 * W0 ** 2 - 2) / d, (1 - B0 + W0 ** 2) / d]
    return out


def cutoffs(sample_rate):
    out = []
    for f in MOD_FREQS:
        w0 = 2 * math.pi * f / sample_rate
        B0 = math.tan(w0 / 2) / 2
        out.append(f - (B0 * sample_rate / (2 * math.pi)))
    return np.array(out)


def erbs(sample_rate, n, low_freq):
    return GO.centre_frequencies(low_freq, sample_rate / 2, n) / 9.26449 + 24.7


def hilbert_kernel(N):
    """g of length N with hilbert(x).imag = circular convolution of x with g: the imaginary part of the inverse DFT of
    scipy.signal.hilbert's multiplier h, in closed form (even N: 2 cot(pi n / N) / N at odd n, else 0; odd N:
    cot(pi n / (2N)) / N at odd n, -tan(pi n / (2N)) / N at even n), evaluated at min(n, N - n) with g[N - n] = -g[n]
    so that no small angle is lost."""
    n = np.arange(N)
    e = np.minimum(n, N - n)
    sign = np.where(n == e, 1.0, -1.0)
    g = np.zeros(N)
    nz = e > 0
    if N % 2 == 0:
        t = np.pi * e / N
        odd = nz & (e % 2 == 1)
        g[odd] = 2 / np.tan(t[odd]) / N
    else:
        t = np.pi * e / (2 * N)
        odd, even = nz & (e % 2 == 1), nz & (e % 2 == 0)
        g[odd] = 1 / np.tan(t[odd]) / N
        g[even] = -np.tan(t[even]) / N
    return sign * g


def hilbert_multiplier(N):
    """scipy.signal.hilbert's h."""
    h = np.zeros(N)
    if N % 2 == 0:
        h[0] = h[N // 2] = 1
        h[1:N // 2] = 2
    else:
        h[0] = 1
        h[1:(N + 1) // 2] = 2
    return h


def srmr_single(x, sample_rate=16000, n=23, low_freq=125):
    """SRMR of one 1-D signal, with every intermediate: dict of nr, compacted, normalised, envelopes (n, nr), means
    (n, 8), bw_index (-1: none), bands (modulation bands in the denominator), value, margin_bw (min over bands of
    |cumulative % - 90|), margin_cutoff (distance of BW to the nearest cutoff)."""
    x = np.asarray(x)
    if np.issubdtype(x.dtype, np.integer):
        x = x.astype(np.float64)
    kept = vad(x, sample_rate)
    s = kept - np.mean(kept)
    s /= np.std(s, keepdims=True)
    y = np.stack(GO.gammatone_filterbank(s, sample_rate, n, low_freq))
    env = np.abs(scipy.signal.hilbert(y, axis=-1))
    W, S = frame_lengths(sample_rate)
    window = scipy.signal.windows.hamming(W, sym=True)
    coef = modulation_coefficients(sample_rate)
    means = np.empty((n, 8))
    for k in range(8):
        m = scipy.signal.lfilter(coef[k, 0], coef[k, 1], env, axis=-1)
        frames = segment_axis(m, W, S)
        means[:, k] = np.mean(np.sum(np.square(window * frames), axis=-1), axis=-1)
    total = np.sum(means)
    cum = np.cumsum(np.sum(means, axis=1) * 100 / total)
    hit = np.flatnonzero(cum > 90)
    bw_index = int(hit[0]) if len(hit) else -1
    erb = erbs(sample_rate, n, low_freq)
    BW = erb[bw_index] if bw_index >= 0 else 0.0
    cut = cutoffs(sample_rate)
    col = np.sum(means, axis=0)
    numerator = np.sum(col[:4])
    denominator = col[4]
    bands = 1
    for i in range(5, 8):
        denominator += col[i]
        bands += 1
        if cut[i - 1] < BW < cut[i]:
            break
    return dict(nr=len(kept), compacted=kept, normalised=s, envelopes=env, means=means, bw_index=bw_index,
                bands=bands, value=numerator / denominator,
                margin_bw=float(np.min(np.abs(cum - 90))) if np.isfinite(cum).all() else 0.0,
                margin_cutoff=float(np.min(np.abs(cut - BW))))


def srmr(signal, sample_rate=16000, n_cochlear_filters=23, low_freq=125):
    """The value(s) only: a float for 1-D input, an array of shape signal.shape[:-1] otherwise."""
    x = np.asarray(signal)
    if x.ndim == 0:
        raise NotImplementedError(0)
    if x.ndim == 1:
        return srmr_single(x, sample_rate, n_cochlear_filters, low_freq)['value']
    rows = x.reshape(-1, x.shape[-1])
    return np.array([srmr_single(r, sample_rate, n_cochlear_filters, low_freq)['value']
                     for r in rows]).reshape(x.shape[:-1])
