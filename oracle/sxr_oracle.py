"""NumPy restatement of SI-SDR (Le Roux et al., "SDR - half-baked or well done?", ICASSP 2019) and of the invasive
SxR of pb_bss.evaluation.sxr_module, written from the formulas, with NumPy's summation order made explicit where the
device kernels reproduce it (np_sum).  The checker of the GPU tests on shapes beyond tests/golden/metrics.npz."""
import itertools

import numpy as np


def np_sum(values):
    """np.sum of a short 1-D float64 sequence in NumPy's order: a left-to-right loop below 8 values, else 8
    accumulators over blocks of 8, combined as ((0 + 1) + (2 + 3)) + ((4 + 5) + (6 + 7)), then the rest in order."""
    v = [np.float64(x) for x in values]
    n = len(v)
    if n < 8:
        s = np.float64(0.0)
        for x in v:
            s = s + x
        return s
    r = v[:8]
    i = 8
    while i < n - n % 8:
        r = [r[j] + v[i + j] for j in range(8)]
        i += 8
    s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for x in v[i:]:
        s = s + x
    return s


def _db(s, x):
    with np.errstate(divide='ignore', invalid='ignore'):
        return 10 * np.log10(np.asarray(s, dtype=np.float64) / np.asarray(x, dtype=np.float64))


def power(x, axis=None, keepdims=False):
    """The mean of |x|^2 in float64: re^2 + im^2 for complex x."""
    x = np.asarray(x)
    p = x.real.astype(np.float64) ** 2 + x.imag.astype(np.float64) ** 2 if np.iscomplexobj(x) \
        else x.astype(np.float64) ** 2
    with np.errstate(invalid='ignore'):
        return np.mean(p, axis=axis, keepdims=keepdims)


def si_sdr(reference, estimation):
    """10 log10(||alpha r||^2 / ||e - alpha r||^2), alpha = <r, e> / <r, r>, over the last axis of the broadcast pair."""
    e, r = np.broadcast_arrays(np.asarray(estimation, dtype=np.float64), np.asarray(reference, dtype=np.float64))
    with np.errstate(divide='ignore', invalid='ignore'):
        alpha = np.sum(r * e, axis=-1, keepdims=True) / np.sum(r * r, axis=-1, keepdims=True)
        target = alpha * r
        residual = e - target
        return 10 * np.log10(np.sum(target * target, axis=-1) / np.sum(residual * residual, axis=-1))


def _mean_rows(v):
    """np.mean(v, axis=0) of v (K, C): the rows added in order, or the pairwise sum when C = 1 (NumPy then reduces one
    contiguous axis)."""
    K, C = v.shape
    if C == 1:
        return np.array([np_sum(v[:, 0]) / K])
    s = np.zeros(C)
    for k in range(K):
        s = s + v[k]
    return s / K


def input_sxr_from_powers(S, N, average_sources=True, average_channels=True):
    """SDR, SIR, SNR of the input from S (K, D) image powers and N (D) noise powers."""
    K, D = S.shape
    I = np.array([[np_sum([S[n, d] for n in range(K) if n != k]) for d in range(D)] for k in range(K)])
    if average_channels:
        S = np.array([np_sum(S[k]) / D for k in range(K)])
        I = np.array([np_sum(I[k]) / D for k in range(K)])
        N = np_sum(N) / D
    sdr, sir, snr = _db(S, I + N), _db(S, I), _db(S, N)
    if average_sources:
        if sdr.ndim == 1:
            return tuple(np_sum(v) / K for v in (sdr, sir, snr))
        return tuple(_mean_rows(v) for v in (sdr, sir, snr))
    return sdr, sir, snr


def input_sxr(images, noise, average_sources=True, average_channels=True):
    return input_sxr_from_powers(power(images, axis=-1), power(noise, axis=-1), average_sources, average_channels)


def output_sxr_from_powers(S, N, average_sources=True):
    """SDR, SIR, SNR and the selection of the output from S (K_source, K_target) and N (K_target): the first (in
    itertools.permutations order) selection of one target per source that maximises the summed power (a NaN wins)."""
    Ks, Kt = S.shape
    best, selection = None, None
    for p in itertools.permutations(range(Kt), Ks):
        m = np_sum([S[k, p[k]] for k in range(Ks)])
        if best is None or (np.isnan(m) and not np.isnan(best)) or (not np.isnan(best) and m > best):
            best, selection = m, p
    if selection is None:
        raise ValueError('attempt to get argmax of an empty sequence')
    selection = np.array(selection, dtype=np.int64)
    SS = np.array([S[k, selection[k]] for k in range(Ks)])
    II = np.array([np_sum([S[n, selection[k]] for n in range(Ks) if n != k]) for k in range(Ks)])
    NN = N[selection]
    out = _db(SS, II + NN), _db(SS, II), _db(SS, NN)
    if average_sources:
        out = tuple(np_sum(v) / Ks for v in out)
    return out + (selection,)


def output_sxr(image_contribution, noise_contribution, average_sources=True):
    return output_sxr_from_powers(power(image_contribution, axis=-1), power(noise_contribution, axis=-1),
                                  average_sources)
