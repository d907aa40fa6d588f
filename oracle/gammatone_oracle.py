"""NumPy restatement of the gammatone filterbank of pb_bss/transform/gammatone.py (Slaney, Apple TR #35): the
centre frequencies, the per-filter coefficients in the reference's tuple form and the filterbank as four
scipy.signal.lfilter passes per filter.  Written from the paper; tests/test_gammatone_oracle.py checks it against
tests/golden/gammatone.npz, which the unmodified reference produced (oracle/make_golden_gammatone.py)."""
import numpy as np
from scipy.signal import lfilter


def hz_to_erbs(f):
    return 21.4 * (np.log(0.00437 * np.asarray(f, dtype=np.float64) + 1) / np.log(10))


def erbs_to_hz(e):
    return (10 ** (np.asarray(e, dtype=np.float64) / 21.4) - 1) / 0.00437


def centre_frequencies(low_f, high_f, n):
    low, high = float(hz_to_erbs(low_f)), float(hz_to_erbs(high_f))
    return erbs_to_hz(low + np.arange(n) * ((high - low) / n))


def coefficients(cfs, sample_rate):
    """(A0, A11, A12, A13, A14, A2, B0, B1, B2, gain): section k has the numerator [A0, A1k, A2] and the denominator
    [B0, B1, B2]; the first numerator is divided by gain, the cascade's magnitude response at the centre frequency."""
    cf = np.asarray(cfs, dtype=np.float64)
    T = 1 / sample_rate
    B = 1.019 * 2 * np.pi * (cf / 9.26449 + 24.7)
    cos, sin, decay = np.cos(2 * cf * np.pi * T), np.sin(2 * cf * np.pi * T), np.exp(B * T)
    rp, rm = (3 + 2 ** 1.5) ** 0.5, (3 - 2 ** 1.5) ** 0.5
    A1 = [-(T * (cos / decay) + r * (T * (sin / decay))) for r in (rp, -rp, rm, -rm)]
    z = np.exp(4j * cf * np.pi * T)
    c1, c2 = -2 * z * T, 2 * np.exp(-1 * B * T + 2j * cf * np.pi * T) * T
    num = ((c1 + c2 * (cos - rm * sin)) * (c1 + c2 * (cos + rm * sin))
           * (c1 + c2 * (cos - rp * sin)) * (c1 + c2 * (cos + rp * sin)))
    gain = np.abs(num / (-2 / np.exp(2 * B * T) - 2 * z + 2 * (1 + z) / decay) ** 4)
    return T, A1[0], A1[1], A1[2], A1[3], 0, 1, -2 * cos / decay, np.exp(-2 * B * T), gain


def gammatone_filterbank(signal, sample_rate=16000, n=23, low_freq=125, high_freq=0):
    """List of n float64 arrays: the signal through each filter's four lfilter passes, along the last axis."""
    if high_freq == 0:
        high_freq = sample_rate / 2
    A0, A11, A12, A13, A14, A2, B0, B1, B2, gain = coefficients(centre_frequencies(low_freq, high_freq, n),
                                                                sample_rate)
    x = np.asarray(signal, dtype=np.float64)
    out = []
    for i in range(n):
        a = [B0, B1[i], B2[i]]
        y = lfilter([A0 / gain[i], A11[i] / gain[i], A2 / gain[i]], a, x)
        for A1k in (A12, A13, A14):
            y = lfilter([A0, A1k[i], A2], a, y)
        out.append(y)
    return out
