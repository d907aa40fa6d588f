"""NumPy restatement of ESTOI, the extended short-time objective intelligibility (Jensen and Taal, "An algorithm for
predicting the intelligibility of speech masked by modulated noise maskers", IEEE/ACM TASLP 24(11), 2016), i.e.
pystoi's ``stoi(x, y, fs, extended=True)``.  Test infrastructure only: pystoi is not a dependency.

The contract is restated from the paper and from pystoi's documented algorithm.  It has not been checked against
pystoi itself, which is not a dependency of this project.

Stages 1-5 are STOI's (oracle/stoi_oracle.py): resampling to 10 kHz, silent-frame removal, the STFT, the one-third
octave band envelopes x_tob, y_tob (15, M), and 1e-5 with a RuntimeWarning below 30 STFT frames.  Then, for each of
the J = M - 29 segments m, X, Y = the (15, 30) windows of bands x frames m .. m + 29, without STOI's clipping and
without scaling Y by ||X|| / ||Y||:
  1. row step, per band: subtract the mean over the 30 frames, divide by the root of the sum of squares;
  2. column step, per frame: subtract the mean over the 15 bands of the row-normalised values, divide by the root of
     the sum of squares;
  3. d_m = (1/30) sum_n sum_b X[b, n] Y[b, n] of the normalised segments;
  4. ESTOI = sum_m d_m / J.

Documented difference from pystoi: pystoi adds N(0, eps^2) noise before each normalisation step; this contract does
not.  Instead a row or column whose centred sum of squares is zero up to rounding, at most TINY = 2^-92 = (64 eps)^2
times its sum of squares before centring, normalises to zeros: the expected value of pystoi's random contribution
there, and the exact-arithmetic value.  Two cases reach it:
  - exactly zero rows, e.g. 30 frames of digital silence in the estimate;
  - a segment of the estimate with one non-zero frame and 29 silent ones (at either end of a silent stretch): every
    band normalises to the same pattern, so in exact arithmetic every column is constant and centres to zero, while
    in floating point it centres to rounding noise of about eps, whose normalised direction depends on the order of
    operations.
Genuine rows and columns are many orders of magnitude above TINY.  NaN and inf propagate as in STOI (a NaN sum
fails the comparison).
"""
import numpy as np

from oracle import stoi_oracle as S

N = S.N
NUMBAND = S.NUMBAND
TINY = 2.0 ** -92   # (64 eps)^2: a centred sum of squares at most TINY times the raw one is zero up to rounding


def _normalise(v, axis):
    """v minus its mean along axis, times 1 / sqrt of the centred sum of squares (0 where that sum is at most TINY
    times the sum of squares of v)."""
    raw = np.sum(v * v, axis=axis, keepdims=True)
    v = v - np.mean(v, axis=axis, keepdims=True)
    ss = np.sum(v * v, axis=axis, keepdims=True)
    inv = np.zeros_like(ss)
    keep = ~(ss <= TINY * raw)
    inv[keep] = 1.0 / np.sqrt(ss[keep])
    return v * inv


def row_col_normalize(seg):
    """(..., 15, 30) segments: the row step over frames, then the column step over bands."""
    return _normalise(_normalise(seg, -1), -2)


def segments(x_tob, y_tob):
    """The (J, 15, 30) segments of the band envelopes (15, M), M >= 30."""
    M = x_tob.shape[1]
    return (np.array([x_tob[:, m:m + N] for m in range(M - N + 1)]),
            np.array([y_tob[:, m:m + N] for m in range(M - N + 1)]))


def segment_values(x_tob, y_tob):
    """d_m of every segment, (J,)."""
    xs, ys = segments(x_tob, y_tob)
    return np.sum(row_col_normalize(xs) * row_col_normalize(ys), axis=(1, 2)) / N


def from_bands(x_tob, y_tob):
    """ESTOI of band envelopes (15, M), M >= 30: the sum over (segment, band, frame) / (30 J)."""
    xs, ys = segments(x_tob, y_tob)
    return np.sum(row_col_normalize(xs) * row_col_normalize(ys)) / (N * xs.shape[0])


def stages(x, y, fs):
    """STOI's intermediates of one pair (oracle/stoi_oracle.py, stages), with the ESTOI value."""
    out = S.stages(x, y, fs)
    if out['M'] >= N:
        out['value'] = from_bands(out['x_tob'], out['y_tob'])
    return out


def stoi(reference, estimation, sample_rate, extended=False):
    """pb_bss.evaluation.stoi with pystoi's extended switch: STOI (oracle/stoi_oracle.py) or ESTOI, broadcast, one
    value per leading index (an array for ndim >= 2)."""
    if not extended:
        return S.stoi(reference, estimation, sample_rate)
    estimation, reference = np.broadcast_arrays(estimation, reference)
    if reference.ndim >= 2:
        return np.array([stoi(x, y, sample_rate, True) for x, y in zip(reference, estimation)])
    return stages(reference, estimation, sample_rate)['value']
