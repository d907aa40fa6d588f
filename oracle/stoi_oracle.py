"""NumPy / SciPy restatement of STOI, the short-time objective intelligibility of pb_bss.evaluation.stoi (which calls
pystoi.stoi(x, y, fs_sig) with extended=False; Taal, Hendriks, Heusdens and Jensen, IEEE TASLP 19(7), 2011).  Test
infrastructure only: pystoi is not a dependency.

x is the reference and y the estimate, both computed in float64 (pystoi would frame float32 input at 10 kHz in
float32).  The steps:
  1. fs != 10000: scipy.signal.resample_poly(s, 10000, fs, window=h / h.sum()) with Octave's Kaiser design of h
     (``resample_window_oct``);
  2. silent-frame removal: 256-sample frames every 128 samples for 128 f < len - 256 (a frame that ends exactly at the
     last sample is not taken), windowed by w = hanning(258)[1:-1]; frame f is kept where
     max E - 40 - E_f < 0 with E_f = 20 log10(||w x_f|| + eps); the kept windowed frames of x, and with the same mask
     those of y, are overlap-added at hop 128;
  3. the STFT of both with the same frame rule, each frame windowed again by w, rfft(n=512);
  4. 15 one-third octave bands from 150 Hz: X_tob = sqrt of the band sums of |X|^2;
  5. fewer than 30 STFT frames: RuntimeWarning and 1e-5;
  6. the 30-frame segments: the clipped, normalised estimate against the reference, mean-removed, unit-norm, and the
     mean of their inner products over (segment, band).

Edge cases, which the device implementation follows:
  - a signal with no frame at all (a length at 10 kHz of at most 256) raises ValueError (NumPy's AxisError);
  - a non-finite reference sample makes max E non-finite, so every frame is dropped: the 1e-5 path;
  - a non-finite estimate sample with a finite reference gives NaN.
"""
import warnings

import numpy as np
import scipy.signal

FS = 10000
N_FRAME = 256
HOP = 128
NFFT = 512
NUMBAND = 15
MINFREQ = 150
N = 30
BETA = -15.
DYN_RANGE = 40
EPS = np.finfo(float).eps
WARNING = ('Not enough STFT frames to compute intermediate intelligibility measure after removing silent frames. '
           'Returning 1e-5. Please check you wav files')


def window():
    return np.hanning(N_FRAME + 2)[1:-1]


def band_edges():
    """(15, 2) int: the [lo, hi) rfft bins of every one-third octave band."""
    f = np.linspace(0, FS, NFFT + 1)[:NFFT // 2 + 1]
    k = np.arange(NUMBAND).astype(float)
    fl = MINFREQ * 2. ** ((2 * k - 1) / 6)
    fh = MINFREQ * 2. ** ((2 * k + 1) / 6)
    return np.array([[np.argmin((f - fl[i]) ** 2), np.argmin((f - fh[i]) ** 2)] for i in range(NUMBAND)])


def rates(fs):
    """(up, down): 10000 / fs in lowest terms."""
    g = np.gcd(FS, int(fs))
    return FS // g, int(fs) // g


def resample_window_oct(p, q):
    """Octave's resample filter: a Kaiser-windowed sinc at 60 dB rejection for the ratio p / q."""
    g = np.gcd(p, q)
    p, q = p / g, q / g
    stopband_cutoff_f = 1. / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = 60.0
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off_width))
    t = np.arange(-L, L + 1)
    ideal_filter = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    beta = 0.1102 * (rejection_db - 8.7)
    return np.kaiser(2 * L + 1, beta) * ideal_filter


def resample(x, fs):
    if fs == FS:
        return np.asarray(x, dtype=np.float64)
    h = resample_window_oct(FS, fs)
    return scipy.signal.resample_poly(np.asarray(x, dtype=np.float64), FS, fs, window=h / np.sum(h))


def resampled_length(n, fs):
    up, down = rates(fs)
    return -(-n * up // down)


def num_frames(length):
    """Frames f of the strict rule 128 f < length - 256."""
    return len(range(0, length - N_FRAME, HOP))


def _frames(x):
    w = window()
    return np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME, HOP)])


def _overlap_add(frames):
    out = np.zeros((len(frames) - 1) * HOP + N_FRAME)
    for i, fr in enumerate(frames):
        out[i * HOP:i * HOP + N_FRAME] += fr
    return out


def remove_silent_frames(x, y):
    """x_sil, y_sil and the keep mask."""
    xf, yf = _frames(x), _frames(y)
    e = 20 * np.log10(np.linalg.norm(xf, axis=1) + EPS)   # AxisError (a ValueError) without a frame
    mask = (np.max(e) - DYN_RANGE - e) < 0
    return _overlap_add(xf[mask]), _overlap_add(yf[mask]), mask, e


def stft(x):
    w = window()
    return np.array([np.fft.rfft(w * x[i:i + N_FRAME], n=NFFT) for i in range(0, len(x) - N_FRAME, HOP)])


def stages(x, y, fs):
    """Every intermediate of one pair of 1-D signals: resampled x and y, the frame energies (dB), the keep mask, K
    (kept frames), M (STFT frames), the band energies x_tob / y_tob (15, M) and the value."""
    x, y = resample(x, fs), resample(y, fs)
    if x.shape != y.shape:
        raise ValueError('x and y should have the same length')
    out = dict(x=x, y=y)
    xs, ys, mask, e = remove_silent_frames(x, y)
    out.update(energy=e, mask=mask, K=int(mask.sum()))
    X, Y = stft(xs), stft(ys)
    M = len(X)
    out['M'] = M
    if M < N:
        warnings.warn(WARNING, RuntimeWarning)
        out.update(x_tob=np.zeros((NUMBAND, M)), y_tob=np.zeros((NUMBAND, M)), value=1e-5)
        return out
    edges = band_edges()
    obm = np.zeros((NUMBAND, NFFT // 2 + 1))
    for i, (a, b) in enumerate(edges):
        obm[i, a:b] = 1
    x_tob = np.sqrt(obm @ np.abs(X.T) ** 2)
    y_tob = np.sqrt(obm @ np.abs(Y.T) ** 2)
    out.update(x_tob=x_tob, y_tob=y_tob)
    xseg = np.array([x_tob[:, m - N:m] for m in range(N, M + 1)])
    yseg = np.array([y_tob[:, m - N:m] for m in range(N, M + 1)])
    c = np.linalg.norm(xseg, axis=2, keepdims=True) / (np.linalg.norm(yseg, axis=2, keepdims=True) + EPS)
    yp = np.minimum(yseg * c, xseg * (1 + 10 ** (-BETA / 20)))
    yp = yp - np.mean(yp, axis=2, keepdims=True)
    xseg = xseg - np.mean(xseg, axis=2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + EPS
    xseg /= np.linalg.norm(xseg, axis=2, keepdims=True) + EPS
    out['value'] = np.sum(yp * xseg) / (xseg.shape[0] * NUMBAND)
    return out


def stoi_1d(x, y, fs):
    return stages(x, y, fs)['value']


def stoi(reference, estimation, sample_rate):
    """pb_bss.evaluation.stoi: broadcast, then one value per leading index (an array for ndim >= 2)."""
    estimation, reference = np.broadcast_arrays(estimation, reference)
    if reference.ndim >= 2:
        return np.array([stoi(x, y, sample_rate) for x, y in zip(reference, estimation)])
    return stoi_1d(reference, estimation, sample_rate)
