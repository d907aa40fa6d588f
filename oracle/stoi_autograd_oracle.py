"""A float64 torch restatement of STOI and ESTOI (oracle/stoi_oracle.py, oracle/estoi_oracle.py) that torch autograd
differentiates: the reference gradients of pb_bss_b200.evaluation.stoi's backward.  Test infrastructure only.

Per row, on whichever device the signals are:
  - the resampler is resample_poly's polyphase filter (module_stoi.polyphase_taps) as one convolution of the
    zero-stuffed signal, sampled at (j + pre_remove) down;
  - the keep mask is computed under no_grad, so it is a constant of the graph;
  - the kept windowed frames are overlap-added, framed again, windowed again, torch.fft.rfft(n=512);
  - band energies are torch.linalg.vector_norm over the band's bins (a zero norm has a zero subgradient);
  - STOI: the clip min(c y, C x) is a torch.where with the forward's rule (the y term where c y < C x or c y is NaN,
    else the x term, so a tie goes to x); the norms are vector_norm;
  - ESTOI: each normalisation is 1 / sqrt of the centred sum of squares, with the 2^-92 rule as a torch.where (the
    tiny rows and columns become constant zeros, which pass no gradient);
  - fewer than 30 STFT frames: the constant 1e-5.
The restatement sums in torch's orders, not the device's, so values agree to rounding, not bitwise.
"""
import numpy as np
import torch
import torch.nn.functional as tF

from pb_bss_b200.evaluation import module_stoi as MS

FRAME, HOP, NFFT, SEG, BANDS = 256, 128, 512, 30, 15
EPS = float(np.finfo(float).eps)
CLIP = 1.0 + 10 ** (15 / 20)
DYN_RANGE = 40.0
TINY = 2.0 ** -92


def resample(x, fs):
    """x (..., n) float64 -> (..., L) at 10 kHz: scipy.signal.resample_poly with pystoi's window, as a convolution."""
    up, down = MS.rates(fs)
    if (up, down) == (1, 1):
        return x
    taps, pre = MS.polyphase_taps(fs)
    h = torch.from_numpy(np.ascontiguousarray(taps.T).reshape(-1).copy()).to(x)   # h[q] = taps[q % up][q // up]
    n = x.shape[-1]
    L = MS.resampled_length(n, fs)
    lead = x.shape[:-1]
    xu = torch.zeros(lead + (n * up,), dtype=x.dtype, device=x.device)
    xu = xu.index_copy(-1, torch.arange(0, n * up, up, device=x.device), x)
    t = (torch.arange(L, device=x.device) + pre) * down
    need = int(t[-1]) + 1
    xp = tF.pad(xu.reshape(-1, 1, n * up), (h.numel() - 1, max(0, need - n * up)))
    full = tF.conv1d(xp, h.flip(0).view(1, 1, -1))          # full[t] = sum_q h[q] xu[t - q]
    return full.reshape(lead + (-1,))[..., t]


def window(like):
    return torch.from_numpy(MS.window()).to(like)


def num_frames(length):
    return len(range(0, length - FRAME, HOP))


def _frames(s, count):
    return s.unfold(-1, FRAME, HOP)[..., :count, :]


def _overlap_add(fr):
    """(K, 256) -> ((K - 1) 128 + 256,)"""
    first = tF.pad(fr[:, :HOP], (0, 0, 0, 1))
    second = tF.pad(fr[:, HOP:], (0, 0, 1, 0))
    return (first + second).reshape(-1)


def band_energies(s, count):
    """(15, count) band energies of the STFT of s (count frames)."""
    w = window(s)
    X = torch.fft.rfft(w * _frames(s, count), n=NFFT)
    return torch.stack([torch.linalg.vector_norm(X[:, lo:hi], dim=-1) for lo, hi in MS.band_edges()], 0)


def stoi_segments(x_tob, y_tob):
    """STOI's per-segment sums of the band correlations, (J,)."""
    xs = x_tob.unfold(1, SEG, 1).transpose(0, 1)     # (J, 15, 30)
    ys = y_tob.unfold(1, SEG, 1).transpose(0, 1)
    c = torch.linalg.vector_norm(xs, dim=-1, keepdim=True) / (torch.linalg.vector_norm(ys, dim=-1, keepdim=True) + EPS)
    a, b = ys * c, xs * CLIP
    yp = torch.where((a < b) | torch.isnan(a), a, b)
    yp = yp - yp.mean(-1, keepdim=True)
    xc = xs - xs.mean(-1, keepdim=True)
    d = (yp * xc).sum(-1) / ((torch.linalg.vector_norm(yp, dim=-1) + EPS) * (torch.linalg.vector_norm(xc, dim=-1) + EPS))
    return d.sum(-1)


def _normalise(v, dim):
    with torch.no_grad():
        raw = (v * v).sum(dim, keepdim=True)
    u = v - v.mean(dim, keepdim=True)
    ss = (u * u).sum(dim, keepdim=True)
    tiny = (ss <= TINY * raw).detach()
    inv = torch.where(tiny, torch.zeros_like(ss), 1.0 / torch.sqrt(torch.where(tiny, torch.ones_like(ss), ss)))
    return u * inv


def estoi_segments(x_tob, y_tob):
    """ESTOI's per-segment sums of the normalised products, (J,) (d_m times 30)."""
    xs = x_tob.unfold(1, SEG, 1).transpose(0, 1)
    ys = y_tob.unfold(1, SEG, 1).transpose(0, 1)
    zx = _normalise(_normalise(xs, -1), -2)
    zy = _normalise(_normalise(ys, -1), -2)
    return (zx * zy).sum((-2, -1))


def stoi_row(x, y, fs, extended=False):
    """dict(value (0-d), K, M, x_tob, y_tob) of one pair of 1-D float64 tensors."""
    xs, ys = resample(x, fs), resample(y, fs)
    L = xs.shape[-1]
    F = num_frames(L)
    w = window(xs)
    xf, yf = w * _frames(xs, F), w * _frames(ys, F)
    with torch.no_grad():
        e = 20 * torch.log10(torch.linalg.vector_norm(xf, dim=-1) + EPS)
        mask = (e.max() - DYN_RANGE - e) < 0
    K = int(mask.sum())
    M = max(K - 1, 0)
    out = dict(K=K, M=M)
    if M < SEG:
        out['value'] = torch.tensor(1e-5, dtype=torch.float64, device=x.device)
        return out
    x_tob = band_energies(_overlap_add(xf[mask]), M)
    y_tob = band_energies(_overlap_add(yf[mask]), M)
    J = M - SEG + 1
    terms = SEG if extended else BANDS
    seg = estoi_segments(x_tob, y_tob) if extended else stoi_segments(x_tob, y_tob)
    out.update(x_tob=x_tob, y_tob=y_tob, value=seg.sum() / (J * terms))
    return out


def stoi(x, y, fs, extended=False):
    """(values (rows,), K list, M list) of x, y (rows, n) float64 tensors (broadcast first if needed)."""
    rows = [stoi_row(a, b, fs, extended) for a, b in zip(x, y)]
    return torch.stack([r['value'] for r in rows]), [r['K'] for r in rows], [r['M'] for r in rows]
