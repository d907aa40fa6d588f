"""CPU checks of the torch restatement of STOI and ESTOI (oracle/stoi_autograd_oracle.py) whose autograd gives the
reference gradients of the device backward: its values against the NumPy restatements (oracle/stoi_oracle.py,
oracle/estoi_oracle.py), and torch.autograd.gradcheck of it on signals just above 30 STFT frames."""
import numpy as np
import pytest
import scipy.signal
import torch

from oracle import estoi_oracle as E
from oracle import stoi_autograd_oracle as A
from oracle import stoi_oracle as O


def signals(rng, n, fs, gaps=()):
    """Coloured noise under a square envelope with a 19 dB swing (segments with the clip active and inactive, every
    frame far above the 40 dB threshold), zero over the fractions `gaps` (dropped frames); the estimate adds noise."""
    t = np.arange(n) / fs
    env = 1 + 0.9 * np.sign(np.sin(2 * np.pi * 4 * t + rng.uniform(0, 6)))
    x = scipy.signal.lfilter([1.0], [1.0, -1.3, 0.6], rng.standard_normal(n)) * env
    for a, b in gaps:
        x[int(a * n):int(b * n)] = 0.0
    y = x + 0.7 * rng.standard_normal(n)
    return x, y


def length_for_frames(frames, fs):
    """n with at least `frames` 256-sample frames at 10 kHz."""
    L = 256 + 128 * frames
    up, down = O.rates(fs)
    return -(-L * down // up)


@pytest.mark.parametrize('extended', [False, True])
@pytest.mark.parametrize('fs', [8000, 10000, 16000, 48000])
@pytest.mark.parametrize('gaps', [(), ((0.3, 0.45),)])
def test_forward_matches_numpy_restatement(fs, extended, gaps):
    rng = np.random.default_rng(fs + 7 * extended + len(gaps))
    n = length_for_frames(70, fs)
    x, y = signals(rng, n, fs, gaps)
    ref = E.stoi(x, y, fs, extended)
    st = O.stages(x, y, fs)
    v, K, M = A.stoi(torch.from_numpy(x)[None], torch.from_numpy(y)[None], fs, extended)
    assert (K[0], M[0]) == (st['K'], st['M'])
    assert M[0] >= 30
    assert abs(float(v[0]) - ref) <= 1e-12


def test_short_row_is_the_constant():
    rng = np.random.default_rng(3)
    x, y = signals(rng, length_for_frames(20, 10000), 10000)
    xt = torch.from_numpy(x)[None].requires_grad_()
    v, _, M = A.stoi(xt, torch.from_numpy(y)[None], 10000)
    assert M[0] < 30 and float(v[0]) == 1e-5 and not v.requires_grad


@pytest.mark.parametrize('extended', [False, True])
@pytest.mark.parametrize('fs', [8000, 10000, 16000])
def test_gradcheck_just_above_30_frames(fs, extended):
    rng = np.random.default_rng(fs + extended)
    x, y = signals(rng, length_for_frames(33, fs), fs)
    xt = torch.from_numpy(x)[None].requires_grad_()
    yt = torch.from_numpy(y)[None].requires_grad_()
    assert A.stoi(xt, yt, fs, extended)[2][0] >= 31
    assert torch.autograd.gradcheck(lambda a, b: A.stoi(a, b, fs, extended)[0], (xt, yt), fast_mode=True)
