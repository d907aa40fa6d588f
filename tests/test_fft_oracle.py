"""CPU checks of oracle/fft_oracle.py, the long-double restatement the FFT kernels are tested against
(tests/test_fft_kernels_gpu.py): the oracle against an mpmath DFT, the float64 model of the kernels' arithmetic
against the oracle's bounds at every size (with at least 2x margin, so the bounds are not tighter than the algorithm
achieves), and the host's tiling rule pbb_stft_frames_per_cta."""
import numpy as np
import pytest
import scipy.signal

from oracle import fft_oracle as FO
from oracle import transform_oracle as TO

SIZES = [64, 128, 256, 512, 1024, 2048, 4096]


def _mp(mpmath, v):
    """A long double as an exact mpf: its 64-bit mantissa is the sum of two doubles."""
    hi = float(v)
    return mpmath.mpf(hi) + mpmath.mpf(float(v - np.longdouble(hi)))


@pytest.mark.parametrize('size', [64, 128])
def test_long_double_oracle_matches_mpmath(size):
    mpmath = pytest.importorskip('mpmath')
    mpmath.mp.dps = 40
    x = FO.spread_signal((3, 2 * size), size, size, zero_runs=False)
    X = FO.stft(x, size, size // 2, fading=False)
    w = TO.analysis_window(size)
    frames = FO._frames(x, size, size // 2, size, False, True)[0, :2]  # two frames of the first row
    W = [mpmath.expjpi(-mpmath.mpf(2 * j) / size) for j in range(size)]
    for t, fr in enumerate(frames):
        v = [mpmath.mpf(float(a)) * mpmath.mpf(float(b)) for a, b in zip(fr, w)]
        nrm2, err2 = mpmath.mpf(0), mpmath.mpf(0)
        for k in range(size // 2 + 1):
            ref = mpmath.fsum(v[j] * W[(j * k) % size] for j in range(size))
            got = mpmath.mpc(_mp(mpmath, X[0, t, k].real), _mp(mpmath, X[0, t, k].imag))
            err2 += abs(got - ref) ** 2
            nrm2 += abs(ref) ** 2
        assert float(mpmath.sqrt(err2 / nrm2)) < 1e-17


@pytest.mark.parametrize('size', SIZES)
def test_model_forward_within_half_the_bound(size):
    worst = 0.0
    for shift, wl in ((size // 4, size), (1, 63), (size - 1, size - 1), (1, 1)):
        n = 24 * size if shift > 1 else wl + 300
        for fading, pad in ((True, True), (False, False)):
            x = FO.spread_signal((2, n), wl, size + shift)
            ratio, _ = FO.forward_ratio(FO.model_stft(x, size, shift, wl, fading, pad),
                                           FO.stft(x, size, shift, wl, fading, pad), size)
            worst = max(worst, ratio.max())
    print(f'size {size}: model forward ratio {worst:.3f} (bound C_F = {FO.C_F})')
    assert worst <= 0.5


@pytest.mark.parametrize('size', SIZES)
def test_model_inverse_within_half_the_bound(size):
    rng = np.random.default_rng(size)
    worst = 0.0
    for shift, wl in ((1, size), (3, size - 1), (size // 4, size), (size, size), (1, 63), (3, 63), (1, 1)):
        T = 12 if shift > 3 else min(size, 256) + 24                  # shift = 1: min(wl, T) frames per sample
        X = rng.standard_normal((2, T, size // 2 + 1)) + 1j * rng.standard_normal((2, T, size // 2 + 1))
        X *= 10.0 ** (-6 * rng.random((2, T, 1)))                    # 120 dB between frames
        X[:, 3] = 0
        for fading in (True, False):
            ref, scale = FO.istft_parts(X, size, shift, wl, fading)
            ratio = FO.inverse_ratio(FO.model_istft(X, size, shift, wl, fading), ref, scale, size)
            worst = max(worst, ratio.max(initial=0.0))
    print(f'size {size}: model inverse ratio {worst:.3f} (C_I = {FO.C_I})')
    assert worst <= 0.5


def test_inverse_constant_is_within_10x_of_the_model():
    rng = np.random.default_rng(0)
    worst = 0.0
    for size in (64, 4096):
        for shift in (size // 4, size):
            X = rng.standard_normal((2, 16, size // 2 + 1)) + 1j * rng.standard_normal((2, 16, size // 2 + 1))
            ref, scale = FO.istft_parts(X, size, shift, size, False)
            worst = max(worst, FO.inverse_ratio(FO.model_istft(X, size, shift, size, False), ref, scale, size).max())
    assert 0.1 <= worst <= 0.5, worst


@pytest.mark.parametrize('size', SIZES)
def test_model_envelope_and_numpy_within_the_bounds(size):
    """The envelope bound against float64 scipy.signal.hilbert (another correct fp64 algorithm), and the forward bound
    against float64 NumPy rfft: both well inside."""
    x = FO.spread_signal((2, 3 * size + 5), size // 4, size)
    a = FO.analytic(x)
    M = 1 << (int(np.ceil(np.log2(2 * x.shape[-1] - 1))))
    for r in range(2):
        assert FO.envelope_ratio(np.abs(scipy.signal.hilbert(x[r])), a[r], M) <= 0.5
    frames = FO._frames(x, size, size // 4, size, True, True) * TO.analysis_window(size)
    ratio, _ = FO.forward_ratio(np.fft.rfft(frames, n=size), FO.stft(x, size, size // 4), size)
    assert ratio.max() <= 0.5


def test_dash_bound_holds_for_the_model():
    """One Griffin-Lim step with the model's X'' and X' = |X| X''/|X''| in float64: within the per-bin bound."""
    size, shift = 256, 64
    rng = np.random.default_rng(1)
    x_hat = FO.spread_signal((3, 4000), size, 2)
    T = TO.num_frames(4000, size, shift, size, True, True)
    X = rng.standard_normal((3, T, size // 2 + 1)) + 1j * rng.standard_normal((3, T, size // 2 + 1))
    Xdd_ref, Xd_ref = FO.griffin_lim_step(x_hat, X, None, size, shift, True)
    Xdd = FO.model_stft(x_hat, size, shift, fading=True)
    h = np.abs(Xdd)
    Xd = np.abs(X) * np.where(h > 0, Xdd / np.where(h > 0, h, 1), 1)
    assert FO.forward_ratio(Xdd, Xdd_ref, size)[0].max() <= 0.5
    assert FO.dash_ratio(Xd, X, Xdd_ref, size).max() <= 0.5
    zero = np.abs(Xdd_ref).sum(-1) == 0
    assert zero.any()
    np.testing.assert_array_equal(Xd[zero], np.abs(X[zero]) + 0j)


def _rule(size, rows, frames, sms):
    fpc = 4096 // size
    while fpc > 1 and rows * -(-frames // fpc) < 2 * sms:
        fpc //= 2
    return fpc


@pytest.mark.parametrize('sms', [114, 132, 16])
def test_frames_per_cta_rule(sms):
    from pb_bss_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(sms)
    for size in SIZES:
        for _ in range(200):
            rows, frames = int(rng.integers(1, 600)), int(rng.integers(1, 3000))
            assert lib.pbb_stft_frames_per_cta(size, rows, frames, sms) == _rule(size, rows, frames, sms)
        assert lib.pbb_stft_frames_per_cta(size, 1 << 20, 1 << 20, sms) == 4096 // size
        assert lib.pbb_stft_frames_per_cta(size, 1, 1, sms) == 1
    # the boundary of the largest tile: rows * ceil(frames / fpc) reaching 2 sms
    assert lib.pbb_stft_frames_per_cta(64, 2 * sms, 64, sms) == 64
    assert lib.pbb_stft_frames_per_cta(64, 2 * sms - 1, 64, sms) == 32
    assert lib.pbb_stft_frames_per_cta(1024, 1, 8 * sms, sms) == 4
    assert lib.pbb_stft_frames_per_cta(1024, 1, 8 * sms - 4, sms) == 2


def test_frames_per_cta_depends_on_the_sm_count():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    # 240 rows of 2 frames at size 128: 240 CTAs give a PCIe part (114 SMs) two each at fpc = 32; an SXM (132 SMs)
    # falls to fpc = 1, where 480 CTAs are enough
    assert lib.pbb_stft_frames_per_cta(128, 240, 2, 114) == 32
    assert lib.pbb_stft_frames_per_cta(128, 240, 2, 132) == 1


def test_frames_per_cta_rejects_bad_arguments():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    assert lib.pbb_stft_frames_per_cta(100, 1, 1, 132) == -1
    assert lib.pbb_stft_frames_per_cta(8192, 1, 1, 132) == -1
    assert lib.pbb_stft_frames_per_cta(256, 0, 1, 132) == -2
    assert lib.pbb_stft_frames_per_cta(256, 1, 0, 132) == -3
    assert lib.pbb_stft_frames_per_cta(256, 1, 1, 0) == -4
