"""CPU checks of the NumPy restatement of the STFT / iSTFT contract (oracle/transform_oracle.py) and of its
Griffin-Lim / MISI iteration against the unmodified reference (tests/golden/transform.npz)."""
import numpy as np
import pytest
import scipy.signal

from oracle import transform_oracle as TO


def _explicit_stft(x, size, shift, wl, fading, pad, symmetric):
    """Pad, frame, window and np.fft.rfft one 1-D signal, frame by frame."""
    w = scipy.signal.windows.blackman(wl) if symmetric else scipy.signal.windows.blackman(wl + 1)[:-1]
    if fading:
        x = np.concatenate([np.zeros(wl - shift), x, np.zeros(wl - shift)])
    if pad:  # zeros at the end until the frames tile the signal exactly
        while len(x) < wl or (len(x) - wl) % shift:
            x = np.append(x, 0.0)
    frames = [np.fft.rfft(x[s:s + wl] * w, n=size) for s in range(0, len(x) - wl + 1, shift)]
    return np.array(frames).reshape(-1, size // 2 + 1)


@pytest.mark.parametrize('size,shift,wl', [(64, 16, None), (256, 100, None), (256, 64, 200), (512, 128, None)])
@pytest.mark.parametrize('fading,pad', [(True, True), (False, True), (False, False), (True, False)])
@pytest.mark.parametrize('length', [37, 1000, 1001])
def test_oracle_stft_is_the_explicit_frame_loop(size, shift, wl, fading, pad, length):
    x = np.random.default_rng(length).standard_normal(length)
    w = wl or size
    for symmetric in (False, True):
        ref = _explicit_stft(x, size, shift, w, fading, pad, symmetric)
        out = TO.stft(x, size=size, shift=shift, window_length=wl, fading=fading, pad=pad, symmetric_window=symmetric)
        assert out.shape == ref.shape
        np.testing.assert_allclose(out, ref, rtol=0, atol=1e-12 * max(1.0, np.abs(ref).max(initial=0)))


def test_oracle_stft_axis_and_leading_dims():
    x = np.random.default_rng(1).standard_normal((2, 3, 700))
    X = TO.stft(x, size=128, shift=32)
    assert X.shape == (2, 3, 25, 65)
    Xa = TO.stft(np.moveaxis(x, -1, 1), size=128, shift=32, axis=1)
    assert Xa.shape == (2, 25, 65, 3)
    np.testing.assert_array_equal(np.moveaxis(Xa, 3, 1), X)
    assert TO.stft(x.astype(np.float32), size=128, shift=32).dtype == np.complex128


@pytest.mark.parametrize('size,shift', [(256, 128), (256, 64), (256, 32), (256, 100), (1024, 256), (64, 8)])
def test_oracle_perfect_reconstruction(size, shift):
    x = np.random.default_rng(size + shift).standard_normal((2, 3000))
    y = TO.istft(TO.stft(x, size=size, shift=shift), size=size, shift=shift)
    assert y.shape[-1] >= x.shape[-1]
    np.testing.assert_allclose(y[..., :x.shape[-1]], x, rtol=0, atol=1e-12 * np.abs(x).max())


def test_oracle_synthesis_window_is_biorthogonal():
    for wl, shift in ((256, 64), (256, 100), (200, 64)):
        wa = TO.analysis_window(wl)
        ws = TO.synthesis_window(wa, shift)
        # sum over the frames covering one sample of w_a * w_s = 1
        tot = np.zeros(wl)
        for i in range(-((wl - 1) // shift), (wl - 1) // shift + 1):
            s = i * shift
            tot[max(s, 0):wl + min(s, 0)] += (wa * ws)[max(-s, 0):wl - max(s, 0)]
        np.testing.assert_allclose(tot, 1, rtol=1e-12)


@pytest.mark.parametrize('name,guess,misi', [('gl', 'istft', False), ('gl_y', 'y', False),
                                             ('misi', 'istft', True), ('misi_y', 'y', True)])
def test_oracle_griffin_lim_matches_reference(golden, name, guess, misi):
    g = golden('transform')
    x_hat, X_dash, X_dash_dash = TO.griffin_lim(g['X'], g['y'], guess, size=128, shift=32, steps=5, misi=misi)
    np.testing.assert_allclose(x_hat, g[name + '_x_hat'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(X_dash, g[name + '_X_dash'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(X_dash_dash, g[name + '_X_dash_dash'], rtol=1e-10, atol=1e-12)


def test_oracle_misi_with_fading_matches_reference(golden):
    g = golden('transform')
    x_hat, X_dash, _ = TO.griffin_lim(g['X_fading'], g['y_fading'], size=128, shift=32, fading=True, steps=5,
                                      misi=True)
    np.testing.assert_allclose(x_hat, g['misi_fading_x_hat'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(X_dash, g['misi_fading_X_dash'], rtol=1e-10, atol=1e-12)
