"""The STFT / iSTFT and the Griffin-Lim / MISI iteration of pb_bss_b200.transform on the device against the NumPy
restatement of the contract (oracle/transform_oracle.py) and against the unmodified reference's GriffinLim / MISI
(tests/golden/transform.npz), plus one audio-to-audio separation pipeline."""
import numpy as np
import pytest
import scipy.signal

from conftest import cos_similarity
from oracle import pb_bss_oracle as O
from oracle import synth
from oracle import transform_oracle as TO

pytestmark = pytest.mark.gpu

SIZES = [64, 128, 256, 512, 1024, 2048, 4096]


def _signal(shape, seed, dtype=np.float64):
    return np.random.default_rng(seed).standard_normal(shape).astype(dtype)


def _assert_rows_close(out, ref, rel=1e-12):
    """atol = rel * max|X| of each row (the frames and bins of one signal)."""
    assert out.shape == ref.shape and out.dtype == ref.dtype
    r = ref.reshape(-1, ref.shape[-2] * ref.shape[-1]) if ref.ndim >= 2 else ref[None]
    o = out.reshape(r.shape)
    scale = np.maximum(np.abs(r).max(axis=-1, keepdims=True), 1e-300)
    assert (np.abs(o - r) <= rel * scale).all(), np.max(np.abs(o - r) / scale)


@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('div', [2, 4, 8])
def test_stft_matches_oracle(size, div):
    from pb_bss_b200.transform import stft
    x = _signal((3, 6 * size + 17), size + div)
    _assert_rows_close(stft(x, size=size, shift=size // div), TO.stft(x, size=size, shift=size // div))


@pytest.mark.parametrize('fading,pad', [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize('size,shift,wl', [(256, 100, None), (512, 128, 400), (1024, 256, 1000), (64, 7, 50)])
def test_stft_options_match_oracle(fading, pad, size, shift, wl):
    from pb_bss_b200.transform import stft
    x = _signal((2, 5000), shift)
    for sym in (False, True):
        kw = dict(size=size, shift=shift, window_length=wl, fading=fading, pad=pad, symmetric_window=sym)
        _assert_rows_close(stft(x, **kw), TO.stft(x, **kw))


def test_stft_float32_leading_dims_axis_and_short_signals():
    import torch
    from pb_bss_b200.transform import stft
    x = _signal((2, 3, 3001), 5)
    for dt in (np.float64, np.float32):
        _assert_rows_close(stft(x.astype(dt), size=512, shift=128), TO.stft(x.astype(dt), size=512, shift=128))
    xa = np.ascontiguousarray(np.moveaxis(x, -1, 1))                  # (2, n, 3), axis = 1
    out = stft(xa, size=256, shift=64, axis=1)
    ref = TO.stft(xa, size=256, shift=64, axis=1)
    assert out.shape == ref.shape == (2, 50, 129, 3)
    _assert_rows_close(np.moveaxis(out, 3, 1), np.moveaxis(ref, 3, 1))
    for n in (1, 10, 255, 256, 257):                                   # shorter than (or about) one window
        s = _signal((2, n), n)
        for fading in (True, False):
            _assert_rows_close(stft(s, size=256, shift=64, fading=fading), TO.stft(s, size=256, shift=64,
                                                                                  fading=fading))
    t = stft(torch.from_numpy(x).cuda().float(), size=512, shift=128)
    assert t.is_cuda and t.dtype == torch.complex128
    _assert_rows_close(t.cpu().numpy(), TO.stft(x.astype(np.float32), size=512, shift=128))


@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('div', [2, 4, 8])
def test_istft_matches_oracle(size, div):
    from pb_bss_b200.transform import istft
    rng = np.random.default_rng(size * div)
    X = rng.standard_normal((2, 11, size // 2 + 1)) + 1j * rng.standard_normal((2, 11, size // 2 + 1))
    for fading in (True, False):
        ref = TO.istft(X, size=size, shift=size // div, fading=fading)
        out = istft(X, size=size, shift=size // div, fading=fading)
        assert out.shape == ref.shape
        np.testing.assert_allclose(out, ref, rtol=0, atol=1e-12 * np.abs(ref).max())


def test_istft_window_length_and_non_dividing_shift():
    from pb_bss_b200.transform import istft
    rng = np.random.default_rng(3)
    for size, shift, wl in ((256, 100, None), (512, 128, 400), (1024, 200, 1000)):
        X = rng.standard_normal((3, 9, size // 2 + 1)) + 1j * rng.standard_normal((3, 9, size // 2 + 1))
        for sym in (False, True):
            kw = dict(size=size, shift=shift, window_length=wl, symmetric_window=sym)
            ref = TO.istft(X, **kw)
            np.testing.assert_allclose(istft(X, **kw), ref, rtol=0, atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize('size,shift', [(256, 128), (256, 64), (256, 32), (256, 100), (1024, 256), (4096, 512)])
def test_perfect_reconstruction_on_the_device(size, shift):
    import torch
    from pb_bss_b200.transform import istft, stft
    x = torch.from_numpy(_signal((2, 20000), shift)).cuda()
    y = istft(stft(x, size=size, shift=shift), size=size, shift=shift)
    assert y.is_cuda and y.shape[-1] >= x.shape[-1]
    err = (y[..., :x.shape[-1]] - x).abs().max().item()
    assert err <= 1e-12 * x.abs().max().item(), err


def test_transforms_are_bitwise_reproducible():
    import torch
    from pb_bss_b200.transform import istft, stft
    x = torch.from_numpy(_signal((8, 40000), 9)).cuda()
    a, b = stft(x, size=1024, shift=256), stft(x, size=1024, shift=256)
    assert torch.equal(a, b)
    assert torch.equal(istft(a, size=1024, shift=256), istft(b, size=1024, shift=256))


def test_errors():
    from pb_bss_b200.transform import istft, stft
    x = _signal(4000, 1)
    for size in (100, 32, 8192, 768):
        with pytest.raises(ValueError, match='power of two'):
            stft(x, size=size, shift=16)
    with pytest.raises(ValueError, match='shift'):
        stft(x, size=256, shift=300)
    with pytest.raises(AssertionError):
        istft(np.zeros((4, 128), np.complex128), size=256, shift=64)
    with pytest.raises(TypeError):
        stft(x.astype(np.complex128), size=256, shift=64)


@pytest.mark.parametrize('name,guess,misi', [('gl', 'istft', False), ('gl_y', 'y', False),
                                             ('misi', 'istft', True), ('misi_y', 'y', True)])
def test_griffin_lim_and_misi_match_the_reference(golden, name, guess, misi):
    from pb_bss_b200.transform import MISI, GriffinLim
    g = golden('transform')
    m = (MISI if misi else GriffinLim)(g['X'], g['y'], first_guess=guess, size=128, shift=32)
    for _ in range(5):
        m.step()
    assert isinstance(m.x_hat, np.ndarray)
    np.testing.assert_allclose(m.x_hat, g[name + '_x_hat'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(m.X_dash, g[name + '_X_dash'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(m.X_dash_dash, g[name + '_X_dash_dash'], rtol=1e-10, atol=1e-12)


def test_misi_with_fading_and_tensor_io(golden):
    import torch
    from pb_bss_b200.transform import MISI
    g = golden('transform')
    m = MISI(torch.from_numpy(g['X_fading']).cuda(), torch.from_numpy(g['y_fading']).cuda(), size=128, shift=32,
             fading=True)
    for _ in range(5):
        m.step()
    assert m.x_hat.is_cuda and m.X_dash.is_cuda and m.X_dash_dash.is_cuda
    np.testing.assert_allclose(m.x_hat.cpu().numpy(), g['misi_fading_x_hat'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(m.X_dash.cpu().numpy(), g['misi_fading_X_dash'], rtol=1e-10, atol=1e-12)


def test_first_guess_branches_and_errors(golden):
    from pb_bss_b200.transform import MISI, GriffinLim
    g = golden('transform')
    X, y = g['X'], g['y']
    np.testing.assert_allclose(GriffinLim(X, first_guess='istft', size=128, shift=32).x_hat,
                               TO.istft(X, size=128, shift=32, fading=False), rtol=0, atol=1e-12 * np.abs(X).max())
    np.testing.assert_array_equal(GriffinLim(X, y, first_guess='y', size=128, shift=32).x_hat,
                                  np.repeat(y[None, :] / 3, 3, axis=0))
    with pytest.raises(TypeError):
        GriffinLim(X, y, first_guess='white_gaussian_noise', size=128, shift=32)
    with pytest.raises(ValueError):
        GriffinLim(X, y, first_guess='zeros', size=128, shift=32)
    m = MISI(X, y[:-5], size=128, shift=32)
    with pytest.raises(ValueError):
        m.step()


def _sources(K, D, n, seed):
    """Mixture of K sources with on/off envelopes (time-frequency sparsity) through random 32-tap filters."""
    rng = np.random.default_rng(seed)
    env = np.repeat(rng.random((K, n // 800 + 1)) > 0.4, 800, axis=1)[:, :n]
    s = rng.standard_normal((K, n)) * env
    h = rng.standard_normal((D, K, 32)) * np.exp(-np.arange(32) / 6)
    return np.stack([sum(scipy.signal.lfilter(h[d, k], 1, s[k]) for k in range(K)) for d in range(D)])


def _oracle_pipeline(y, init, iterations, stft_size):
    model = O.cacgmm_fit(y, init, iterations)
    aff = O.cacgmm_predict(y, model)                       # (F, K, T)
    plan = O.dhtv_plan_from_stft_size(stft_size)
    mask = np.ascontiguousarray(aff.transpose(1, 0, 2))
    mapping = O.dhtv_calculate_mapping(mask, plan)
    aligned = O.apply_mapping(mask, mapping).transpose(1, 0, 2)
    Y = np.ascontiguousarray(np.swapaxes(y, -1, -2))
    psd = O.power_spectral_density(Y, aligned)
    noise = psd.sum(1, keepdims=True) - psd
    vec = O.gev_vector(psd, noise)
    enh = O.apply_beamforming_vector(vec.transpose(1, 0, 2), Y[None])
    return aligned, mapping, vec, enh.transpose(1, 0, 2)


def test_audio_to_audio_pipeline_matches_the_host_chain():
    """time signal -> device stft -> CACGMMTrainer.fit -> predict -> DHTV -> PSD -> GEV -> apply -> device istft,
    against the same chain with the oracle's transforms on the host.  GEV vectors are defined up to a phase per bin,
    so the separated spectra are compared in magnitude and the device iSTFT against the oracle's iSTFT of the same
    device spectrum."""
    import torch
    from pb_bss_b200.parallel import sharded_separation
    from pb_bss_b200.transform import istft, stft
    K, D, n, size, shift, I = 3, 6, 16000, 512, 128, 12
    x = _sources(K, D, n, seed=4)
    X_ref = TO.stft(x, size=size, shift=shift)                             # (D, T, F)
    X = stft(torch.from_numpy(x).cuda(), size=size, shift=shift)
    _assert_rows_close(X.cpu().numpy(), X_ref)
    F, T = X_ref.shape[-1], X_ref.shape[-2]
    init = synth.init_affiliation(F, K, T, seed=3)
    y_ref = np.ascontiguousarray(X_ref.transpose(2, 1, 0))                 # (F, T, D)
    aligned, mapping, vec, enh = _oracle_pipeline(y_ref, init, I, size)
    out = sharded_separation(X.permute(2, 1, 0).contiguous(), torch.from_numpy(init).cuda(), F, iterations=I,
                             stft_size=size)
    np.testing.assert_array_equal(out['mapping'].cpu().numpy(), mapping)
    np.testing.assert_allclose(out['affiliation'].cpu().numpy(), aligned, rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(cos_similarity(out['vectors'].cpu().numpy(), vec), 1, atol=1e-7)
    enh_dev = out['enhanced'].permute(1, 2, 0).contiguous()                # (K, T, F)
    np.testing.assert_allclose(np.abs(enh_dev.cpu().numpy()), np.abs(enh.transpose(1, 2, 0)), rtol=1e-5, atol=1e-8)
    audio = istft(enh_dev, size=size, shift=shift)
    assert audio.is_cuda and audio.shape[0] == K and audio.shape[-1] >= n
    ref_audio = TO.istft(enh_dev.cpu().numpy(), size=size, shift=shift)
    np.testing.assert_allclose(audio.cpu().numpy(), ref_audio, rtol=0, atol=1e-12 * np.abs(ref_audio).max())
