"""CPU checks of STOI: the NumPy restatement of pystoi (oracle/stoi_oracle.py) against the numbers the reference
publishes (tests/golden/stoi.npz with the signals of tests/golden/bss_eval.npz), its edge cases, the host-built
tables of pb_bss_b200.evaluation.module_stoi against the oracle's, and the argument checks that raise before any
device work."""
import warnings

import numpy as np
import pytest
import scipy.signal

from oracle import stoi_oracle as O
from oracle.make_golden_bss_eval import input_signals
from pb_bss_b200.evaluation import module_stoi as M

RATES = (8000, 10000, 16000, 22050, 44100, 48000)


def test_input_metrics_anchor(golden):
    g, b = golden('stoi'), golden('bss_eval')
    ref, est = input_signals(b)
    v = O.stoi(ref, est, int(g['sample_rate']))
    assert v.shape == (2, 3)
    np.testing.assert_allclose(v, g['input_stoi'], rtol=float(g['input_rtol']))


def test_output_metrics_anchor(golden):
    g, b = golden('stoi'), golden('bss_eval')
    v = O.stoi(b['output_reference'], b['output_estimation'], int(g['sample_rate']))
    np.testing.assert_allclose(v, g['output_stoi'], rtol=float(g['output_rtol']))


def test_doctest_anchor(golden):
    g, b = golden('stoi'), golden('bss_eval')
    v = O.stoi(b['doctest_reference'], b['doctest_estimation'], int(g['sample_rate']))
    np.testing.assert_array_equal(np.round(v, int(g['doctest_decimals'])), g['doctest_stoi'])


def test_one_dimensional_input_gives_a_scalar(golden):
    b = golden('bss_eval')
    v = O.stoi(b['output_reference'][0], b['output_estimation'][0], 8000)
    assert np.ndim(v) == 0


def test_no_frame_raises_value_error():
    n = 256                               # 256 samples at 10 kHz: 128 f < 0 has no solution
    with pytest.raises(ValueError):
        O.stoi(np.ones(n), np.ones(n), 10000)
    assert O.num_frames(256) == 0 and O.num_frames(257) == 1


@pytest.mark.parametrize('bad', [np.nan, np.inf, -np.inf])
def test_non_finite_reference_drops_every_frame(bad):
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal(8000), rng.standard_normal(8000)
    x[1234] = bad
    with pytest.warns(RuntimeWarning, match='Not enough STFT frames'):
        st = O.stages(x, y, 10000)
    assert st['K'] == 0 and st['M'] == 0 and st['value'] == 1e-5


def test_non_finite_estimate_gives_nan():
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal(8000), rng.standard_normal(8000)
    y[1234] = np.nan
    assert np.isnan(O.stoi(x, y, 10000))


@pytest.mark.parametrize('frames', [29, 30, 31])
def test_thirty_frame_boundary(frames):
    """Stationary noise keeps every frame, so M = F - 1 with F = ceil((L - 256) / 128)."""
    L = 256 + 128 * (frames + 1)
    rng = np.random.default_rng(frames)
    x, y = rng.standard_normal(L), rng.standard_normal(L)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        st = O.stages(x, y, 10000)
    assert st['M'] == frames and st['K'] == frames + 1
    assert (len(w) == 1) == (frames < 30)
    assert (st['value'] == 1e-5) == (frames < 30)


@pytest.mark.parametrize('fs', [r for r in RATES if r != 10000])
def test_polyphase_taps_are_resample_polys_filter(fs):
    """The per-phase table holds exactly window * up after n_pre_pad zeros, and the polyphase sum reproduces
    scipy.signal.resample_poly (the model of stoi_resample_kernel)."""
    up, down = M.rates(fs)
    assert (up, down) == O.rates(fs)
    h = O.resample_window_oct(O.FS, fs)
    w = h / np.sum(h)
    np.testing.assert_array_equal(M.resample_filter(fs), w)
    taps, pre_remove = M.polyphase_taps(fs)
    half_len = (w.size - 1) // 2
    pad = down - half_len % down
    flat = taps.T.reshape(-1)
    np.testing.assert_array_equal(flat[:pad], 0)
    np.testing.assert_array_equal(flat[pad:pad + w.size], w * up)
    np.testing.assert_array_equal(flat[pad + w.size:], 0)
    assert pre_remove == (half_len + pad) // down
    x = np.random.default_rng(fs).standard_normal(3 * fs // 100 + 7)
    ref = scipy.signal.resample_poly(x, O.FS, fs, window=w)
    L = M.resampled_length(x.size, fs)
    assert L == ref.size
    t = (np.arange(L) + pre_remove) * down
    ph, i0 = t % up, t // up
    idx = i0[:, None] - np.arange(taps.shape[1])[None]
    xs = np.where((idx >= 0) & (idx < x.size), x[np.clip(idx, 0, x.size - 1)], 0.0)
    model = np.sum(taps[ph] * xs, axis=1)
    np.testing.assert_allclose(model, ref, rtol=0, atol=1e-13 * np.abs(x).max())


def test_band_edges_and_window():
    np.testing.assert_array_equal(M.band_edges(), O.band_edges())
    assert M.band_edges().dtype == np.int32
    np.testing.assert_array_equal(M.window(), O.window())
    edges = O.band_edges()
    np.testing.assert_array_equal(edges[1:, 0], edges[:-1, 1])


@pytest.mark.parametrize('fs', RATES)
def test_resampled_length(fs):
    for n in (1, 2, 3, 255, 1000, 4097, 160000):
        assert M.resampled_length(n, fs) == O.resampled_length(n, fs)
        if fs != 10000 and n > 1:
            assert M.resampled_length(n, fs) == len(O.resample(np.zeros(n), fs))


def test_bad_arguments_raise_before_device_work():
    x = np.zeros(4000)
    with pytest.raises(TypeError):
        M.stoi(x.astype(complex), x, 8000)
    with pytest.raises(TypeError):
        M.stoi(x, x.astype(np.complex64), 8000)
    with pytest.raises(ValueError):
        M.stoi(np.zeros((2, 4000)), np.zeros((3, 4000)), 8000)
    with pytest.raises(ValueError):
        M.stoi(x, np.zeros(4001), 8000)
    with pytest.raises(ValueError):
        M.stoi(np.zeros(204), np.zeros(204), 8000)        # 255 samples at 10 kHz: no frame
    with pytest.raises(ValueError):
        M.stoi(np.float64(1.0), np.float64(1.0), 8000)
    big = np.broadcast_to(np.float32(0), (M.MAX_SAMPLES + 1,))
    with pytest.raises(ValueError):
        M.stoi(big, big, 10000)
    long = np.broadcast_to(np.float32(0), (M.MAX_SAMPLES,))
    with pytest.raises(ValueError):
        M.stoi(long, long, 4000)                          # 2.5 * 2^22 samples at 10 kHz
    for fs in (0, -8000, 8000.5, True):
        with pytest.raises(ValueError):
            M.stoi(x, x, fs)


def test_abi_rejects_bad_shapes():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    assert lib.pbb_stoi_workspace_bytes(1, 4000, 5, 4) > 0
    assert lib.pbb_stoi_workspace_bytes(1, 204, 5, 4) == 0          # no frame
    assert lib.pbb_stoi_workspace_bytes(1, 4000, 10, 8) == 0        # not in lowest terms
    assert lib.pbb_stoi_workspace_bytes(0, 4000, 5, 4) == 0
    assert lib.pbb_stoi_workspace_bytes(1, M.MAX_SAMPLES + 1, 1, 1) == 0
    rc = lib.pbb_stoi(None, None, _lib.PBB_F64, 1, 4000, 5, 4, None, 0, 0, None, None, None, 1, None, 0, None,
                      None, None, None, None, None)
    assert rc == -1 and b'x is null' in lib.pbb_last_error()
    rc = lib.pbb_stoi(1, 1, _lib.PBB_F64, 1, 204, 5, 4, None, 0, 0, None, None, None, 1, None, 0, None,
                      None, None, None, None, None)
    assert rc == -5
