"""GPU checks of STOI (pb_bss_b200.evaluation.stoi): the numbers the reference publishes, agreement with the NumPy
restatement (oracle/stoi_oracle.py) at 8 to 48 kHz over lengths from the shortest valid signal to 2^22 samples,
every stage (resampled signals, frame counts, band energies), broadcasting and input types, bitwise
reproducibility across batches and groups, the < 30-frame warning and every error."""
import warnings

import numpy as np
import pytest
import scipy.signal

from oracle import stoi_oracle as O
from oracle.make_golden_bss_eval import input_signals

pytestmark = pytest.mark.gpu

RATES = (8000, 10000, 16000, 22050, 44100, 48000)
ATOL = 1e-13   # d is in [-1, 1]; the largest difference measured on the H100 is 6.7e-16


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _length_at_least(L, fs):
    """The smallest n whose length at 10 kHz is at least L."""
    up, down = O.rates(fs)
    n = max(1, (L - 1) * down // up)
    while O.resampled_length(n, fs) < L:
        n += 1
    return n


def _length_for(L, fs):
    """The smallest n whose length at 10 kHz is L, or None."""
    n = _length_at_least(L, fs)
    return n if O.resampled_length(n, fs) == L else None


def speech_like(rng, n, fs, gaps=()):
    """AR(2)-coloured noise under a 3 Hz envelope spanning about 42 dB (frames fall on both sides of the 40 dB
    threshold), zero over the fractions `gaps`; the estimate is the reference through a short filter plus noise.
    Asserts that no frame energy lies within 1e-9 dB of the threshold, so the keep mask is not a rounding decision."""
    t = np.arange(n) / fs
    env = (1.2 + np.sin(2 * np.pi * 3 * t + rng.uniform(0, 6))) ** 2
    x = scipy.signal.lfilter([1.0], [1.0, -1.3, 0.6], rng.standard_normal(n)) * env
    for a, b in gaps:
        x[int(a * n):int(b * n)] = 0.0
    y = scipy.signal.lfilter([1.0, 0.4, -0.2], [1.0], x) + 0.5 * rng.standard_normal(n) * np.sqrt(env)
    xr = O.resample(x, fs)
    if O.num_frames(len(xr)):
        e = 20 * np.log10(np.linalg.norm(O._frames(xr), axis=1) + O.EPS)
        assert np.all(np.abs(e - (e.max() - O.DYN_RANGE)) > 1e-9)
    return x, y


def _cases():
    out = []
    for fs in RATES:
        out.append((fs, _length_at_least(257, fs), ()))          # the shortest valid signal: one frame
        for frames in (29, 30, 31):                    # M = frames STFT frames when every frame is kept
            out.append((fs, _length_at_least(256 + 128 * frames + 64, fs), 'stationary'))
        for k in (40, 41):                             # L - 256 = 128 k, +- 1: the strict frame rule
            for d in (-1, 0, 1):
                n = _length_for(256 + 128 * k + d, fs)
                if n is not None:
                    out.append((fs, n, ()))
        out.append((fs, 10 * fs, ((0.2, 0.3), (0.6, 0.62))))    # 10 s with silent gaps
        out.append((fs, 2 * fs, ((0.0, 0.45), (0.55, 1.0))))    # mostly silent: fewer than 30 frames kept
    out.append((8000, 1 << 22, ((0.5, 0.51),)))
    out.append((44100, 1 << 22, ()))
    return out


CASES = _cases()


def _signals(fs, n, gaps, seed):
    rng = np.random.default_rng(seed)
    if gaps == 'stationary':
        return rng.standard_normal(n), rng.standard_normal(n)
    return speech_like(rng, n, fs, gaps)


def test_input_metrics_anchor(golden):
    import torch
    from pb_bss_b200.evaluation import stoi
    g, b = golden('stoi'), golden('bss_eval')
    ref, est = input_signals(b)
    v = stoi(ref, est, 8000)
    assert isinstance(v, np.ndarray) and v.shape == (2, 3) and v.dtype == np.float64
    np.testing.assert_allclose(v, g['input_stoi'], rtol=float(g['input_rtol']))
    # InputMetrics' broadcasting: (K, 1, T) against (1, D, T)
    src, obs = b['input_source'], b['input_observation']
    np.testing.assert_array_equal(stoi(src[:, None], obs[None], 8000), v)
    t = stoi(_cuda(ref), _cuda(est), 8000)
    assert isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.shape == (2, 3)
    np.testing.assert_array_equal(t.cpu().numpy(), v)


def test_output_metrics_anchor(golden):
    from pb_bss_b200.evaluation import stoi
    g, b = golden('stoi'), golden('bss_eval')
    v = stoi(b['output_reference'], b['output_estimation'], 8000)
    np.testing.assert_allclose(v, g['output_stoi'], rtol=float(g['output_rtol']))
    t = stoi(_cuda(b['output_reference']), _cuda(b['output_estimation']), 8000)
    np.testing.assert_allclose(t.cpu().numpy(), g['output_stoi'], rtol=float(g['output_rtol']))


def test_doctest_anchor(golden):
    from pb_bss_b200.evaluation import stoi
    g, b = golden('stoi'), golden('bss_eval')
    v = stoi(b['doctest_reference'], b['doctest_estimation'], 8000)
    np.testing.assert_array_equal(np.round(v, int(g['doctest_decimals'])), g['doctest_stoi'])
    t = stoi(_cuda(b['doctest_reference']), _cuda(b['doctest_estimation']), 8000)
    np.testing.assert_array_equal(np.round(t.cpu().numpy(), int(g['doctest_decimals'])), g['doctest_stoi'])


@pytest.mark.parametrize('i', range(len(CASES)), ids=[f'{fs}-{n}-{len(g)}' for fs, n, g in CASES])
def test_every_stage_matches_the_oracle(i):
    from pb_bss_b200.evaluation import module_stoi as M
    fs, n, gaps = CASES[i]
    x, y = _signals(fs, n, gaps, i)
    with warnings.catch_warnings(record=True):
        warnings.simplefilter('always')
        ref = O.stages(x, y, fs)
        st = M._stages(_cuda(x[None]), _cuda(y[None]), fs)
    # resampled signals against scipy.signal.resample_poly
    if st['resampled'] is not None:
        r = st['resampled'][0].cpu().numpy()
        np.testing.assert_allclose(r[0], ref['x'], rtol=0, atol=1e-13 * np.abs(x).max())
        np.testing.assert_allclose(r[1], ref['y'], rtol=0, atol=1e-13 * np.abs(y).max())
    else:
        assert fs == 10000
    K, Mr = st['frames'][0].tolist()
    assert (K, Mr) == (ref['K'], ref['M'])
    e =st['energies'][0].cpu().numpy()[:, :, :Mr]
    if Mr >= 30:
        for got, want in ((e[0], ref['x_tob']), (e[1], ref['y_tob'])):
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * want.max())
    v = float(st['value'][0])
    if Mr < 30:
        assert v == 1e-5 and ref['value'] == 1e-5
    else:
        assert abs(v - ref['value']) <= ATOL, (v, ref['value'])


def test_types_and_shapes():
    import torch
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(5)
    x, y = speech_like(rng, 16000, 16000)
    v = stoi(x, y, 16000)
    assert type(v) is np.float64
    assert abs(v - O.stoi(x, y, 16000)) <= ATOL
    t = stoi(_cuda(x), y, 16000)
    assert isinstance(t, torch.Tensor) and t.shape == () and t.dtype == torch.float64
    assert float(t) == v
    # float32 and int16 are computed in fp64 from their values
    x32, y32 = x.astype(np.float32), y.astype(np.float32)
    assert abs(stoi(x32, y32, 16000) - O.stoi(x32.astype(np.float64), y32.astype(np.float64), 16000)) <= ATOL
    assert stoi(x32, y32, 16000) == stoi(_cuda(x32), _cuda(y32), 16000).item()
    xi = np.round(x / np.abs(x).max() * 20000).astype(np.int16)
    yi = np.round(y / np.abs(y).max() * 20000).astype(np.int16)
    assert abs(stoi(xi, yi, 16000) - O.stoi(xi.astype(np.float64), yi.astype(np.float64), 16000)) <= ATOL
    # mixed float32 / float64 pairs are computed from the float64 values of both
    assert stoi(x32, y, 16000) == stoi(x32.astype(np.float64), y, 16000)
    # 3-D broadcasting, and an empty leading dim
    X = np.stack([x, y])[:, None]
    Y = np.stack([y, x, 0.5 * y])[None]
    out = stoi(X, Y, 16000)
    assert out.shape == (2, 3)
    for a in range(2):
        for b in range(3):
            assert out[a, b] == stoi(X[a, 0], Y[0, b], 16000)
    assert stoi(np.zeros((0, 16000)), np.zeros((0, 16000)), 16000).shape == (0,)


def test_rows_do_not_depend_on_the_batch_or_the_grouping(monkeypatch):
    from pb_bss_b200.evaluation import module_stoi as M
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(7)
    pairs = [speech_like(rng, 48000, 16000, gaps) for gaps in ((), ((0.1, 0.3),), ((0.0, 0.9),), ())]
    X = np.stack([p[0] for p in pairs])
    Y = np.stack([p[1] for p in pairs])
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        batch = stoi(X, Y, 16000)
        alone = np.array([stoi(X[i], Y[i], 16000) for i in range(4)])
        np.testing.assert_array_equal(batch, alone)
        per_row = M._lib.load().pbb_stoi_workspace_bytes(1, 48000, *M.rates(16000))
        for g in (1, 3):
            monkeypatch.setattr(M, 'WORKSPACE_BYTES', per_row * g)
            np.testing.assert_array_equal(stoi(X, Y, 16000), batch)
    assert batch[2] == 1e-5


def test_fewer_than_thirty_frames_warns_and_gives_1e_5():
    import torch
    from pb_bss_b200 import _device
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(3)
    x, y = rng.standard_normal(256 + 128 * 30), rng.standard_normal(256 + 128 * 30)   # M = 29
    with pytest.warns(RuntimeWarning, match='Not enough STFT frames'):
        assert stoi(x, y, 10000) == 1e-5
    X, Y = rng.standard_normal((3, 8000)), rng.standard_normal((3, 8000))
    X[1, 2000:] = 0.0                      # about 16 frames kept
    with pytest.warns(RuntimeWarning, match='row 1'):
        v = stoi(X, Y, 10000)
    assert v[1] == 1e-5 and v[0] != 1e-5 and v[2] != 1e-5
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        with _device.deferred_status():
            t = stoi(_cuda(x), _cuda(y), 10000)
            assert isinstance(t, torch.Tensor)
            assert not [m for m in w if issubclass(m.category, RuntimeWarning)]
        assert len([m for m in w if issubclass(m.category, RuntimeWarning)]) == 1
    assert t.item() == 1e-5


@pytest.mark.parametrize('bad', [np.nan, np.inf])
@pytest.mark.parametrize('fs', [10000, 16000])
def test_non_finite_samples_follow_the_oracle(bad, fs):
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(11)
    x, y = speech_like(rng, 2 * fs, fs)
    xb = x.copy()
    xb[fs // 2] = bad
    with pytest.warns(RuntimeWarning):
        assert O.stoi(xb, y, fs) == 1e-5
    with pytest.warns(RuntimeWarning):
        assert stoi(xb, y, fs) == 1e-5
    yb = y.copy()
    yb[fs // 2] = bad
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        want = O.stoi(x, yb, fs)
    got = stoi(x, yb, fs)
    assert np.isnan(want) and np.isnan(got)


def test_errors():
    from pb_bss_b200.evaluation import stoi
    x = np.zeros(4000)
    with pytest.raises(TypeError):
        stoi(_cuda(x.astype(np.complex128)), _cuda(x), 8000)
    with pytest.raises(ValueError):
        stoi(_cuda(np.zeros((2, 4000))), _cuda(np.zeros((3, 4000))), 8000)
    with pytest.raises(ValueError):
        stoi(_cuda(np.zeros(200)), _cuda(np.zeros(200)), 8000)
