"""GPU checks of ESTOI (pb_bss_b200.evaluation.stoi with extended=True, pbb_estoi): agreement with the NumPy
restatement (oracle/estoi_oracle.py) at 8 to 48 kHz over lengths from the shortest valid signal to 2^22 samples, the
stages it shares with STOI bit for bit, its invariances and range, silent estimates, non-finite samples, broadcasting
and input types, bitwise reproducibility across batches and groups, the < 30-frame warning and every error."""
import warnings

import numpy as np
import pytest

from oracle import estoi_oracle as E
from test_stoi_gpu import CASES, _cuda, _signals, speech_like

pytestmark = pytest.mark.gpu

ATOL = 1e-13   # the value is a mean of d_m in [-1, 1]


@pytest.mark.parametrize('i', range(len(CASES)), ids=[f'{fs}-{n}-{len(g)}' for fs, n, g in CASES])
def test_matches_the_oracle(i):
    from pb_bss_b200.evaluation import module_stoi as M
    fs, n, gaps = CASES[i]
    x, y = _signals(fs, n, gaps, i)
    with warnings.catch_warnings(record=True):
        warnings.simplefilter('always')
        ref = E.stages(x, y, fs)
        st = M._stages(_cuda(x[None]), _cuda(y[None]), fs, extended=True)
    K, Mr = st['frames'][0].tolist()
    assert (K, Mr) == (ref['K'], ref['M'])
    v = float(st['value'][0])
    if Mr < 30:
        assert v == 1e-5 and ref['value'] == 1e-5
    else:
        assert abs(v - ref['value']) <= ATOL, (v, ref['value'])


@pytest.mark.parametrize('fs', [8000, 16000, 44100])
def test_shares_the_stoi_stages_bit_for_bit(fs):
    from pb_bss_b200.evaluation import module_stoi as M
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(fs)
    pairs = [speech_like(rng, 3 * fs, fs, gaps) for gaps in ((), ((0.2, 0.4),), ((0.0, 0.95),))]
    X, Y = _cuda(np.stack([p[0] for p in pairs])), _cuda(np.stack([p[1] for p in pairs]))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        a = M._stages(X, Y, fs)
        b = M._stages(X, Y, fs, extended=True)
        for k in ('frames', 'resampled', 'energies'):
            assert a[k].equal(b[k]), k
        assert a['value'][2].item() == b['value'][2].item() == 1e-5
        assert not a['value'][:2].equal(b['value'][:2])
        # extended=False is the default call, bit for bit
        np.testing.assert_array_equal(stoi(X, Y, fs, extended=False).cpu().numpy(), stoi(X, Y, fs).cpu().numpy())
        np.testing.assert_array_equal(stoi(X, Y, fs, False).cpu().numpy(), a['value'].cpu().numpy())


def test_identical_signals_give_one_and_values_lie_in_minus_one_to_one():
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(1)
    for fs in (8000, 16000, 48000):
        x, y = speech_like(rng, 5 * fs, fs, ((0.3, 0.4),))
        assert abs(stoi(x, x, fs, extended=True) - 1.0) <= ATOL
        v = stoi(np.stack([x, x, x]), np.stack([y, -y, rng.standard_normal(x.size)]), fs, extended=True)
        assert np.all(np.abs(v) <= 1.0)
        assert abs(v[0] - E.stoi(x, y, fs, extended=True)) <= ATOL


@pytest.mark.parametrize('fs', [10000, 16000])
def test_estimate_silent_over_many_frames(fs):
    """The estimate is digital silence over about 100 kept frames: all-zero band rows, and at both ends of the silence
    a segment with one non-zero frame, whose constant columns normalise to zeros."""
    from pb_bss_b200.evaluation import module_stoi as M
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(fs + 1)
    x, y = speech_like(rng, 3 * fs, fs)
    y[fs:fs + 3 * fs // 2] = 0.0
    ref = E.stages(x, y, fs)
    st = M._stages(_cuda(x[None]), _cuda(y[None]), fs, extended=True)
    e = st['energies'][0, 1].cpu().numpy()[:, :ref['M']]
    assert np.sum(np.all(e == 0.0, axis=0)) >= 30
    assert np.isfinite(ref['value'])
    assert abs(float(st['value'][0]) - ref['value']) <= ATOL
    assert abs(stoi(x, y, fs, extended=True) - ref['value']) <= ATOL
    # the whole estimate silent: every segment normalises to zeros
    assert stoi(x, np.zeros_like(y), fs, extended=True) == 0.0 == E.stoi(x, np.zeros_like(y), fs, extended=True)


@pytest.mark.parametrize('bad', [np.nan, np.inf])
@pytest.mark.parametrize('fs', [10000, 16000])
def test_non_finite_samples_follow_the_oracle(bad, fs):
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(11)
    x, y = speech_like(rng, 2 * fs, fs)
    xb = x.copy()
    xb[fs // 2] = bad
    with pytest.warns(RuntimeWarning):
        assert E.stoi(xb, y, fs, extended=True) == 1e-5
    with pytest.warns(RuntimeWarning):
        assert stoi(xb, y, fs, extended=True) == 1e-5
    yb = y.copy()
    yb[fs // 2] = bad
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        want = E.stoi(x, yb, fs, extended=True)
    got = stoi(x, yb, fs, extended=True)
    assert np.isnan(want) and np.isnan(got)


def test_types_and_shapes():
    import torch
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(5)
    x, y = speech_like(rng, 16000, 16000)
    v = stoi(x, y, 16000, extended=True)
    assert type(v) is np.float64
    assert abs(v - E.stoi(x, y, 16000, extended=True)) <= ATOL
    t = stoi(_cuda(x), y, 16000, extended=True)
    assert isinstance(t, torch.Tensor) and t.is_cuda and t.shape == () and t.dtype == torch.float64
    assert float(t) == v
    # float32 and int16 are computed in fp64 from their values
    x32, y32 = x.astype(np.float32), y.astype(np.float32)
    want = E.stoi(x32.astype(np.float64), y32.astype(np.float64), 16000, extended=True)
    assert abs(stoi(x32, y32, 16000, extended=True) - want) <= ATOL
    assert stoi(x32, y32, 16000, extended=True) == stoi(_cuda(x32), _cuda(y32), 16000, extended=True).item()
    xi = np.round(x / np.abs(x).max() * 20000).astype(np.int16)
    yi = np.round(y / np.abs(y).max() * 20000).astype(np.int16)
    want = E.stoi(xi.astype(np.float64), yi.astype(np.float64), 16000, extended=True)
    assert abs(stoi(xi, yi, 16000, extended=True) - want) <= ATOL
    assert stoi(x32, y, 16000, extended=True) == stoi(x32.astype(np.float64), y, 16000, extended=True)
    # 3-D broadcasting, and an empty leading dim
    X = np.stack([x, y])[:, None]
    Y = np.stack([y, x, 0.5 * y])[None]
    out = stoi(X, Y, 16000, extended=True)
    assert isinstance(out, np.ndarray) and out.shape == (2, 3) and out.dtype == np.float64
    for a in range(2):
        for b in range(3):
            assert out[a, b] == stoi(X[a, 0], Y[0, b], 16000, extended=True)
    t = stoi(_cuda(X), _cuda(Y), 16000, extended=True)
    assert t.is_cuda and t.shape == (2, 3) and t.dtype == torch.float64
    np.testing.assert_array_equal(t.cpu().numpy(), out)
    e = stoi(np.zeros((0, 16000)), np.zeros((0, 16000)), 16000, extended=True)
    assert e.shape == (0,)


def test_rows_do_not_depend_on_the_batch_or_the_grouping(monkeypatch):
    from pb_bss_b200.evaluation import module_stoi as M
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(7)
    pairs = [speech_like(rng, 48000, 16000, gaps) for gaps in ((), ((0.1, 0.3),), ((0.0, 0.9),), ())]
    X = np.stack([p[0] for p in pairs])
    Y = np.stack([p[1] for p in pairs])
    Y[3, 8000:30000] = 0.0
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        batch = stoi(X, Y, 16000, extended=True)
        alone = np.array([stoi(X[i], Y[i], 16000, extended=True) for i in range(4)])
        np.testing.assert_array_equal(batch, alone)
        per_row = M._lib.load().pbb_stoi_workspace_bytes(1, 48000, *M.rates(16000))
        for g in (1, 3):
            monkeypatch.setattr(M, 'WORKSPACE_BYTES', per_row * g)
            np.testing.assert_array_equal(stoi(X, Y, 16000, extended=True), batch)
        np.testing.assert_array_equal(stoi(X, Y, 16000, extended=True), batch)
    assert batch[2] == 1e-5
    for i in (0, 1, 3):
        assert abs(batch[i] - E.stoi(X[i], Y[i], 16000, extended=True)) <= ATOL


def test_fewer_than_thirty_frames_warns_and_gives_1e_5():
    import torch
    from pb_bss_b200 import _device
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(3)
    x, y = rng.standard_normal(256 + 128 * 30), rng.standard_normal(256 + 128 * 30)   # M = 29
    with pytest.warns(RuntimeWarning, match='Not enough STFT frames'):
        assert stoi(x, y, 10000, extended=True) == 1e-5
    X, Y = rng.standard_normal((3, 8000)), rng.standard_normal((3, 8000))
    X[1, 2000:] = 0.0                      # about 16 frames kept
    with pytest.warns(RuntimeWarning, match='row 1'):
        v = stoi(X, Y, 10000, extended=True)
    assert v[1] == 1e-5 and v[0] != 1e-5 and v[2] != 1e-5
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        with _device.deferred_status():
            t = stoi(_cuda(x), _cuda(y), 10000, extended=True)
            assert isinstance(t, torch.Tensor)
            assert not [m for m in w if issubclass(m.category, RuntimeWarning)]
        assert len([m for m in w if issubclass(m.category, RuntimeWarning)]) == 1
    assert t.item() == 1e-5


def test_errors():
    from pb_bss_b200.evaluation import stoi
    x = np.zeros(4000)
    with pytest.raises(TypeError):
        stoi(_cuda(x.astype(np.complex128)), _cuda(x), 8000, extended=True)
    with pytest.raises(TypeError):
        stoi(x, x.astype(np.complex64), 8000, extended=True)
    with pytest.raises(ValueError):
        stoi(_cuda(np.zeros((2, 4000))), _cuda(np.zeros((3, 4000))), 8000, extended=True)
    with pytest.raises(ValueError):
        stoi(_cuda(np.zeros(200)), _cuda(np.zeros(200)), 8000, extended=True)
    with pytest.raises(ValueError):
        stoi(np.float64(1.0), np.float64(1.0), 8000, extended=True)
    for fs in (0, -8000, 8000.5, True):
        with pytest.raises(ValueError):
            stoi(x, x, fs, extended=True)

