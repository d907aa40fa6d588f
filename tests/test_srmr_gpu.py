"""pb_bss_b200.evaluation.srmr on the device against the unmodified reference (tests/golden/srmr.npz) and the NumPy
restatement (oracle/srmr_oracle.py): values, VAD lengths and kept samples, Hilbert envelopes across the passes of the
global-memory FFT (csrc/fft_large.cuh), the modulation energies at the frame-count edges, batching and grouping
(bitwise), non-finite input and the limits."""
import numpy as np
import pytest
import scipy.signal

from oracle import srmr_oracle as SO
from oracle.make_golden_srmr import cases as _fixture_cases, signal, vad_output

pytestmark = pytest.mark.gpu

CASES = sorted(_fixture_cases(np.random.RandomState(0)))
VAD_CASES = [c for c in CASES if 'vad' in c]


def _params(g, case):
    sr, n, lo, default = g[case + '_params']
    kw = {} if default else {'low_freq': lo}
    return int(sr), int(n), kw


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('case', CASES)
def test_fixture_values_match_the_reference(golden, case):
    from pb_bss_b200.evaluation import srmr
    g = golden('srmr')
    sr, n, kw = _params(g, case)
    x, ref = signal(g, case), g[case + '_value']
    v = srmr(x, sr, n, **kw)
    if x.ndim == 1:
        assert isinstance(v, np.float64)
    else:
        assert isinstance(v, np.ndarray) and v.dtype == np.float64 and v.shape == x.shape[:-1]
    # 48 kHz with one band at 300 Hz: the gammatone cascade carries 1 / gain ~ 1e10 in its states, and its rounding
    # alone moves this value by ~1e-10 (the NumPy restatement differs from the reference by 2e-12 there)
    rel = 1e-5 if x.dtype == np.float32 else 5e-10 if case == 'sr48k_n1_low300' else 1e-10
    np.testing.assert_allclose(v, ref, rtol=rel, atol=0)


@pytest.mark.parametrize('case', CASES)
def test_vad_lengths_match(golden, case):
    from pb_bss_b200.evaluation import module_srmr as M
    g = golden('srmr')
    sr, _, _ = _params(g, case)
    x = signal(g, case)
    x = x.astype(np.float64) if x.dtype == np.int16 else x
    rows = x.reshape(-1, x.shape[-1])
    out, nr = M._vad(_cuda(rows), sr, False)
    out, nr = out.cpu().numpy(), nr.cpu().numpy()
    for r, row in enumerate(rows):
        kept = SO.vad(row, sr)
        assert nr[r] == len(kept)
        np.testing.assert_array_equal(out[r, :nr[r]], kept.astype(np.float64))
        assert not out[r, nr[r]:].any()
    if case in VAD_CASES:
        ref = vad_output(g, case)
        assert nr[0] == len(ref) < x.shape[-1]
        np.testing.assert_array_equal(out[0, :nr[0]], ref.astype(np.float64))


def _envelope_check(rows_np, nr=None):
    from pb_bss_b200.evaluation import module_srmr as M
    import torch
    rows, N = rows_np.shape
    nr = np.full(rows, N) if nr is None else np.asarray(nr)
    y = _cuda(rows_np[None].copy())
    M._hilbert_envelopes(y, torch.from_numpy(nr.astype(np.int64)).cuda())
    out = y.cpu().numpy()[0]
    for r in range(rows):
        a = scipy.signal.hilbert(rows_np[r, :nr[r]])
        ref = np.abs(a)
        err = np.max(np.abs(out[r, :nr[r]] - ref))
        assert err <= 1e-12 * np.abs(a).max(), (N, nr[r], err / np.abs(a).max())
    return out


ENVELOPE_LENGTHS = ([1, 2, 3] + [v for k in (5, 10, 11, 12, 13, 17) for v in (2 ** k - 1, 2 ** k, 2 ** k + 1)]
                    + [160001])


@pytest.mark.parametrize('N', ENVELOPE_LENGTHS)
def test_envelopes_match_scipy_hilbert(N):
    _envelope_check(np.random.RandomState(N).randn(2, N))


@pytest.mark.parametrize('N', [4194303, 4194304])
def test_envelopes_at_the_largest_size(N):
    _envelope_check(np.random.RandomState(1).randn(1, N))


def test_envelopes_of_rows_with_different_lengths():
    x = np.random.RandomState(5).randn(3, 5000)
    _envelope_check(x, nr=[5000, 1, 2500])


@pytest.mark.parametrize('sr', [16000, 44100])
@pytest.mark.parametrize('edge', ['W-1', 'W', 'W+1', 'W+S-1', 'W+S'])
def test_means_at_the_frame_count_edges(sr, edge):
    from pb_bss_b200.evaluation import module_srmr as M
    W, S = SO.frame_lengths(sr)
    N = eval(edge, {'W': W, 'S': S})
    x = np.random.RandomState(N).randn(2, N)
    st = M._stages(_cuda(x), sr, 4, 125)
    assert (st['nr'].cpu().numpy() == N).all()
    means = st['means'].cpu().numpy()
    for r in range(2):
        o = SO.srmr_single(x[r], sr, 4, 125)
        scale = np.abs(o['means']).max()
        # 44.1 kHz: the lowest band's gammatone filter (1 / gain ~ 1e10 in its states) is accurate to ~1e-11 of its
        # output, which the squared frame energies double
        tol = 1e-9 if sr == 44100 else 1e-10
        assert np.abs(means[r] - o['means']).max() <= tol * scale
        np.testing.assert_allclose(st['value'].cpu().numpy()[r], o['value'], rtol=1e-10)


def _mixed_batch(sr=16000):
    """Rows of very different N_r: one with two long silences, one without, one mostly silent."""
    rng = np.random.RandomState(11)
    N = 30000
    x = rng.randn(3, N)
    x[0, 3000:9000] = 0
    x[0, 20000:26000] = 0
    x[2, 2000:] = 0
    x[2, 29000] = 1.0
    return x


def test_batch_rows_equal_single_rows_bitwise():
    from pb_bss_b200.evaluation import module_srmr as M
    x = _mixed_batch()
    st = M._stages(_cuda(x), 16000, 23, 125)
    nr = st['nr'].cpu().numpy()
    assert len(set(nr)) == 3
    for r in range(3):
        one = M._stages(_cuda(x[r:r + 1]), 16000, 23, 125)
        assert one['nr'].item() == nr[r]
        np.testing.assert_array_equal(one['means'].cpu().numpy()[0], st['means'].cpu().numpy()[r])
        np.testing.assert_array_equal(one['value'].cpu().numpy()[0], st['value'].cpu().numpy()[r])
        o = SO.srmr_single(x[r], 16000, 23, 125)
        assert o['nr'] == nr[r]
        np.testing.assert_allclose(st['value'].cpu().numpy()[r], o['value'], rtol=1e-10)


def test_workspace_groups_do_not_change_the_result(monkeypatch):
    from pb_bss_b200.evaluation import module_srmr as M
    x = _mixed_batch()
    full = M._stages(_cuda(x), 16000, 23, 125)
    P = 1 << 15                         # M = 2^16 for N = 30000
    monkeypatch.setattr(M, 'HILBERT_WORKSPACE_BYTES', 7 * 16 * P)
    grouped = M._stages(_cuda(x), 16000, 23, 125)
    np.testing.assert_array_equal(grouped['envelopes'].cpu().numpy(), full['envelopes'].cpu().numpy())
    np.testing.assert_array_equal(grouped['value'].cpu().numpy(), full['value'].cpu().numpy())


def test_repeated_calls_are_bitwise_identical():
    from pb_bss_b200.evaluation import srmr
    x = _mixed_batch()
    np.testing.assert_array_equal(srmr(x, 16000), srmr(x, 16000))


def test_non_finite_and_silent_rows_give_nan():
    import torch
    from pb_bss_b200.evaluation import srmr
    x = np.random.RandomState(3).randn(4, 20000)
    x[0, 777] = np.nan
    x[1] = 0
    x[2, 12345] = np.inf
    v = srmr(x, 16000)
    torch.cuda.synchronize()
    assert np.isnan(v[:3]).all() and np.isfinite(v[3])


def test_cuda_tensor_in_gives_cuda_tensor_out_on_the_current_stream():
    import torch
    from pb_bss_b200.evaluation import srmr
    g = np.random.RandomState(4).randn(2, 3, 9000)
    ref = srmr(g, 8000, 4)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        xs = _cuda(g)
        v = srmr(xs, 8000, 4)
        v1 = srmr(xs[1, 2], 8000, 4)
    s.synchronize()
    assert v.is_cuda and v.dtype == torch.float64 and tuple(v.shape) == (2, 3)
    assert v1.is_cuda and v1.dim() == 0
    np.testing.assert_array_equal(v.cpu().numpy(), ref)
    assert v1.item() == ref[1, 2]


def test_float32_and_integer_tensors():
    import torch
    from pb_bss_b200.evaluation import srmr
    x = np.round(np.random.RandomState(6).randn(12000) * 3000).astype(np.int16)
    ref = SO.srmr(x.astype(np.float64), 16000, 4)
    np.testing.assert_allclose(srmr(x, 16000, 4), ref, rtol=1e-10)
    np.testing.assert_allclose(srmr(_cuda(x), 16000, 4).item(), ref, rtol=1e-10)
    f = x.astype(np.float32) / 3000
    np.testing.assert_allclose(srmr(torch.from_numpy(f).cuda(), 16000, 4).item(), SO.srmr(f, 16000, 4), rtol=1e-5)


def test_limits_and_errors(golden):
    from pb_bss_b200.evaluation import srmr
    from pb_bss_b200.evaluation.module_srmr import SRMR
    g = golden('srmr')
    with pytest.raises(ValueError):
        srmr(np.zeros(2 ** 22 + 1), 16000)
    with pytest.raises(ValueError):
        srmr(np.random.randn(4000), 999)
    with pytest.raises(AssertionError):
        srmr(np.zeros((30, 100)), 16000)
    with pytest.raises(NotImplementedError):
        srmr(np.float64(1.0), 16000)
    assert str(g['error_dim30']) == 'AssertionError' and str(g['error_ndim0']) == 'NotImplementedError'
    with pytest.raises(ZeroDivisionError):
        srmr(np.random.randn(4000), 16000, 0)
    x = np.random.RandomState(9).randn(20000)
    assert SRMR(x, 16000, 4) == srmr(x, 16000, 4)
