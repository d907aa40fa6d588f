"""GPU checks of BSS Eval (pb_bss_b200.evaluation.mir_eval_sources): the mir_eval numbers the reference publishes,
the structural cases of the reference's test_mir_eval.py, agreement with the NumPy restatement over K = 1..8,
E = K and K + 1 and T from 1 to 2^22, input types, bitwise reproducibility and batching, and every error."""
import numpy as np
import pytest
import scipy.signal

from oracle import bss_eval_oracle as O
from oracle.make_golden_bss_eval import input_signals
from test_bss_eval_oracle import structural_cases

pytestmark = pytest.mark.gpu

L = 512


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def test_input_metrics_anchor(golden):
    from pb_bss_b200.evaluation import mir_eval_sources
    g = golden('bss_eval')
    ref, est = input_signals(g)
    out = mir_eval_sources(ref, est, return_dict=True, compute_permutation=False)
    assert sorted(out) == ['sar', 'sdr', 'sir']
    for name in ('sdr', 'sir', 'sar'):
        assert out[name].shape == (2, 3) and out[name].dtype == np.float64
        np.testing.assert_allclose(out[name], g['input_' + name], rtol=float(g['input_rtol']))


def test_output_metrics_anchor(golden):
    from pb_bss_b200.evaluation import mir_eval_sources
    g = golden('bss_eval')
    sdr, sir, sar, sel = mir_eval_sources(g['output_reference'], g['output_estimation'])
    for name, v in (('sdr', sdr), ('sir', sir), ('sar', sar)):
        np.testing.assert_allclose(v, g['output_' + name], rtol=float(g['output_rtol']))
    np.testing.assert_array_equal(sel, g['output_selection'])
    assert sel.dtype == np.int64


def test_doctest_anchor(golden):
    """kappa(G) is about 5.8e19 here; LU with partial pivoting reproduces the 4 printed decimals."""
    from pb_bss_b200.evaluation import mir_eval_sources
    g = golden('bss_eval')
    sdr, sir, sar, sel = mir_eval_sources(g['doctest_reference'], g['doctest_estimation'])
    for name, v in (('sdr', sdr), ('sir', sir), ('sar', sar)):
        np.testing.assert_array_equal(np.round(v, 4), g['doctest_' + name])
    np.testing.assert_array_equal(sel, g['doctest_selection'])


@pytest.mark.parametrize('case', sorted(structural_cases()))
def test_structural_cases(case):
    from pb_bss_b200.evaluation import mir_eval_sources
    ref, est, selection = structural_cases()[case]
    sdr, sir, sar, sel = mir_eval_sources(ref, est)
    for v in (sdr, sir, sar):
        assert v.shape == ref.shape[:-1] and np.all(v > 100), v
    assert sel.shape == ref.shape[:-1] and sel.dtype == np.int64
    np.testing.assert_array_equal(sel, selection)


def speech_like(rng, K, E, T):
    """K sources of AR(2)-coloured noise under a slow amplitude envelope, and E estimates: estimate e is source e
    through a short random filter (a gain for e = 0), plus the other sources at a level from -130 dB to +5 dB and white noise,
    so that the values span negative to more than 100 dB; an estimate K (E = K + 1) is mostly noise."""
    src = np.empty((K, T))
    for k in range(K):
        a = [1, -1.6 + 0.1 * k / max(K, 1), 0.8]
        env = 0.6 + 0.4 * np.sin(2 * np.pi * np.arange(T) / 4000 * (1 + 0.3 * k) + k)
        src[k] = scipy.signal.lfilter([1], a, rng.standard_normal(T)) * env
    levels = [10 ** (-130 / 20), 1e-5, 1e-3, 0.1, 0.5, 1.8]
    est = np.empty((E, T))
    for e in range(E):
        if e == K:
            est[e] = rng.standard_normal(T) + 0.2 * src.sum(0)
            continue
        h = rng.standard_normal(8) * np.exp(-np.arange(8))
        h[0] = 1.0
        if e == 0:
            h = h[:1]   # the tail of a longer filter is cut at T, which alone keeps SIR below about 70 dB
        own = scipy.signal.lfilter(h, [1], src[e])
        lv = levels[e % len(levels)]
        est[e] = own + lv * (src.sum(0) - src[e]) + 1e-2 * lv * rng.standard_normal(T) * np.std(own)
    return src, est


def _domain():
    out = [(1, T) for T in (1, 511, 512, 513, 4096, 160000)]
    out += [(K, T) for K in range(2, 9) for T in (4096, 160000) if T + L - 1 > K * L]
    out += [(2, 1 << 22)]
    return [(K, E, T) for K, T in out for E in (K, K + 1)]


# above this value a ratio compares a signal with a residual at the rounding level of the projection; both sides
# must then agree that it is that large, not on its value
NOISE_DB = 200.0


def _tolerance(v):
    """1e-7 dB up to 60 dB.  Above, the residual is 10^(-v / 20) of the signal, and the same absolute rounding error
    of the projection (eps kappa(G)) weighs 10^((v - 60) / 20) times more in dB."""
    return 1e-7 * 10 ** (np.maximum(np.abs(v) - 60.0, 0.0) / 20)


def _assert_close_db(dev, ref, what):
    dev, ref = np.asarray(dev), np.asarray(ref)
    assert dev.shape == ref.shape, (what, dev.shape, ref.shape)
    big = (ref > NOISE_DB) | (dev > NOISE_DB)
    np.testing.assert_array_equal(big & ~((ref > NOISE_DB) & (dev > NOISE_DB)), False, err_msg=what)
    d, r = dev[~big], ref[~big]
    np.testing.assert_array_equal(np.isfinite(d), np.isfinite(r), err_msg=what)
    np.testing.assert_array_equal(d[~np.isfinite(r)], r[~np.isfinite(r)], err_msg=what)
    fin = np.isfinite(r)
    err = np.abs(d[fin] - r[fin])
    tol = _tolerance(r[fin])
    assert np.all(err <= tol), (what, float(np.max(err / tol)), r[fin][np.argmax(err / tol)])


@pytest.mark.parametrize('K, E, T', _domain())
def test_every_pair_matches_the_oracle(K, E, T):
    from pb_bss_b200.evaluation import module_mir_eval as M
    rng = np.random.default_rng(1000 * K + 10 * E + T % 997)
    src, est = speech_like(rng, K, E, T)
    x = M._stack(src, est, K, E, T)
    sdr, sir, sar, sel, pairs = M._evaluate(x, K, E, T, True, pairs=True)
    pairs = pairs.cpu().numpy()[0]
    oracle = O.pair_matrices(src, est)
    for name, d, r in zip(('sdr', 'sir', 'sar'), pairs, oracle):
        _assert_close_db(d, r, f'{name} K={K} E={E} T={T}')
    # the public call, with and without the permutation, on the same item
    o_sdr, o_sir, o_sar, o_sel = O.select(*oracle)
    d_sdr, d_sir, d_sar, d_sel = M.mir_eval_sources(src, est)
    np.testing.assert_array_equal(d_sel, o_sel)
    for d, r in ((d_sdr, o_sdr), (d_sir, o_sir), (d_sar, o_sar)):
        _assert_close_db(d, r, 'selected')
    if E == K:
        d = M.mir_eval_sources(src, est, compute_permutation=False)
        for dv, r in zip(d, O.select(*oracle, compute_permutation=False)[:3]):
            _assert_close_db(dv, r, 'diagonal')


def test_values_span_negative_to_above_100_db():
    """The generator of the oracle comparison reaches both ends of the scale."""
    rng = np.random.default_rng(7)
    src, est = speech_like(rng, 3, 4, 20000)
    sdr, sir, sar = O.pair_matrices(src, est)
    assert sdr.min() < 0 and sir.min() < 0 and np.isfinite(sir).all() and sir.max() > 100


@pytest.mark.parametrize('middle', [(3,), (2, 2)])
@pytest.mark.parametrize('compute_permutation', [True, False])
def test_multichannel_shapes_match_the_oracle(middle, compute_permutation):
    from pb_bss_b200.evaluation import mir_eval_sources
    rng = np.random.default_rng(len(middle))
    K, T = 2, 3000
    E = K + 1 if compute_permutation else K
    ref = np.empty((K, *middle, T))
    est = np.empty((E, *middle, T))
    for m in np.ndindex(*middle):
        ref[(slice(None), *m)], est[(slice(None), *m)] = speech_like(rng, K, E, T)
    dev = mir_eval_sources(ref, est, compute_permutation=compute_permutation, return_dict=True)
    orc = O.mir_eval_sources(ref, est, compute_permutation=compute_permutation, return_dict=True)
    assert sorted(dev) == sorted(orc)
    for name in ('sdr', 'sir', 'sar'):
        assert dev[name].shape == (K, *middle)
        _assert_close_db(dev[name], orc[name], name)
    if compute_permutation:
        assert dev['selection'].dtype == np.int64
        np.testing.assert_array_equal(dev['selection'], orc['selection'])


def test_float32_and_integer_input_are_computed_in_fp64():
    from pb_bss_b200.evaluation import mir_eval_sources
    rng = np.random.default_rng(3)
    src, est = speech_like(rng, 2, 2, 6000)
    for dtype in (np.float32, np.int16):
        r = (src / np.abs(src).max() * 20000).astype(dtype)
        e = (est / np.abs(est).max() * 20000).astype(dtype)
        dev = mir_eval_sources(r, e)
        orc = O.mir_eval_sources(r.astype(np.float64), e.astype(np.float64))
        for d, o in zip(dev[:3], orc[:3]):
            assert d.dtype == np.float64
            _assert_close_db(d, o, str(dtype))
        np.testing.assert_array_equal(dev[3], orc[3])
        dev_t = mir_eval_sources(_cuda(r), _cuda(e))
        for d, o in zip(dev_t, dev):
            np.testing.assert_array_equal(d.cpu().numpy(), o)


def test_cuda_tensors_in_give_cuda_tensors_out_without_synchronising():
    import torch
    import pb_bss_b200
    from pb_bss_b200.evaluation import mir_eval_sources
    rng = np.random.default_rng(4)
    src, est = speech_like(rng, 2, 3, 5000)
    want = mir_eval_sources(src, est)
    r, e = _cuda(src), _cuda(est)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode('error')
    try:
        with pb_bss_b200.deferred_status():
            got = mir_eval_sources(r, e)
            torch.cuda.set_sync_debug_mode(prev)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert [v.device.type for v in got] == ['cuda'] * 4
    assert [v.dtype for v in got] == [torch.float64] * 3 + [torch.int64]
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g.cpu().numpy(), w)


def test_repeated_calls_are_bitwise_identical():
    from pb_bss_b200.evaluation import mir_eval_sources
    rng = np.random.default_rng(5)
    src, est = speech_like(rng, 3, 4, 30000)
    a = mir_eval_sources(src, est)
    b = mir_eval_sources(src, est)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_an_item_alone_equals_the_item_in_a_grouped_batch(monkeypatch):
    """Items of a (K, D, T) batch against the same items evaluated one by one, with a workspace cap that forces
    groups of one and of two items."""
    from pb_bss_b200.evaluation import module_mir_eval as M
    rng = np.random.default_rng(6)
    K, D, T = 2, 5, 9000
    ref = np.empty((K, D, T))
    est = np.empty((K + 1, D, T))
    for d in range(D):
        ref[:, d], est[:, d] = speech_like(rng, K, K + 1, T)
    alone = [M.mir_eval_sources(ref[:, d], est[:, d]) for d in range(D)]
    per_item = M._lib.load().pbb_bss_eval_workspace_bytes(1, K, K + 1, T)
    for cap in (per_item, 2 * per_item + 1, M.WORKSPACE_BYTES):
        monkeypatch.setattr(M, 'WORKSPACE_BYTES', cap)
        batch = M.mir_eval_sources(ref, est)
        for d in range(D):
            for x, y in zip(batch, alone[d]):
                np.testing.assert_array_equal(x[:, d], y)


def test_errors():
    import torch
    import pb_bss_b200
    from pb_bss_b200.evaluation import mir_eval_sources
    rng = np.random.default_rng(8)
    src, est = speech_like(rng, 2, 3, 2000)
    zero_ref = src.copy()
    zero_ref[1] = 0
    for e in (est[:2], est):                   # E = K and the K + 1 path
        with pytest.raises(ValueError, match='batch item 0: an all-zero'):
            mir_eval_sources(zero_ref, e)
    zero_est = est.copy()
    zero_est[2] = 0
    with pytest.raises(ValueError, match='all-zero'):
        mir_eval_sources(src, zero_est)
    ref3 = np.stack([src] * 3, axis=1)
    est3 = np.stack([est] * 3, axis=1)
    est3[0, 2, 17] = np.nan
    with pytest.raises(ValueError, match='batch item 2: a non-finite sample'):
        mir_eval_sources(ref3, est3)
    est3[0, 2, 17] = np.inf
    with pytest.raises(ValueError, match='batch item 2: a non-finite'):
        with pb_bss_b200.deferred_status():
            mir_eval_sources(_cuda(ref3), _cuda(est3))
    # T = 1, two equal references: every 2 x 2 block of G is [[1, 1], [1, 1]], an exactly zero pivot
    with pytest.raises(ValueError, match='zero LU pivot'):
        mir_eval_sources(np.ones((2, 1)), np.ones((2, 1)))
    with pytest.raises(ValueError):
        mir_eval_sources(np.ones((9, 100)), np.ones((9, 100)))
    with pytest.raises(TypeError):
        mir_eval_sources(_cuda(src).to(torch.complex128), _cuda(est))
    with pytest.raises(NotImplementedError):
        mir_eval_sources(src, est, compute_permutation=False)
    with pytest.raises(AssertionError):
        mir_eval_sources(ref3, est3[:, :2])
    with pytest.raises(ValueError):
        mir_eval_sources(src[0], est[0])
