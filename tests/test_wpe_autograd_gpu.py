"""The device backward passes of WPE (wpe_step, wpe, get_power, get_power_inverse) against torch.autograd.gradcheck,
the long-double closed forms of oracle/wpe_autograd_oracle.py within its per-bin bounds, and torch autograd of its
restatement through the DNN-WPE front end."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import wpe_autograd_oracle as WA

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200 import wpe as W
    from pb_bss_b200.evaluation import si_sdr
    from pb_bss_b200.extraction import beamformer as B
    from pb_bss_b200.transform import istft, stft

DEV = 'cuda'


def _t(a, grad=True, dtype=None):
    return torch.tensor(a, device=DEV, dtype=dtype, requires_grad=grad)


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _gradcheck(fn, *inputs):
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-7, rtol=1e-5, nondet_tol=0.0)


# ---- 1. gradcheck at small shapes ---------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_gradcheck_wpe_step(mode):
    rng = np.random.default_rng(0)
    Y, w = _t(_cplx(rng, 2, 2, 24)), _t(rng.uniform(0.5, 2.0, (2, 24)))
    _gradcheck(lambda y, w: W.wpe_step(y, w, taps=2, delay=1, statistics_mode=mode), Y, w)


@pytest.mark.parametrize('iterations', [1, 2, 3])
@pytest.mark.parametrize('psd_context', [0, 1, np.inf])
@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_gradcheck_wpe(iterations, psd_context, mode):
    rng = np.random.default_rng(1)
    Y = _t(_cplx(rng, 2, 2, 20))
    _gradcheck(lambda y: W.wpe(y, taps=2, delay=1, iterations=iterations, psd_context=psd_context,
                               statistics_mode=mode), Y)


@pytest.mark.parametrize('psd_context', [0, 2, np.inf])
def test_gradcheck_get_power(psd_context):
    rng = np.random.default_rng(2)
    Y = _t(_cplx(rng, 3, 2, 15))
    _gradcheck(lambda y: W.get_power(y, psd_context), Y)
    _gradcheck(lambda y: W.get_power_inverse(y, psd_context), Y)


# ---- 2. against the long-double closed forms over the shape domain ------------------------------------------------

SHAPES = [(1, 1), (1, 96), (2, 10), (6, 10), (8, 12), (12, 8), (30, 3)]
FRAMES = [1, 63, 64, 65, 128, 129, 1024, 1025, 3000]


def _frames(D, taps):
    """T across the chunk and part edges at which R is well conditioned (at least 3 n frames) -- and every T for
    n = 1"""
    n = D * taps
    ts = [T for T in FRAMES if T >= 3 * n]
    return ts if n == 1 else ts[:2] + ts[-1:]


def _check_bins(got, ref, kappas, n, T, roundings, what, terms):
    for b in range(ref.shape[0]):
        bound = WA.grad_bound(ref[b], kappas[b], n, T, roundings, terms[b])
        err = float(np.max(np.abs(got[b] - ref[b].astype(np.clongdouble))))
        assert err <= bound, (what, b, err, bound)


@pytest.mark.parametrize('D,taps', SHAPES)
@pytest.mark.parametrize('dtype', [torch.complex64, torch.complex128])
def test_wpe_step_gradients_match_long_double(D, taps, dtype):
    rng = np.random.default_rng(10 + D + taps)
    single = dtype == torch.complex64
    for T in _frames(D, taps):
        for delay, mode in ((0, 'full'), (1, 'valid'), (3, 'full')):
            if mode == 'full' and T <= delay:
                continue   # Yt is zero: R is singular, the NaN case below
            bins = 2
            Y = _cplx(rng, bins, D, T)
            xbar = _cplx(rng, bins, D, T)
            if single:
                Y, xbar = Y.astype(np.complex64), xbar.astype(np.complex64)
            w = rng.uniform(0.5, 2.0, (bins, T))
            Yt, wt = _t(Y, dtype=dtype), _t(w)
            X = W.wpe_step(Yt, wt, taps=taps, delay=delay, statistics_mode=mode)
            gy, gw = torch.autograd.grad(X, (Yt, wt), _t(xbar, False, dtype=X.dtype))
            assert gy.dtype == dtype and gw.dtype == torch.float64
            gy, gw = gy.cpu().numpy(), gw.cpu().numpy()
            refs, kap = [], []
            for b in range(bins):
                yl, wl = Y[b].astype(np.clongdouble), w[b].astype(np.longdouble)
                _, G, R = WA.step_forward(yl, wl, taps, delay, mode)
                refs.append(WA.step_backward(yl, wl, G, R, xbar[b].astype(np.clongdouble), taps, delay, mode))
                kap.append([WA.kappa(R)])
            ty = np.abs(xbar).max(axis=(1, 2))
            _check_bins(gy, np.stack([r[0] for r in refs]), kap, D * taps, T, int(single), ('Y', T, delay), ty)
            _check_bins(gw, np.stack([r[1] for r in refs]), kap, D * taps, T, 0, ('w', T, delay),
                        ty / w.min(axis=1))


@pytest.mark.parametrize('D,taps', SHAPES)
@pytest.mark.parametrize('psd_context', [0, 2, np.inf])
def test_wpe_gradients_match_long_double(D, taps, psd_context):
    rng = np.random.default_rng(20 + D + taps)
    for T in _frames(D, taps)[-2:]:
        for delay, iterations in ((0, 1), (1, 2), (3, 3)):
            Y = _cplx(rng, 2, D, T)
            xbar = _cplx(rng, 2, D, T)
            Yt = _t(Y)
            X = W.wpe(Yt, taps=taps, delay=delay, iterations=iterations, psd_context=psd_context)
            gy = torch.autograd.grad(X, Yt, _t(xbar, False))[0].cpu().numpy()
            refs, kap = [], []
            for b in range(2):
                yl = Y[b].astype(np.clongdouble)
                _, stages = WA.wpe_forward(yl, taps, delay, iterations, psd_context, 'full')
                refs.append(WA.wpe_backward(yl, stages, xbar[b].astype(np.clongdouble), taps, delay, psd_context,
                                            'full'))
                kap.append([WA.kappa(st[2]) for st in stages])
            _check_bins(gy, np.stack(refs), kap, D * taps, T, 0, (T, delay, iterations),
                        np.abs(xbar).max(axis=(1, 2)))


def test_leading_dims_views_and_groups(monkeypatch):
    """(2, 3) leading dims of a transposed view, complex64, and bins spread over several workspace groups"""
    rng = np.random.default_rng(30)
    base = _cplx(rng, 3, 2, 4, 200).astype(np.complex64)
    xbar = _cplx(rng, 2, 3, 4, 200).astype(np.complex64)
    w = rng.uniform(0.5, 2.0, (3, 2, 200)).astype(np.float32)

    def run():
        Yb = _t(base)
        Y = Yb.transpose(0, 1)                             # (2, 3, 4, 200), not dense over the leading dims
        wt = _t(w)
        wv = wt.transpose(0, 1)
        X = W.wpe_step(Y, wv, taps=3, delay=2)
        Z = W.wpe(Y, taps=3, delay=2, iterations=2, psd_context=1)
        g = torch.autograd.grad((X, Z), (Yb, wt), (_t(xbar, False, torch.complex64),) * 2)
        return [t.cpu().numpy() for t in g]

    one = run()
    lib = W._lib.load()
    per_bin = min(lib.pbb_wpe_workspace_bytes(1, 4, 200, 3, 2, 0),
                  lib.pbb_wpe_backward_workspace_bytes(1, 4, 200, 3, 2, 0))
    monkeypatch.setattr(W, 'WORKSPACE_BYTES', 2 * per_bin + 1)     # groups of at most two bins, forward and backward
    grouped = run()
    for a, b in zip(one, grouped):
        np.testing.assert_array_equal(a, b)
    assert one[0].dtype == np.complex64 and one[1].dtype == np.float32
    # against the long-double closed forms
    Yn = base.transpose(1, 0, 2, 3)
    for i in range(2):
        for j in range(3):
            yl = Yn[i, j].astype(np.clongdouble)
            wl = w[j, i].astype(np.longdouble)
            _, G, R = WA.step_forward(yl, wl, 3, 2)
            gy, gw = WA.step_backward(yl, wl, G, R, xbar[i, j].astype(np.clongdouble), 3, 2)
            _, st = WA.wpe_forward(yl, 3, 2, 2, 1, 'full')
            gy = gy + WA.wpe_backward(yl, st, xbar[i, j].astype(np.clongdouble), 3, 2, 1, 'full')
            k = [WA.kappa(R)] + [WA.kappa(s[2]) for s in st]
            t = np.abs(xbar[i, j]).max()
            # Y's gradient: two complex64 gradients and their complex64 sum
            _check_bins(one[0][j, i][None], gy[None], [k], 12, 200, 3, 'Y', [t])
            _check_bins(one[1][j, i][None], gw[None], [k[:1]], 12, 200, 1, 'w', [t / w[j, i].min()])


# ---- 3. invariants -------------------------------------------------------------------------------------------------

def test_forwards_bitwise_unchanged_by_requires_grad():
    rng = np.random.default_rng(40)
    for dtype in (np.complex64, np.complex128):
        Y = _cplx(rng, 5, 3, 300).astype(dtype)
        w = rng.uniform(0.5, 2.0, (5, 300))
        for kw in ({}, {'iterations': 2, 'psd_context': np.inf, 'statistics_mode': 'valid'}, {'iterations': 0}):
            ref = W.wpe(Y, taps=4, delay=2, **kw)
            np.testing.assert_array_equal(W.wpe(_t(Y), taps=4, delay=2, **kw).detach().cpu().numpy(), ref)
            np.testing.assert_array_equal(W.wpe(_t(Y, False), taps=4, delay=2, **kw).cpu().numpy(), ref)
        step = W.wpe_step(Y, w, taps=4, delay=2)
        np.testing.assert_array_equal(W.wpe_step(_t(Y), _t(w), taps=4, delay=2).detach().cpu().numpy(), step)
        for fn in (W.get_power, W.get_power_inverse):
            np.testing.assert_array_equal(fn(_t(Y), 2).detach().cpu().numpy(), fn(Y, 2))


def test_backward_repeatable_and_double_backward_raises():
    rng = np.random.default_rng(41)
    Y, w = _t(_cplx(rng, 4, 3, 500)), _t(rng.uniform(0.5, 2.0, (4, 500)))
    g = _t(_cplx(rng, 4, 3, 500), False)

    def grads():
        X = W.wpe(Y, taps=5, delay=3, iterations=3, psd_context=2) + W.wpe_step(Y, w, taps=5, delay=3)
        P = W.get_power(Y, 1).sum() + W.get_power_inverse(Y, np.inf).sum()
        return torch.autograd.grad((X, P), (Y, w), (g, torch.ones((), device=DEV, dtype=torch.float64)))

    a, b = grads(), grads()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    X = W.wpe(Y, taps=5, delay=3, iterations=2)
    (gy,) = torch.autograd.grad(X, Y, g, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gy.abs().sum(), Y)


def test_inplace_with_grad_raises_and_online_has_no_graph():
    rng = np.random.default_rng(42)
    Y = _t(_cplx(rng, 3, 2, 50))
    with pytest.raises(RuntimeError):
        W.wpe(Y, taps=2, delay=1, inplace=True)
    assert not W.get_power_online(Y).requires_grad
    assert not W.online_wpe(Y.transpose(-1, -2).permute(1, 0, 2), 2, 1, 0.99)[0].requires_grad
    with pytest.raises(ValueError):
        W.wpe_step(Y, _t(np.ones((3, 49))), taps=2, delay=1)
    with pytest.raises(ValueError):
        W.wpe_step(Y, _t(np.ones((3, 50)), dtype=torch.complex128), taps=2, delay=1)


# ---- 4. NaN policy per bin -----------------------------------------------------------------------------------------

@pytest.mark.parametrize('case', ['dead_channel', 'zero_bin', 'nan_sample'])
@pytest.mark.parametrize('fn', ['wpe_step', 'wpe'])
def test_nan_policy_per_bin(case, fn):
    rng = np.random.default_rng(50)
    Y = _cplx(rng, 4, 3, 200)
    w = rng.uniform(0.5, 2.0, (4, 200))
    xbar = _cplx(rng, 4, 3, 200)
    bad = Y.copy()
    if case == 'dead_channel':
        bad[2, 1] = 0
    elif case == 'zero_bin':
        bad[2] = 0
    else:
        bad[2, 0, 77] = np.nan

    def grads(Yn, keep):
        Yt, wt = _t(Yn[keep]), _t(w[keep])
        if fn == 'wpe_step':
            X = W.wpe_step(Yt, wt, taps=4, delay=2)
        else:
            X = W.wpe(Yt, taps=4, delay=2, iterations=2)
        return [g.cpu().numpy() if g is not None else None
                for g in torch.autograd.grad(X, (Yt, wt), _t(xbar[keep], False), allow_unused=True)]

    full = grads(bad, slice(None))
    others = [0, 1, 3]
    clean = grads(bad, others)
    assert np.isnan(full[0][2]).all()
    np.testing.assert_array_equal(full[0][others], clean[0])
    if fn == 'wpe_step':
        assert np.isnan(full[1][2]).all()
        np.testing.assert_array_equal(full[1][others], clean[1])


# ---- 5. the DNN-WPE front end end to end ---------------------------------------------------------------------------

SIZE, SHIFT, D = 512, 128, 6
N_SAMPLES = 999 * SHIFT - 3
TAPS, DELAY, EPS = 10, 3, 1e-10


def _front_end(mod, y, logits, target, iterations):
    """sigmoid(logits[:, 0]) mean_d |Y|^2 as the power, WPE, Souden MVDR from the masks sigmoid(logits[:, 1:]),
    apply, iSTFT, -SI-SDR; mod None: the torch restatement"""
    power = torch.sigmoid(logits[:, 0]).to(torch.float64) * (y.abs() ** 2).mean(-2)
    inv = 1 / torch.clamp(power, min=EPS)
    mask = torch.sigmoid(logits[:, 1:]).to(torch.float64)
    if mod is None:
        if iterations:
            x = WA.wpe(y, TAPS, DELAY, iterations)
        else:
            x = WA.wpe_step(y, inv, TAPS, DELAY)[0]
        pt = AO.power_spectral_density(x, mask[:, 0])
        pn = AO.power_spectral_density(x, mask[:, 1])
        w, _ = AO.mvdr_vector_souden(pt, pn, 0)
        s = AO.apply_beamforming_vector(w, x)
        out = AO.istft(s.transpose(0, 1), SIZE, SHIFT)
        return -AO.si_sdr(target, out[:target.shape[-1]].to(torch.float64))
    x = W.wpe(y, TAPS, DELAY, iterations) if iterations else W.wpe_step(y, inv, TAPS, DELAY)
    pt = B.get_power_spectral_density_matrix(x, mask[:, 0])
    pn = B.get_power_spectral_density_matrix(x, mask[:, 1])
    w = B.get_mvdr_vector_souden(pt, pn, 0)
    s = B.apply_beamforming_vector(w, x)
    out = istft(s.transpose(0, 1), size=SIZE, shift=SHIFT)
    return -si_sdr(target, out[:target.shape[-1]].to(torch.float64))


def _front_end_inputs(grad_y):
    x = np.random.default_rng(60).standard_normal((D, N_SAMPLES))
    y = stft(torch.tensor(x, device=DEV), size=SIZE, shift=SHIFT).permute(2, 0, 1).contiguous()   # (F, D, T)
    y.requires_grad_(grad_y)
    F, _, T = y.shape
    logits = torch.tensor(np.random.default_rng(61).standard_normal((F, 3, T)), dtype=torch.float32, device=DEV,
                          requires_grad=True)
    target = torch.tensor(np.random.default_rng(62).standard_normal(N_SAMPLES), device=DEV)
    return y, logits, target


@pytest.mark.parametrize('iterations', [0, 2])   # 0: wpe_step with the network's power; 2: wpe itself
def test_dnn_wpe_front_end_matches_torch(iterations):
    y, logits, target = _front_end_inputs(iterations > 0)
    inputs = (logits, y) if iterations else (logits,)
    loss = _front_end(W, y, logits, target, iterations)
    got = torch.autograd.grad(loss, inputs)
    ref_loss = _front_end(None, y, logits, target, iterations)
    ref = torch.autograd.grad(ref_loss, inputs)
    np.testing.assert_allclose(loss.item(), ref_loss.item(), rtol=1e-9)
    for g, r in zip(got, ref):
        assert g.dtype == r.dtype
        err = (g - r).abs().max().item()
        assert err <= 1e-6 * r.abs().max().item(), (err, r.abs().max().item())


@pytest.mark.parametrize('iterations', [0, 2])
def test_dnn_wpe_backward_enqueues_only(iterations):
    y, logits, target = _front_end_inputs(iterations > 0)
    loss = _front_end(W, y, logits, target, iterations)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(logits.grad).all()
    if iterations:
        assert torch.isfinite(y.grad).all()
