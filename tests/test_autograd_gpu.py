"""The device backward passes of the mask-based beamforming chain (stft, istft, PSD, Souden MVDR,
apply_beamforming_vector, si_sdr) against torch.autograd.gradcheck and against torch autograd of the pure-torch
restatement in oracle/autograd_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200.evaluation import si_sdr
    from pb_bss_b200.extraction import beamformer as B
    from pb_bss_b200.transform import istft, stft

DEV = 'cuda'


def _t(a, grad=True):
    return torch.tensor(a, device=DEV, requires_grad=grad)


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _gradcheck(fn, *inputs):
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-7, rtol=1e-5, nondet_tol=0.0)


def _bound(got, ref, rel):
    got, ref = got.detach(), ref.detach()
    assert got.dtype == ref.dtype, (got.dtype, ref.dtype)
    err = (got - ref).abs().max().item()
    assert err <= rel * ref.abs().max().item(), (err, ref.abs().max().item())


# ---- gradcheck at small shapes --------------------------------------------------------------------------------------

@pytest.mark.parametrize('wl, fading, pad', [(None, True, True), (None, False, True), (None, True, False),
                                             (48, False, False), (48, True, True)])
def test_gradcheck_stft_istft(wl, fading, pad):
    rng = np.random.default_rng(0)
    x = _t(rng.standard_normal((2, 301)))
    _gradcheck(lambda x: stft(x, size=64, shift=16, window_length=wl, fading=fading, pad=pad), x)
    T = 9
    X = _t(_cplx(rng, 2, T, 33))
    _gradcheck(lambda X: istft(X, size=64, shift=16, window_length=wl, fading=fading), X)


@pytest.mark.parametrize('mask_shape, source_dim, normalize', [
    ((3, 20), -2, True), ((3, 2, 20), -2, True), ((3, 2, 20), -2, False), ((2, 3, 20), 0, True), (None, -2, True)])
def test_gradcheck_psd(mask_shape, source_dim, normalize):
    rng = np.random.default_rng(1)
    y = _t(_cplx(rng, 3, 3, 20))
    if mask_shape is None:
        _gradcheck(lambda y: B.get_power_spectral_density_matrix(y), y)
        return
    m = _t(rng.uniform(0.1, 1.0, mask_shape))
    _gradcheck(lambda y, m: B.get_power_spectral_density_matrix(y, m, source_dim=source_dim, normalize=normalize),
               y, m)


def test_gradcheck_souden():
    t = _t(synth.pos_def_hermitian(4, 3, 3, seed=2))
    n = _t(synth.pos_def_hermitian(4, 3, 3, seed=3))
    _gradcheck(lambda t, n: B.get_mvdr_vector_souden(t, n, ref_channel=1), t, n)


def test_gradcheck_apply_plain_and_shared():
    rng = np.random.default_rng(4)
    v = _t(_cplx(rng, 4, 3))
    y = _t(_cplx(rng, 4, 3, 20))
    _gradcheck(B.apply_beamforming_vector, v, y)
    vs = _t(_cplx(rng, 2, 4, 3))  # two beamformers sharing the one mix: the shared-mix kernel
    _gradcheck(B.apply_beamforming_vector, vs, y)


def test_gradcheck_si_sdr_broadcast():
    rng = np.random.default_rng(5)
    r = _t(rng.standard_normal((1, 50)))
    e = _t(r.detach().cpu().numpy() + 0.5 * rng.standard_normal((3, 50)))
    _gradcheck(si_sdr, r, e)
    _gradcheck(si_sdr, r[0], e)


# ---- parity with torch autograd of the restatement at F = 257, D = 6, T ~ 1000, K = 2 ------------------------------

SIZE, SHIFT, D, K = 512, 128, 6, 2
N_SAMPLES = 999 * SHIFT - 3


def _signal(seed, rows=D):
    return np.random.default_rng(seed).standard_normal((rows, N_SAMPLES))


def _grads(out, inputs, g):
    return torch.autograd.grad(out, inputs, g)


def test_parity_stft_istft():
    x = _t(_signal(10))
    X = stft(x, size=SIZE, shift=SHIFT)
    g = torch.randn_like(X)
    ref = AO.stft(x, SIZE, SHIFT)
    _bound(_grads(X, x, g)[0], _grads(ref, x, g)[0], 1e-10)
    Xs = _t(X.detach().cpu().numpy())
    out = istft(Xs, size=SIZE, shift=SHIFT)
    go = torch.randn_like(out)
    _bound(_grads(out, Xs, go)[0], _grads(AO.istft(Xs, SIZE, SHIFT), Xs, go)[0], 1e-10)


def _stft_obs(seed):
    X = stft(torch.tensor(_signal(seed), device=DEV), size=SIZE, shift=SHIFT)  # (D, T, F)
    return X.permute(2, 0, 1).contiguous()                                    # (F, D, T)


@pytest.mark.parametrize('normalize', [True, False])
def test_parity_psd(normalize):
    y = _stft_obs(11).requires_grad_()
    F, _, T = y.shape
    m = _t(np.random.default_rng(12).uniform(size=(F, K, T)))
    phi = B.get_power_spectral_density_matrix(y, m, normalize=normalize)
    g = torch.randn_like(phi)
    got = _grads(phi, (y, m), g)
    ref = _grads(AO.power_spectral_density(y, m, normalize), (y, m), g)
    for a, b in zip(got, ref):
        _bound(a, b, 1e-10)


def test_parity_souden():
    t = _t(synth.pos_def_hermitian(257, D, D, seed=13))
    n = _t(synth.pos_def_hermitian(257, D, D, seed=14))
    w, ref_channel = B.get_mvdr_vector_souden(t, n, return_ref_channel=True)
    w_ref, r = AO.mvdr_vector_souden(t, n)
    assert r == ref_channel
    g = torch.randn_like(w)
    for a, b in zip(_grads(w, (t, n), g), _grads(w_ref, (t, n), g)):
        _bound(a, b, 1e-8)


def test_parity_apply():
    y = _stft_obs(15).requires_grad_()
    F, _, T = y.shape
    rng = np.random.default_rng(16)
    for v in (_t(_cplx(rng, F, D)), _t(_cplx(rng, K, F, D))):
        out = B.apply_beamforming_vector(v, y)
        g = torch.randn_like(out)
        for a, b in zip(_grads(out, (v, y), g), _grads(AO.apply_beamforming_vector(v, y), (v, y), g)):
            _bound(a, b, 1e-10)


def test_parity_si_sdr():
    rng = np.random.default_rng(17)
    r = _t(rng.standard_normal((1, N_SAMPLES)))
    e = _t(r.detach().cpu().numpy() + 0.3 * rng.standard_normal((K, N_SAMPLES)))
    s = si_sdr(r, e)
    g = torch.randn_like(s)
    for a, b in zip(_grads(s, (r, e), g), _grads(AO.si_sdr(r, e), (r, e), g)):
        _bound(a, b, 1e-10)


# ---- the full chain -------------------------------------------------------------------------------------------------

def _chain(mod, y, logits, target, ref_channel=None):
    mask = torch.sigmoid(logits)
    if mod is None:
        pt = AO.power_spectral_density(y, mask[:, 0])
        pn = AO.power_spectral_density(y, mask[:, 1])
        w, ref = AO.mvdr_vector_souden(pt, pn, ref_channel)
        s = AO.apply_beamforming_vector(w, y)
        x = AO.istft(s.transpose(0, 1), SIZE, SHIFT)
        return -AO.si_sdr(target, x[:target.shape[-1]].to(torch.float64)), ref
    pt = B.get_power_spectral_density_matrix(y, mask[:, 0])
    pn = B.get_power_spectral_density_matrix(y, mask[:, 1])
    w, ref = B.get_mvdr_vector_souden(pt, pn, ref_channel, return_ref_channel=True)
    s = B.apply_beamforming_vector(w, y)
    x = istft(s.transpose(0, 1), size=SIZE, shift=SHIFT)
    return -si_sdr(target, x[:target.shape[-1]].to(torch.float64)), ref


def _chain_inputs():
    y = _stft_obs(20)
    F, _, T = y.shape
    logits = torch.tensor(np.random.default_rng(21).standard_normal((F, 2, T)), dtype=torch.float32, device=DEV,
                          requires_grad=True)
    target = torch.tensor(_signal(22, 1)[0], device=DEV)
    return y, logits, target


def test_full_chain_mask_gradient_matches_torch():
    y, logits, target = _chain_inputs()
    loss, ref = _chain(B, y, logits, target)
    (g,) = torch.autograd.grad(loss, logits)
    loss_ref, _ = _chain(None, y, logits, target, ref)
    (g_ref,) = torch.autograd.grad(loss_ref, logits)
    assert g.dtype == torch.float32
    np.testing.assert_allclose(loss.item(), loss_ref.item(), rtol=1e-9)
    _bound(g, g_ref, 1e-8)


def test_backward_enqueues_only():
    y, logits, target = _chain_inputs()
    loss, _ = _chain(B, y, logits, target)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(logits.grad).all()


def test_backward_is_bitwise_repeatable():
    y, logits, target = _chain_inputs()
    grads = []
    for _ in range(2):
        loss, _ = _chain(B, y, logits, target)
        grads.append(torch.autograd.grad(loss, logits)[0])
    assert torch.equal(grads[0], grads[1])


# ---- invariants ---------------------------------------------------------------------------------------------------

def test_forwards_unchanged_by_requires_grad_and_equal_numpy():
    rng = np.random.default_rng(30)
    x = rng.standard_normal((2, 3000))
    X = stft(x, size=256, shift=64)
    assert torch.equal(stft(_t(x), size=256, shift=64), stft(_t(x, False), size=256, shift=64))
    np.testing.assert_array_equal(stft(_t(x), size=256, shift=64).detach().cpu().numpy(), X)
    np.testing.assert_array_equal(istft(_t(X), size=256, shift=64).detach().cpu().numpy(),
                                  istft(X, size=256, shift=64))
    y = _cplx(rng, 5, 4, 60)
    m = rng.uniform(size=(5, 2, 60))
    psd = B.get_power_spectral_density_matrix(y, m)
    np.testing.assert_array_equal(B.get_power_spectral_density_matrix(_t(y), _t(m)).detach().cpu().numpy(), psd)
    with torch.no_grad():
        np.testing.assert_array_equal(B.get_power_spectral_density_matrix(_t(y), _t(m)).cpu().numpy(), psd)
    w = B.get_mvdr_vector_souden(psd[:, 0], psd[:, 1])
    np.testing.assert_array_equal(B.get_mvdr_vector_souden(_t(psd[:, 0]), _t(psd[:, 1])).detach().cpu().numpy(), w)
    out = B.apply_beamforming_vector(w, y)
    np.testing.assert_array_equal(B.apply_beamforming_vector(_t(w), _t(y)).detach().cpu().numpy(), out)
    r, e = x[0], x[0] + x[1]
    assert si_sdr(_t(r), _t(e)).item() == si_sdr(r, e)


def test_gradient_dtypes_follow_inputs():
    rng = np.random.default_rng(31)
    x = torch.tensor(rng.standard_normal((2, 2000)), dtype=torch.float32, device=DEV, requires_grad=True)
    stft(x, size=128, shift=32).abs().sum().backward()
    assert x.grad.dtype == torch.float32
    y = torch.tensor(_cplx(rng, 5, 4, 60), dtype=torch.complex64, device=DEV, requires_grad=True)
    m = torch.tensor(rng.uniform(size=(5, 2, 60)), dtype=torch.float32, device=DEV, requires_grad=True)
    B.get_power_spectral_density_matrix(y, m).abs().sum().backward()
    assert y.grad.dtype == torch.complex64 and m.grad.dtype == torch.float32
    y.grad = None
    v = _t(_cplx(rng, 5, 4))
    B.apply_beamforming_vector(v, y).abs().sum().backward()
    assert y.grad.dtype == torch.complex64 and v.grad.dtype == torch.complex128


def test_double_backward_raises():
    rng = np.random.default_rng(32)
    y = _t(_cplx(rng, 3, 3, 20))
    (g,) = torch.autograd.grad(B.get_power_spectral_density_matrix(y).abs().sum(), y, create_graph=True)
    with pytest.raises(RuntimeError):
        g.abs().sum().backward()


def test_singular_noise_bin_gives_nan_gradient_there_only():
    t = synth.pos_def_hermitian(6, 3, 3, seed=33)
    n = synth.pos_def_hermitian(6, 3, 3, seed=34)
    n[2] = 0.0
    tt, nn = _t(t), _t(n)
    w = B.get_mvdr_vector_souden(tt, nn, ref_channel=0)
    gt, gn = torch.autograd.grad(w, (tt, nn), torch.ones_like(w))
    for g in (gt, gn):
        assert torch.isnan(g[2]).all()
        assert torch.isfinite(g[[0, 1, 3, 4, 5]]).all()
