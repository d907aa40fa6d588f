"""The device backward passes of the get_bf_vector beamformers (GEV, PCA, MVDR, BAN, the rank-1 estimates and the
scaled GEV ATF) against torch.autograd.gradcheck, torch autograd of the phase-fixed restatements in
oracle/bf_autograd_oracle.py and its long-double references."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import bf_autograd_oracle as BO
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200 import _device, _lib
    from pb_bss_b200.evaluation import si_sdr
    from pb_bss_b200.extraction import beamformer as B
    from pb_bss_b200.extraction import beamformer_wrapper as W
    from pb_bss_b200.transform import istft, stft

DEV = 'cuda'


def _t(a, grad=True, dtype=torch.complex128):
    return torch.tensor(a, device=DEV, dtype=dtype, requires_grad=grad)


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _gradcheck(fn, *inputs):
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-7, rtol=1e-5, nondet_tol=0.0)


def _outer(w):
    """w w^H: does not depend on the eigenvector's per-bin phase"""
    return w[..., :, None] * w.conj()[..., None, :]


def _psds(n, D, seed):
    return synth.pos_def_hermitian(n, D, D, seed=seed), synth.pos_def_hermitian(n, D, D, seed=seed + 1) + 0.1 * np.eye(D)


# ---- 1. gradcheck at small shapes ---------------------------------------------------------------------------------

def test_gradcheck_mvdr_ban_rank_one_matvec():
    rng = np.random.default_rng(1)
    _, n = _psds(4, 3, 1)
    a, N = _t(_cplx(rng, 4, 3)), _t(n)
    _gradcheck(B.get_mvdr_vector, a, N)
    _gradcheck(B.blind_analytic_normalization, a, _t(n + 0.2 * _cplx(rng, 4, 3, 3)))
    _gradcheck(W._rank_one, a, _t(_cplx(rng, 4, 3, 3)))
    _gradcheck(W._matvec, _t(_cplx(rng, 4, 3, 3)), a)


def test_gradcheck_gev_pca_through_outer_product():
    t, n = _psds(4, 3, 2)
    T, N = _t(t), _t(n)
    _gradcheck(lambda a, b: _outer(B.get_gev_vector(a, b)), T, N)
    for scaling in (None, 'trace', 'eigenvalue'):
        _gradcheck(lambda a: _outer(B.get_pca_vector(a, scaling=scaling)), T)
    _gradcheck(lambda a: B.get_pca(a)[1], T)
    _gradcheck(lambda a, b: _outer(W.get_bf_vector('gev+ban', a, b)), T, N)
    _gradcheck(lambda a, b: _outer(W.get_bf_vector('pca+mvdr', a, b)), T, N)


# ---- 2. every get_bf_vector string ------------------------------------------------------------------------------

def _restated(name, t, n):
    """the get_bf_vector chain restated with oracle/bf_autograd_oracle.py (a phase-free loss needs no phase alignment)"""
    ban = name.endswith('+ban')
    core = name[:-4] if ban else name
    if core.startswith('rank1_'):
        kind, core = core.split('+', 1)
        if kind == 'rank1_pca':
            a = BO.pca(t)[1]
        else:
            a = BO.matvec(n, BO.gev_vector(t, n)[0])
        t = BO.rank_one_estimate(a, t)
    if core == 'pca':
        w = BO.pca(t)[1]
    elif core == 'gev':
        w = BO.gev_vector(t, n)[0]
    elif core == 'pca+mvdr':
        w = BO.mvdr_vector(BO.pca(t)[1], n)
    elif core == 'scaled_gev_atf+mvdr':
        w = BO.mvdr_vector(BO.matvec(n, BO.gev_vector(t, n)[0]), n)
    else:
        w = AO.mvdr_vector_souden(t, n, 0)[0]
    return BO.blind_analytic_normalization(w, n) if ban else w


NAMES = ['pca', 'gev', 'pca+mvdr', 'scaled_gev_atf+mvdr', 'mvdr_souden', 'rank1_pca+mvdr_souden',
         'rank1_gev+mvdr_souden', 'rank1_pca+gev', 'rank1_gev+gev']


@pytest.mark.parametrize('name', NAMES + [n + '+ban' for n in NAMES])
def test_every_bf_string_through_a_phase_free_loss(name):
    t, n = _psds(40, 4, 4)
    M = _t(synth.pos_def_hermitian(40, 4, 4, seed=9), False)
    kw = {'ref_channel': 0} if 'souden' in name else {}

    def loss(w):
        return ((w.conj()[..., None, :] @ M @ w[..., :, None]).real.sum())

    T, N = _t(t), _t(n)
    got = torch.autograd.grad(loss(W.get_bf_vector(name, T, N, **kw)), (T, N), allow_unused=True)
    Tr, Nr = _t(t), _t(n)
    ref = torch.autograd.grad(loss(_restated(name, Tr, Nr)), (Tr, Nr), allow_unused=True)
    for a, b in zip(got, ref):
        if b is None:
            assert a is None or torch.count_nonzero(a) == 0
            continue
        assert torch.isfinite(a).all()
        err = (a - b).abs().max().item()
        assert err <= 1e-8 * b.abs().max().item(), (name, err, b.abs().max().item())
    if name.startswith('rank1_') and 'souden' in name:  # no phase in these: gradcheck the vector itself
        t3, n3 = _psds(3, 3, 5)
        _gradcheck(lambda a, b: W.get_bf_vector(name, a, b, ref_channel=0), _t(t3), _t(n3))


def test_ch_constant_and_wmwf_raises():
    t, n = _psds(3, 3, 6)
    T = _t(t)
    w = W.get_bf_vector('ch1', T, _t(n))
    assert not w.requires_grad
    with pytest.raises(NotImplementedError):
        W.get_bf_vector('wmwf', T, _t(n))


# ---- 3. device gradients against the long-double references -----------------------------------------------------

DS = [1, 2, 3, 5, 8, 9, 16, 33, 64]


def _ratio_ok(ratio, what):
    ratio = np.asarray(ratio)
    assert np.all(ratio <= 1), (what, float(np.max(ratio)), int(np.argmax(ratio)))


def _c64_bound(bound, ref, dtype):
    """the bound plus the final rounding of a complex64 gradient, normwise per bin"""
    if dtype != torch.complex64:
        return bound
    r = np.abs(np.asarray(ref)).astype(np.float64)
    return bound + 2 * AO.U32 * np.sqrt((r ** 2).reshape(len(bound), -1).sum(-1))


def _inputs(n, D, seed, dtype):
    t, nz = _psds(n, D, seed)
    if dtype == torch.complex64:  # the references read what the device reads: the complex64 values
        t, nz = t.astype(np.complex64).astype(np.complex128), nz.astype(np.complex64).astype(np.complex128)
    return t, nz


@pytest.mark.parametrize('dtype', [torch.complex128, torch.complex64])
@pytest.mark.parametrize('D', DS)
def test_eigenvector_gradients_against_long_double(D, dtype):
    n = 3000 if D == 3 else 200
    rng = np.random.default_rng(10 + D)
    t, nz = _inputs(n, D, 20 + D, dtype)
    T, N = _t(t, dtype=dtype), _t(nz, dtype=dtype)
    w = B.get_gev_vector(T, N)
    g = _cplx(rng, n, D)
    gT, gN = torch.autograd.grad(w, (T, N), torch.tensor(g, device=DEV))
    assert gT.dtype == dtype and gN.dtype == dtype
    rA, rB, bA, bB = BO.eig_grad_ref(t, nz, w.detach().cpu().numpy(), g)
    _ratio_ok(BO.normwise_ratio(gT.cpu().numpy(), rA, _c64_bound(bA, rA, dtype)), 'gev target')
    _ratio_ok(BO.normwise_ratio(gN.cpu().numpy(), rB, _c64_bound(bB, rB, dtype)), 'gev noise')
    T = _t(t, dtype=dtype)
    vec, val = B.get_pca(T)
    gl = rng.standard_normal(n)
    (gT,) = torch.autograd.grad((vec, val), T, (torch.tensor(g, device=DEV), torch.tensor(gl, device=DEV)))
    rA, _, bA, _ = BO.eig_grad_ref(t, None, vec.detach().cpu().numpy(), g, gl)
    _ratio_ok(BO.normwise_ratio(gT.cpu().numpy(), rA, _c64_bound(bA, rA, dtype)), 'pca')


@pytest.mark.parametrize('dtype', [torch.complex128, torch.complex64])
@pytest.mark.parametrize('D', DS)
def test_mvdr_ban_rank_one_matvec_gradients_against_long_double(D, dtype):
    n = 3000 if D == 3 else 200
    rng = np.random.default_rng(30 + D)
    _, nz = _inputs(n, D, 40 + D, dtype)
    a = _cplx(rng, n, D)
    if dtype == torch.complex64:
        a = a.astype(np.complex64).astype(np.complex128)
    g = _cplx(rng, n, D)
    gt = torch.tensor(g, device=DEV)
    A, N = _t(a, dtype=dtype), _t(nz, dtype=dtype)
    ga, gN = torch.autograd.grad(B.get_mvdr_vector(A, N), (A, N), gt)
    ra, rN, ba, bN = BO.mvdr_grad_ref(a, nz, g)
    _ratio_ok(BO.normwise_ratio(ga.cpu().numpy(), ra, _c64_bound(ba, ra, dtype)), 'mvdr atf')
    _ratio_ok(BO.normwise_ratio(gN.cpu().numpy(), rN, _c64_bound(bN, rN, dtype)), 'mvdr noise')
    Nb = nz + 0.3 * _cplx(rng, n, D, D)  # BAN reads N as given: a non-Hermitian one
    if dtype == torch.complex64:
        Nb = Nb.astype(np.complex64).astype(np.complex128)
    A, N = _t(a, dtype=dtype), _t(Nb, dtype=dtype)
    gw, gN = torch.autograd.grad(B.blind_analytic_normalization(A, N), (A, N), gt)
    rw, rN, bw, bN = BO.ban_grad_ref(a, Nb, g)
    _ratio_ok(BO.normwise_ratio(gw.cpu().numpy(), rw, _c64_bound(bw, rw, dtype)), 'ban vector')
    _ratio_ok(BO.normwise_ratio(gN.cpu().numpy(), rN, _c64_bound(bN, rN, dtype)), 'ban noise')
    G = _cplx(rng, n, D, D)
    A, C = _t(a, dtype=dtype), _t(Nb, dtype=dtype)
    ga, gC = torch.autograd.grad(W._rank_one(A, C), (A, C), torch.tensor(G, device=DEV))
    ra, rC, ba, bC = BO.rank_one_grad_ref(a, Nb, G)
    ndt = np.complex64 if dtype == torch.complex64 else np.complex128
    _ratio_ok(AO._ratio(AO._err(ga.cpu().numpy(), ra), AO._rounded(ba, ra, ndt)), 'rank-1 vector')
    _ratio_ok(AO._ratio(AO._err(gC.cpu().numpy(), rC), AO._rounded(bC, rC, ndt)), 'rank-1 covariance')
    M, X = _t(Nb, dtype=dtype), _t(a, dtype=dtype)
    gM, gx = torch.autograd.grad(W._matvec(M, X), (M, X), gt)
    rM, rx, bM, bx = BO.matvec_grad_ref(Nb, a, g)
    _ratio_ok(AO._ratio(AO._err(gM.cpu().numpy(), rM), AO._rounded(bM, rM, ndt)), 'matvec matrix')
    _ratio_ok(AO._ratio(AO._err(gx.cpu().numpy(), rx), AO._rounded(bx, rx, ndt)), 'matvec vector')


# ---- 4. forwards unchanged, backward repeatable -----------------------------------------------------------------

def test_forwards_bitwise_unchanged_and_backward_repeatable():
    t, n = _psds(50, 5, 7)
    for name in ('gev+ban', 'pca+mvdr', 'rank1_gev+mvdr_souden+ban', 'scaled_gev_atf+mvdr', 'pca'):
        kw = {'ref_channel': 1} if 'souden' in name else {}
        ref = W.get_bf_vector(name, t, n, **kw)  # numpy in, numpy out: no graph
        T, N = _t(t), _t(n)
        w = W.get_bf_vector(name, T, N, **kw)
        np.testing.assert_array_equal(w.detach().cpu().numpy(), ref)
        with torch.no_grad():
            np.testing.assert_array_equal(W.get_bf_vector(name, _t(t, False), _t(n, False), **kw).cpu().numpy(), ref)
        g = torch.randn_like(w)
        g1 = torch.autograd.grad(W.get_bf_vector(name, T, N, **kw), (T, N), g, allow_unused=True)
        g2 = torch.autograd.grad(W.get_bf_vector(name, T, N, **kw), (T, N), g, allow_unused=True)
        for a, b in zip(g1, g2):
            assert (a is None and b is None) or torch.equal(a, b)
    vec, val = B.get_pca(t)
    tv, tl = B.get_pca(_t(t))
    np.testing.assert_array_equal(tv.detach().cpu().numpy(), vec)
    np.testing.assert_array_equal(tl.detach().cpu().numpy(), val)


def test_double_backward_raises():
    t, n = _psds(3, 3, 8)
    T = _t(t)
    (g,) = torch.autograd.grad(_outer(B.get_gev_vector(T, _t(n, False))).abs().sum(), T, create_graph=True)
    with pytest.raises(RuntimeError):
        g.abs().sum().backward()


# ---- 5. the NaN policy, bin by bin ------------------------------------------------------------------------------

def _finite_and_equal(got, ref, bad):
    """NaN in the bins of `bad`, and elsewhere equal to the gradient of the call without those bins"""
    keep = [i for i in range(got.shape[0]) if i not in bad]
    assert torch.isnan(got[bad]).all()
    assert torch.isfinite(got[keep]).all()
    err = (got[keep] - ref).abs().max().item()
    assert err <= 1e-12 * ref.abs().max().item(), err


def test_tied_top_eigenvalue_gives_nan_in_its_bin_only():
    rng = np.random.default_rng(11)
    t, n = _psds(5, 3, 11)
    t[2] = np.diag([3.0, 3.0, 1.0])
    n[2] = np.eye(3)
    g = torch.tensor(_cplx(rng, 5, 3), device=DEV)
    T, N = _t(t), _t(n)
    gT, gN = torch.autograd.grad(B.get_gev_vector(T, N), (T, N), g)
    T2, N2 = _t(np.delete(t, 2, 0)), _t(np.delete(n, 2, 0))
    rT, rN = torch.autograd.grad(B.get_gev_vector(T2, N2), (T2, N2), g[[0, 1, 3, 4]])
    _finite_and_equal(gT, rT, [2])
    _finite_and_equal(gN, rN, [2])
    T = _t(t)
    (gT,) = torch.autograd.grad(B.get_pca_vector(T), T, g)
    T2 = _t(np.delete(t, 2, 0))
    (rT,) = torch.autograd.grad(B.get_pca_vector(T2), T2, g[[0, 1, 3, 4]])
    _finite_and_equal(gT, rT, [2])


def test_singular_mvdr_noise_gives_nan_in_its_bin_only():
    rng = np.random.default_rng(12)
    a = _cplx(rng, 5, 3)
    _, n = _psds(5, 3, 12)
    n[1] = np.diag([1.0, 2.0, 0.0])  # an exactly zero pivot: the forward's minimum-norm branch
    A, N = _t(a), _t(n)
    g = torch.tensor(_cplx(rng, 5, 3), device=DEV)
    w = B.get_mvdr_vector(A, N)
    assert torch.isfinite(w).all()
    ga, gN = torch.autograd.grad(w, (A, N), g)
    A2, N2 = _t(np.delete(a, 1, 0)), _t(np.delete(n, 1, 0))
    ra, rN = torch.autograd.grad(B.get_mvdr_vector(A2, N2), (A2, N2), g[[0, 2, 3, 4]])
    _finite_and_equal(ga, ra, [1])
    _finite_and_equal(gN, rN, [1])


def test_singular_mvdr_noise_beyond_the_lstsq_limit_gives_nan_there():
    """D > 40: the forward raises on a singular bin, so the C entry is called directly with the forward's x and w of
    the regular bins (the singular bin's are any finite values)"""
    D, nb = 44, 3
    rng = np.random.default_rng(13)
    a = _cplx(rng, nb, D)
    _, n = _psds(nb, D, 13)
    A, N = _t(a, False), _t(n, False)
    x = torch.linalg.solve((N + N.conj().transpose(-1, -2)) / 2, A[..., None])[..., 0].contiguous()
    w = B.get_mvdr_vector(A, N).contiguous()
    g = torch.tensor(_cplx(rng, nb, D), device=DEV)
    Ns = N.clone()
    Ns[0] = torch.diag(torch.tensor([1.0] * (D - 1) + [0.0], dtype=torch.complex128, device=DEV))
    ga = torch.empty_like(A)
    gN = torch.empty_like(N)
    scratch = torch.empty_like(A)
    lib = _lib.load()
    _lib.check(lib.pbb_mvdr_backward(_device.ptr(A), _device.ptr(Ns), _device.ptr(x), _device.ptr(w), _device.ptr(g),
                                     nb, D, _device.ptr(ga), _device.ptr(gN), _device.ptr(scratch),
                                     _device.stream_ptr()), 'pbb_mvdr_backward')
    A1, N1 = _t(a[1:]), _t(n[1:])
    ra, rN = torch.autograd.grad(B.get_mvdr_vector(A1, N1), (A1, N1), g[1:])
    _finite_and_equal(ga, ra, [0])
    _finite_and_equal(gN, rN, [0])


def test_ban_zero_numerator_nan_zero_denominator_zero():
    rng = np.random.default_rng(14)
    w = _cplx(rng, 5, 2)
    n = synth.pos_def_hermitian(5, 2, 2, seed=14) + 0.3 * _cplx(rng, 5, 2, 2)
    n[1] = [[0.0, 1.0], [0.0, 0.0]]   # nilpotent: w^H N N w = 0, w^H N w = conj(w_0) w_1 != 0  -> NaN
    n[3] = [[0.0, 1.0], [-1.0, 0.0]]  # w = e_0: w^H N w = 0 (the forward's scale is the constant 0) -> zero gradient
    w[3] = [1.0, 0.0]
    V, N = _t(w), _t(n)
    g = torch.tensor(_cplx(rng, 5, 2), device=DEV)
    gv, gN = torch.autograd.grad(B.blind_analytic_normalization(V, N), (V, N), g)
    assert torch.count_nonzero(gv[3]) == 0 and torch.count_nonzero(gN[3]) == 0
    keep = [0, 2, 3, 4]
    V2, N2 = _t(w[keep]), _t(n[keep])
    rv, rN = torch.autograd.grad(B.blind_analytic_normalization(V2, N2), (V2, N2), g[keep])
    _finite_and_equal(gv, rv, [1])
    _finite_and_equal(gN, rN, [1])


def test_rank_one_of_a_zero_vector_gives_nan_in_its_bin_only():
    rng = np.random.default_rng(15)
    a = _cplx(rng, 4, 3)
    a[2] = 0
    c = _cplx(rng, 4, 3, 3)
    A, C = _t(a), _t(c)
    G = torch.tensor(_cplx(rng, 4, 3, 3), device=DEV)
    ga, gC = torch.autograd.grad(W._rank_one(A, C), (A, C), G)
    A2, C2 = _t(a[[0, 1, 3]]), _t(c[[0, 1, 3]])
    ra, rC = torch.autograd.grad(W._rank_one(A2, C2), (A2, C2), G[[0, 1, 3]])
    _finite_and_equal(ga, ra, [2])
    _finite_and_equal(gC, rC, [2])


# ---- 6. the end-to-end gev+ban chain ----------------------------------------------------------------------------

SIZE, SHIFT, D = 512, 128, 6
N_SAMPLES = 999 * SHIFT - 3


def _chain_inputs():
    rng = np.random.default_rng(20)
    y = stft(torch.tensor(rng.standard_normal((D, N_SAMPLES)), device=DEV), size=SIZE, shift=SHIFT)
    y = y.permute(2, 0, 1).contiguous()  # (F, D, T)
    F, _, T = y.shape
    logits = torch.tensor(rng.standard_normal((F, 2, T)), dtype=torch.float32, device=DEV, requires_grad=True)
    target = torch.tensor(rng.standard_normal(N_SAMPLES), device=DEV)
    return y, logits, target


def _chain(y, logits, target, ref_w=None):
    """device chain (ref_w None) -> (loss, the GEV vector); else the torch restatement with its eigenvectors aligned to
    the device's phase (ref_w), so that the phase-dependent SI-SDR loss is the same function"""
    mask = torch.sigmoid(logits)
    if ref_w is None:
        pt = B.get_power_spectral_density_matrix(y, mask[:, 0])
        pn = B.get_power_spectral_density_matrix(y, mask[:, 1])
        w = B.get_gev_vector(pt, pn)
        wb = B.blind_analytic_normalization(w, pn)
        x = istft(B.apply_beamforming_vector(wb, y).transpose(0, 1), size=SIZE, shift=SHIFT)
    else:
        pt = AO.power_spectral_density(y, mask[:, 0])
        pn = AO.power_spectral_density(y, mask[:, 1])
        w = BO.gev_vector(pt, pn, ref_w)[0]
        wb = BO.blind_analytic_normalization(w, pn)
        x = AO.istft(AO.apply_beamforming_vector(wb, y).transpose(0, 1), SIZE, SHIFT)
    return -si_sdr(target, x[:target.shape[-1]].to(torch.float64)) if ref_w is None else \
        -AO.si_sdr(target, x[:target.shape[-1]].to(torch.float64)), w


def test_gev_ban_chain_mask_gradient_matches_the_phase_fixed_restatement():
    y, logits, target = _chain_inputs()
    loss, w = _chain(y, logits, target)
    (g,) = torch.autograd.grad(loss, logits)
    loss_ref, _ = _chain(y, logits, target, w.detach())
    (g_ref,) = torch.autograd.grad(loss_ref, logits)
    assert g.dtype == torch.float32 and torch.isfinite(g).all()
    np.testing.assert_allclose(loss.item(), loss_ref.item(), rtol=1e-8)
    err = (g - g_ref).abs().max().item()
    assert err <= 1e-5 * g_ref.abs().max().item(), (err, g_ref.abs().max().item())


def test_gev_ban_chain_backward_enqueues_only():
    y, logits, target = _chain_inputs()
    loss, _ = _chain(y, logits, target)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(logits.grad).all()
