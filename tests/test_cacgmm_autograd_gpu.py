"""The device backward passes of the cACGMM (pbb_cacgmm_mstep_backward, pbb_cacgmm_predict_backward) against
torch.autograd.gradcheck and against torch autograd of the float64 restatement (oracle/cacgmm_autograd_oracle.py),
over the forward's shape domain, the options with a graph, and the invariants of the backward."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import cacgmm_autograd_oracle as A
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200.distribution import CACGMM, CACGMMTrainer, ComplexAngularCentralGaussian
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    from pb_bss_b200.evaluation import si_sdr
    from pb_bss_b200.extraction import beamformer as B
    from pb_bss_b200.transform import istft, stft

DEV = 'cuda'


def _t(a, grad=False, dtype=None):
    t = torch.tensor(np.ascontiguousarray(a), device=DEV, dtype=dtype)
    return t.requires_grad_() if grad else t


def _gradcheck(fn, *inputs):
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-6, rtol=1e-5, nondet_tol=0.0)


def _model(m):
    return m.cacg.covariance_eigenvectors, m.cacg.covariance_eigenvalues, m.weight


def _probe_loss(model, y, R):
    """a loss that sees the model through predict and log_likelihood: sum R * affiliation + log-likelihood"""
    return (R * model.predict(y)).sum() + 0.1 * model.log_likelihood(y)


def _probe_loss_ref(model, y, R):
    return (R * A.predict(y, model)).sum() + 0.1 * A.log_likelihood(y, model)


def _per_bin_err(got, ref, lead):
    """max over bins of max|got - ref| / max|ref| in the bin"""
    g = (got.detach() - ref.detach()).abs().reshape(lead, -1).max(-1).values
    s = ref.detach().abs().reshape(lead, -1).max(-1).values.clamp(min=1e-300)
    return (g / s).max().item()


# ---- gradcheck at small shapes --------------------------------------------------------------------------------------

@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
def test_gradcheck_m_step(norm):
    F, T, D, K = 2, 10, 3, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=1)
    init = synth.init_affiliation(F, K, T, seed=2)
    rng = np.random.RandomState(3)
    q, sal = rng.uniform(0.5, 2.0, (F, K, T)), rng.uniform(0.2, 1.0, (F, T))
    probe = _t(synth.structured_stft(F, 6, D, K, seed=4)[0])

    def fn(y_, a_, q_, s_):
        m = cacgmm_m_step(y_, q_, a_, saliency=s_, covariance_norm=norm)
        return m.log_likelihood(probe), m.predict(probe), m.weight
    _gradcheck(fn, _t(y, True), _t(init, True), _t(q, True), _t(sal, True))


def test_gradcheck_predict_log_likelihood_and_fit():
    F, T, D, K = 2, 9, 3, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=5)
    init = synth.init_affiliation(F, K, T, seed=6)
    m = CACGMMTrainer().fit(_t(y), initialization=_t(init), iterations=2)
    V, lam, w = (x.clone().requires_grad_() for x in _model(m))

    def pred(y_, V_, l_, w_):
        mm = CACGMM(weight=w_, cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=V_,
                                                                  covariance_eigenvalues=l_))
        aff, q = mm.predict(y_, return_quadratic_form=True)
        return aff, q, mm.log_likelihood(y_)
    _gradcheck(pred, _t(y, True), V, lam, w)
    _gradcheck(lambda y_, a_: CACGMMTrainer().fit(y_, initialization=a_, iterations=2).log_likelihood(y_),
               _t(y, True), _t(init, True))


# ---- parity with the restatement over the shape domain ---------------------------------------------------------------

CASES = [
    # D, K, T, iterations, options
    (2, 2, 127, 1, {}),
    (3, 3, 128, 2, {'covariance_norm': 'trace'}),
    (8, 3, 129, 5, {'saliency': True}),
    (13, 7, 1000, 2, {'covariance_norm': False}),
    (34, 19, 129, 1, {}),
    (8, 2, 300, 2, {'mask': True}),
    (4, 3, 200, 2, {'weight_constant_axis': -2}),
    (6, 4, 128, 2, {'affiliation_eps': 0.}),
    (8, 3, 250, 2, {'warm': True}),
    (4, 2, 200, 2, {'c64': True}),
    (4, 2, 150, 2, {'lead': True}),
]


def _case_inputs(D, K, T, opts, F=3):
    y, _ = synth.structured_stft(F, T, D, K, seed=D * 100 + K)
    init = synth.init_affiliation(F, K, T, seed=T)
    rng = np.random.RandomState(D + K)
    kw, kw_ref = {}, {}
    for name in ('covariance_norm', 'weight_constant_axis', 'affiliation_eps'):
        if name in opts:
            kw[name] = kw_ref[name] = opts[name]
    sal = mask = None
    if opts.get('saliency'):
        sal = _t(rng.uniform(0.1, 1.0, (F, T)), True)
        kw['saliency'] = kw_ref['saliency'] = sal
    if opts.get('mask'):
        mask = _t(rng.uniform(size=(F, K, T)) > 0.2)
        kw['source_activity_mask'] = kw_ref['source_activity_mask'] = mask
    if opts.get('lead'):  # y (2, F, T, D) with an initialisation broadcast over the first dim
        y = np.stack([y, synth.structured_stft(F, T, D, K, seed=7)[0]])
        init = init[None]
    return y, init, kw, kw_ref, sal


@pytest.mark.parametrize('D,K,T,iterations,opts', CASES)
def test_fit_gradient_matches_restatement(D, K, T, iterations, opts):
    y, init, kw, kw_ref, sal = _case_inputs(D, K, T, opts)
    dtype = torch.complex64 if opts.get('c64') else torch.complex128
    yt = _t(y, dtype=dtype).requires_grad_()
    R = _t(np.random.RandomState(9).standard_normal(y.shape[:-2] + (K, T)))
    inputs = [yt] + ([sal] if sal is not None else [])
    if opts.get('warm'):
        m0 = CACGMMTrainer().fit(_t(y), initialization=_t(init), iterations=2)
        V, lam, w = (x.clone().requires_grad_() for x in _model(m0))
        start = CACGMM(weight=w, cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=V,
                                                                    covariance_eigenvalues=lam))
        start_ref = A.from_eig(V, lam, w)
        inputs += [V, lam, w]
    else:
        start = start_ref = _t(init, True)
        inputs.append(start)
    m = CACGMMTrainer().fit(yt, initialization=start, iterations=iterations, **kw)
    loss = _probe_loss(m, yt, R)
    grads = torch.autograd.grad(loss, inputs)
    m_ref = A.fit(yt, start_ref, iterations, **kw_ref)
    loss_ref = _probe_loss_ref(m_ref, yt, R)
    grads_ref = torch.autograd.grad(loss_ref, inputs)
    rel = 1e-4 if opts.get('c64') else 1e-7
    np.testing.assert_allclose(loss.item(), loss_ref.item(), rtol=rel)
    errs = []
    for g, r in zip(grads, grads_ref):
        assert g.dtype == r.dtype and torch.isfinite(g).all()
        errs.append(_per_bin_err(g, r, g.shape[0] if g.dim() > 2 else 1))
    print(f'\ncacgmm autograd parity D={D} K={K} T={T} it={iterations} {opts}: max per-bin rel diff '
          + ' '.join(f'{e:.2e}' for e in errs))
    assert max(errs) <= rel, errs


def test_m_step_and_predict_gradients_match_restatement():
    D, K, T, F = 8, 3, 129, 4
    y, _ = synth.structured_stft(F, T, D, K, seed=11)
    init = synth.init_affiliation(F, K, T, seed=12)
    q = np.random.RandomState(13).uniform(0.3, 3.0, (F, K, T))
    yt, at, qt = _t(y, True), _t(init, True), _t(q, True)
    R = _t(np.random.RandomState(14).standard_normal((F, K, T)))
    m = cacgmm_m_step(yt, qt, at)
    aff, qq = m.predict(yt, return_quadratic_form=True)
    loss = (R * aff).sum() + (R * qq.log()).sum() + m.log_likelihood(yt)
    g = torch.autograd.grad(loss, (yt, at, qt))
    mr = A.m_step(yt, qt, at)
    affr, qr = A.predict(yt, mr, return_quadratic_form=True)
    lr = (R * affr).sum() + (R * qr.log()).sum() + A.log_likelihood(yt, mr)
    gr = torch.autograd.grad(lr, (yt, at, qt))
    for a, b in zip(g, gr):
        assert _per_bin_err(a, b, F) <= 1e-8


def test_rank_deficient_observation_gives_finite_gradients_equal_to_restatement():
    rng = np.random.RandomState(0)
    F, T, D, K = 6, 96, 8, 2
    basis = rng.randn(F, 2, D) + 1j * rng.randn(F, 2, D)
    coeff = rng.randn(F, T, 2) + 1j * rng.randn(F, T, 2)
    y = np.einsum('ftr,frd->ftd', coeff, basis)
    init = synth.init_affiliation(F, K, T, seed=2)
    yt, at = _t(y, True), _t(init, True)
    R = _t(rng.standard_normal((F, K, T)))
    m = CACGMMTrainer().fit(yt, initialization=at, iterations=4)
    g = torch.autograd.grad(_probe_loss(m, yt, R), (yt, at))
    mr = A.fit(yt, at, 4)
    gr = torch.autograd.grad(_probe_loss_ref(mr, yt, R), (yt, at))
    # B^-1 holds 1 / floor = 1e10 on the floored subspace, which z leaves only by rounding: the gradient's part out of
    # the subspace is that rounding times 1e10 in both implementations, so the bound scales with 1 / floor
    bound = 1e3 * np.finfo(np.float64).eps / 1e-10
    for a, b in zip(g, gr):
        assert torch.isfinite(a).all()
        err = _per_bin_err(a, b, F)
        print(f'\ncacgmm autograd rank-deficient: max per-bin rel diff {err:.2e} (bound {bound:.1e})')
        assert err <= bound


# ---- invariants -----------------------------------------------------------------------------------------------------

def test_forwards_bitwise_unchanged_by_requires_grad():
    F, T, D, K = 5, 300, 6, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=20)
    init = synth.init_affiliation(F, K, T, seed=21)
    q = np.random.RandomState(22).uniform(0.5, 2.0, (F, K, T))
    plain = cacgmm_m_step(_t(y), _t(q), _t(init))
    graph = cacgmm_m_step(_t(y, True), _t(q, True), _t(init, True))
    for a, b in zip(_model(plain), _model(graph)):
        assert torch.equal(a, b.detach())
    V, lam, w = (x.clone().requires_grad_() for x in _model(plain))
    mg = CACGMM(weight=w, cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=V, covariance_eigenvalues=lam))
    for yy in (_t(y), _t(y, True)):
        a0, q0 = plain.predict(_t(y), return_quadratic_form=True)
        a1, q1 = mg.predict(yy, return_quadratic_form=True)
        assert torch.equal(a0, a1.detach()) and torch.equal(q0, q1.detach())
        assert torch.equal(plain.log_likelihood(_t(y)), mg.log_likelihood(yy).detach())


def test_graph_fit_is_the_hand_written_loop_and_close_to_the_plain_fit():
    F, T, D, K, I = 40, 300, 8, 3, 6
    y, _ = synth.structured_stft(F, T, D, K, seed=3)
    init = synth.init_affiliation(F, K, T, seed=5)
    yt = _t(y, True)
    m = CACGMMTrainer().fit(yt, initialization=_t(init), iterations=I)
    ref = cacgmm_m_step(yt, None, _t(init))
    for _ in range(I - 1):
        aff, q = ref._run_predict(yt, None, 1e-10, want_q=True)[:2]
        ref = cacgmm_m_step(yt, q, aff)
    for a, b in zip(_model(m), _model(ref)):
        assert torch.equal(a, b)
    plain = CACGMMTrainer().fit(_t(y), initialization=_t(init), iterations=I)
    np.testing.assert_allclose(m.weight.detach().cpu().numpy(), plain.weight.cpu().numpy(), rtol=1e-8, atol=1e-11)


def test_coupled_options_raise_with_a_graph():
    F, T, D, K = 3, 50, 4, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=8)
    init = synth.init_affiliation(F, K, T, seed=9)
    with pytest.raises(NotImplementedError):
        CACGMMTrainer().fit(_t(y, True), initialization=_t(init), iterations=2, weight_constant_axis=(-3,))
    with pytest.raises(NotImplementedError):
        cacgmm_m_step(_t(y, True), None, _t(init), weight_constant_axis=(-3, -1))
    m = CACGMMTrainer().fit(_t(y), initialization=_t(init), iterations=2, weight_constant_axis=(-3,))
    with pytest.raises(NotImplementedError):
        m.predict(_t(y, True))


def _small_graph(seed=30):
    F, T, D, K = 6, 200, 6, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=seed)
    init = synth.init_affiliation(F, K, T, seed=seed + 1)
    yt, at = _t(y, True), _t(init, True)
    m = CACGMMTrainer().fit(yt, initialization=at, iterations=3)
    return _probe_loss(m, yt, _t(np.random.RandomState(seed).standard_normal((F, K, T)))), (yt, at)


def test_backward_is_bitwise_repeatable_and_enqueues_only():
    loss, inputs = _small_graph()
    g1 = torch.autograd.grad(loss, inputs, retain_graph=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        g2 = torch.autograd.grad(loss, inputs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


def test_double_backward_raises():
    loss, inputs = _small_graph()
    g = torch.autograd.grad(loss, inputs, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(g[0].abs().sum(), inputs)


def test_nan_stays_in_its_bin():
    F, T, D, K = 4, 100, 4, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=40)
    init = synth.init_affiliation(F, K, T, seed=41)
    m = CACGMMTrainer().fit(_t(y), initialization=_t(init), iterations=3)
    R = _t(np.random.RandomState(42).standard_normal((F, K, T)))

    def grads(y_np, lam_fix=None):
        V, lam, w = (x.clone() for x in _model(m))
        if lam_fix is not None:
            lam[lam_fix] = 0.
        V, lam, w = V.requires_grad_(), lam.requires_grad_(), w.requires_grad_()
        mm = CACGMM(weight=w, cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=V, covariance_eigenvalues=lam))
        yt = _t(y_np, True)
        return torch.autograd.grad((R * mm.predict(yt)).sum(), (yt, V, lam, w))

    clean = grads(y)
    bad = y.copy()
    bad[1, 5, 2] = np.nan
    for hit, got in ((1, grads(bad)), (2, grads(y, (2, 0, 0)))):
        others = [f for f in range(F) if f != hit]
        for a, b in zip(got, clean):
            assert torch.equal(a[others], b[others])
        assert not all(torch.isfinite(a[hit]).all() for a in got)


# ---- end to end -----------------------------------------------------------------------------------------------------

SIZE, SHIFT, DC, KC = 256, 64, 4, 2
N_SAMPLES = 160 * SHIFT - 5


def _chain(dev, y, logits, target):
    init = torch.softmax(logits, dim=1)                       # (F, K, T)
    obs = y.transpose(-1, -2)                                 # (F, T, D)
    if dev:
        mask = CACGMMTrainer().fit(obs, initialization=init, iterations=3).predict(obs)
        pt = B.get_power_spectral_density_matrix(y, mask[:, 0])
        pn = B.get_power_spectral_density_matrix(y, mask[:, 1])
        w = B.get_mvdr_vector_souden(pt, pn, ref_channel=0)
        x = istft(B.apply_beamforming_vector(w, y).transpose(0, 1), size=SIZE, shift=SHIFT)
        return -si_sdr(target, x[:target.shape[-1]].to(torch.float64))
    mask = A.predict(obs, A.fit(obs, init, 3))
    pt = AO.power_spectral_density(y, mask[:, 0])
    pn = AO.power_spectral_density(y, mask[:, 1])
    w, _ = AO.mvdr_vector_souden(pt, pn, 0)
    x = AO.istft(AO.apply_beamforming_vector(w, y).transpose(0, 1), SIZE, SHIFT)
    return -AO.si_sdr(target, x[:target.shape[-1]].to(torch.float64))


def test_unrolled_em_chain_to_si_sdr_matches_restatement():
    rng = np.random.default_rng(50)
    s = rng.standard_normal((DC, N_SAMPLES))
    X = stft(_t(s), size=SIZE, shift=SHIFT)                  # (D, T, F)
    y = X.permute(2, 0, 1).contiguous()                       # (F, D, T)
    F, _, T = y.shape
    logits = _t(rng.standard_normal((F, KC, T)), True)
    target = _t(s[0])
    loss = _chain(True, y, logits, target)
    (g,) = torch.autograd.grad(loss, logits)
    loss_ref = _chain(False, y, logits, target)
    (g_ref,) = torch.autograd.grad(loss_ref, logits)
    assert torch.isfinite(g).all()
    np.testing.assert_allclose(loss.item(), loss_ref.item(), rtol=1e-8)
    err = (g - g_ref).abs().max().item()
    print(f'\ncacgmm unrolled EM chain: max |grad - restatement| {err:.2e} of {g_ref.abs().max().item():.2e}')
    assert err <= 1e-6 * g_ref.abs().max().item()


def test_unsupervised_likelihood_loss_decreases():
    F, T, D, K = 16, 200, 6, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=60)
    yt = _t(y)
    torch.manual_seed(0)
    logits = torch.randn(F, K, T, device=DEV, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([logits], lr=0.1)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = -cacgmm_m_step(yt, None, torch.softmax(logits, dim=1)).log_likelihood(yt)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0], losses
