"""The float64 torch restatement of the cACGMM (oracle/cacgmm_autograd_oracle.py): its values against the NumPy
oracle, gradcheck of its graph, and the Loewner backward of its spectral model against central differences at a
floored bin.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import cacgmm_autograd_oracle as A
from oracle import pb_bss_oracle as O
from oracle import synth


def _binv(model):
    V, lam = model['eigenvectors'], model['eigenvalues']
    return np.einsum('...dx,...x,...ex->...de', V, 1 / lam, V.conj())


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def _doctest_data():
    """complex_angular_central_gaussian.py's _fit doctest: frames e1, e1, e2, e2 of D = 3 (a rank-2 scatter, one
    floored eigenvalue), with affiliations that keep the two unfloored eigenvalues apart"""
    y = np.array([[1, 0, 0], [1, 0, 0], [0, 1, 0], [0, 1, 0]], dtype=np.complex128)[None]
    aff = np.array([[0.9, 0.8, 0.3, 0.4], [0.1, 0.2, 0.7, 0.6]])[None]
    return y, aff


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('with_saliency', [False, True])
def test_values_match_numpy_oracle(norm, with_saliency):
    F, T, D, K = 3, 60, 4, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=4)
    init = synth.init_affiliation(F, K, T, seed=5)
    sal = np.random.RandomState(1).uniform(0.2, 1.0, (F, T)) if with_saliency else None
    q = np.random.RandomState(2).uniform(0.5, 2.0, (F, K, T))
    z = O.normalize_observation_cacg(y)
    ref = O.cacgmm_m_step(z, q, init, sal, covariance_norm=norm)
    got = A.m_step(_t(y), _t(q), _t(init), None if sal is None else _t(sal), covariance_norm=norm)
    np.testing.assert_allclose(got['weight'].numpy(), ref['weight'], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(got['eigenvalues'].numpy(), ref['eigenvalues'], rtol=1e-12, atol=1e-15)
    scale = np.abs(_binv(ref)).max()
    np.testing.assert_allclose(got['binv'].detach().numpy(), _binv(ref), rtol=0, atol=1e-12 * scale)
    gamma, qq, _ = A.e_step(_t(y), got, affiliation_eps=1e-10)
    rg, rq, _ = O.cacgmm_e_step(z, ref, affiliation_eps=1e-10)
    np.testing.assert_allclose(gamma.detach().numpy(), rg, rtol=0, atol=1e-12)
    np.testing.assert_allclose(qq.detach().numpy(), rq, rtol=1e-12)
    ll = A.log_likelihood(_t(y), got).item()
    np.testing.assert_allclose(ll, O.cacgmm_log_likelihood(y, ref), rtol=1e-12)


def test_fit_matches_numpy_oracle():
    F, T, D, K = 2, 80, 3, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=6)
    init = synth.init_affiliation(F, K, T, seed=7)
    mask = np.random.RandomState(3).uniform(size=(F, K, T)) > 0.1
    ref = O.cacgmm_fit(y, init, 4, source_activity_mask=mask)
    got = A.fit(_t(y), _t(init), 4, source_activity_mask=_t(mask))
    np.testing.assert_allclose(got['weight'].numpy(), ref['weight'], rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(got['eigenvalues'].numpy(), ref['eigenvalues'], rtol=1e-10, atol=1e-15)


def _gradcheck(fn, *args):
    assert torch.autograd.gradcheck(fn, args, eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
def test_gradcheck_m_step_through_log_likelihood(norm):
    F, T, D, K = 1, 10, 3, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=8)
    init = synth.init_affiliation(F, K, T, seed=9)
    q = np.random.RandomState(4).uniform(0.5, 2.0, (F, K, T))
    sal = np.random.RandomState(5).uniform(0.2, 1.0, (F, T))
    args = [_t(v).requires_grad_() for v in (y, q, init, sal)]
    _gradcheck(lambda y_, q_, a_, s_: A.log_likelihood(y_, A.m_step(y_, q_, a_, s_, covariance_norm=norm)), *args)


def test_gradcheck_predict_and_fit():
    F, T, D, K = 1, 9, 3, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=10)
    init = synth.init_affiliation(F, K, T, seed=11)
    model = A.m_step(_t(y), None, _t(init))
    V = model['eigenvectors'].clone().requires_grad_()
    lam = model['eigenvalues'].clone().requires_grad_()
    w = model['weight'].clone().requires_grad_()
    yt = _t(y).requires_grad_()
    _gradcheck(lambda y_, V_, l_, w_: A.predict(y_, A.from_eig(V_, l_, w_)), yt, V, lam, w)
    _gradcheck(lambda y_, a_: A.log_likelihood(y_, A.fit(y_, a_, 2)), yt, _t(init).requires_grad_())


def test_gradcheck_floored_rank2_doctest_data():
    y, aff = _doctest_data()
    model = A.m_step(_t(y), None, _t(aff))
    np.testing.assert_allclose(model['eigenvalues'][0, 0, 0].item(), 1e-10)
    probe = _t(np.array([[1, 0.5j, 0.2], [0.3, 1, -0.4j]], dtype=np.complex128)[None])
    _gradcheck(lambda y_, a_: A.log_likelihood(probe, A.m_step(y_, None, a_)),
               _t(y).requires_grad_(), _t(aff).requires_grad_())


def test_loewner_backward_matches_central_differences_at_a_floored_bin():
    rng = np.random.RandomState(12)
    D = 4
    B = rng.randn(D, 2) + 1j * rng.randn(D, 2)
    C = B @ B.conj().T                       # rank 2: two floored eigenvalues
    C = _t(C)
    G = _t(rng.randn(D, D) + 1j * rng.randn(D, D))
    gld = 0.3

    def loss(c):
        c = (c + c.mH) / 2
        top = torch.linalg.eigh(c)[1][..., -1:]
        m = (top.mH @ c @ top).real[..., 0]
        binv, ld = A.SpectralModel.apply(c, m, 1e-3, 'eigenvalue')
        return (G.conj() * binv).real.sum() + gld * ld

    Cg = C.clone().requires_grad_()
    loss(Cg).backward()
    h = 1e-6
    for i, j, part in [(0, 0, 1), (0, 1, 1), (0, 1, 1j), (2, 3, 1j), (3, 3, 1)]:
        E = torch.zeros(D, D, dtype=torch.complex128)
        E[i, j] = part
        E[j, i] += np.conj(part) if i != j else 0
        num = (loss(C + h * E) - loss(C - h * E)).item() / (2 * h)
        ana = (Cg.grad.conj() * E).real.sum().item()
        assert abs(num - ana) <= 1e-5 * max(1.0, abs(num)), (i, j, part, num, ana)


# ---- the restatement's gradients against mpmath directional derivatives ----------------------------------------------
U = np.finfo(np.float64).eps


def _dirs(rng, inputs):
    return {k: (rng.standard_normal(v.shape) + 1j * rng.standard_normal(v.shape)) if np.iscomplexobj(v)
            else rng.standard_normal(v.shape) for k, v in inputs.items()}


def _check_mp(grads, inputs, rng, bound, n_dirs=2, **kw):
    """Re <grad, dir> against mpmath's directional derivative along random directions: |err| <= bound * sum |grad|
    |dir| (the derivative's own scale); returns the worst err / bound"""
    worst = 0.0
    for _ in range(n_dirs):
        dirs = _dirs(rng, inputs)
        ref = A.mp_directional(inputs, dirs, **kw)
        got = A.directional(grads, dirs)
        scale = sum(float(np.sum(np.abs(grads[k]) * np.abs(dirs[k]))) for k in dirs)
        ratio = abs(got - ref) / (bound * scale)
        assert ratio <= 1, (got, ref, scale)
        worst = max(worst, ratio)
    return worst


def _m_step_grads(y, init, q, sal, R, probe=None, mask=None, iterations=1, **kw):
    """gradients of sum R * predict(probe) + 0.1 log_likelihood(probe) through the restatement's m_step / fit"""
    inputs = dict(y=y, init=init)
    if q is not None:
        inputs['q'] = q
    if sal is not None:
        inputs['saliency'] = sal
    ts = {k: _t(v).requires_grad_() for k, v in inputs.items()}
    if iterations == 1:
        m = A.m_step(ts['y'], ts.get('q'), ts['init'], ts.get('saliency'), **kw)
    else:
        m = A.fit(ts['y'], ts['init'], iterations, saliency=ts.get('saliency'),
                  source_activity_mask=None if mask is None else _t(mask), **kw)
    yp = ts['y'] if probe is None else _t(probe)
    loss = (_t(R) * A.predict(yp, m)).sum() + 0.1 * A.log_likelihood(yp, m)
    g = torch.autograd.grad(loss, list(ts.values()))
    return {k: v.numpy() for k, v in zip(ts, g)}, inputs, m


MP_CASES = [
    # norm, options
    ('eigenvalue', {}),
    ('trace', {}),
    (False, {}),
    ('eigenvalue', {'saliency': True}),
    ('trace', {'saliency': True, 'q': True}),
    ('eigenvalue', {'weight_constant_axis': -2, 'q': True}),
    ('eigenvalue', {'iterations': 2, 'mask': True}),
    ('trace', {'iterations': 3, 'affiliation_eps': 0.}),
    (False, {'iterations': 2, 'saliency': True}),
]


@pytest.mark.parametrize('norm,opts', MP_CASES)
def test_m_step_and_fit_gradients_match_mpmath(norm, opts):
    F, T, D, K = 1, 10, 4, 2
    y, _ = synth.structured_stft(F, T, D, K, seed=21)
    init = synth.init_affiliation(F, K, T, seed=22)
    rng = np.random.RandomState(23)
    q = rng.uniform(0.5, 2.0, (F, K, T)) if opts.get('q') else None
    sal = rng.uniform(0.2, 1.0, (F, T)) if opts.get('saliency') else None
    mask = rng.uniform(size=(F, K, T)) > 0.25 if opts.get('mask') else None
    R = rng.standard_normal((F, K, T))
    it = opts.get('iterations', 1)
    kw = dict(covariance_norm=norm)
    mp_kw = dict(covariance_norm=norm, iterations=it, R=R, mask=mask)
    if 'weight_constant_axis' in opts:
        kw['weight_constant_axis'] = mp_kw['weight_constant_axis'] = opts['weight_constant_axis']
    if it > 1:
        kw['affiliation_eps'] = mp_kw['affiliation_eps'] = opts.get('affiliation_eps', 1e-10)
    grads, inputs, _ = _m_step_grads(y, init, q, sal, R, mask=mask, iterations=it, **kw)
    worst = _check_mp(grads, inputs, rng, 1e-11, **mp_kw)
    print(f'\nrestatement vs mpmath {norm} {opts}: worst err / bound {worst:.2e}')


def test_predict_and_log_likelihood_gradients_match_mpmath():
    F, T, D, K = 2, 12, 4, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=24)
    init = synth.init_affiliation(F, K, T, seed=25)
    m0 = A.m_step(_t(y), None, _t(init))
    inputs = dict(y=y, V=m0['eigenvectors'].numpy(), lam=m0['eigenvalues'].numpy(), w=m0['weight'][..., 0].numpy())
    rng = np.random.RandomState(26)
    R = rng.standard_normal((F, K, T))
    ts = {k: _t(v).requires_grad_() for k, v in inputs.items()}
    m = A.from_eig(ts['V'], ts['lam'], ts['w'][..., None])
    loss = (_t(R) * A.predict(ts['y'], m)).sum() + 0.1 * A.log_likelihood(ts['y'], m)
    g = dict(zip(ts, (v.numpy() for v in torch.autograd.grad(loss, list(ts.values())))))
    _check_mp(g, inputs, rng, 1e-11, iterations=0, R=R)


# ---- ties, near ties, floored blocks and the top eigenvalue ----------------------------------------------------------
@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
def test_spectral_model_at_an_exact_unfloored_tie_matches_central_differences(norm):
    """C = diag(0.5, 0.5, 1): a perturbation that splits the tied pair changes B^-1 at first order (the divided
    difference tends to -lam' / lam^2, not to 0)"""
    C = _t(np.diag([0.5, 0.5, 1.0]).astype(np.complex128))
    G = _t(np.random.RandomState(13).randn(3, 3) + 1j * np.random.RandomState(14).randn(3, 3))

    def loss(c):
        c = (c + c.mH) / 2
        with torch.no_grad():
            top = torch.linalg.eigh(c)[1][..., -1:]
        m = (top.mH @ c @ top).real[..., 0]
        binv, ld = A.SpectralModel.apply(c, m, 1e-3, norm)
        return (G.conj() * binv).real.sum() + 0.3 * ld

    Cg = C.clone().requires_grad_()
    loss(Cg).backward()
    h = 1e-6
    for i, j, part in [(0, 1, 1), (0, 1, 1j), (0, 0, 1), (1, 2, 1), (0, 2, 1j)]:
        E = torch.zeros(3, 3, dtype=torch.complex128)
        E[i, j] = part
        E[j, i] += np.conj(part) if i != j else 0
        num = (loss(C + h * E) - loss(C - h * E)).item() / (2 * h)
        ana = (Cg.grad.conj() * E).real.sum().item()
        assert abs(num - ana) <= 1e-6 * max(1.0, abs(num)), (i, j, part, num, ana)


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('D', [3, 5])
def test_exact_ties_below_the_top_match_mpmath(norm, D):
    # class 0: a pair tied below the top; class 1: one pair (D = 3) or two pairs (D = 5) tied below a simple top
    w0 = [0.3, 0.3] + [0.5 + 0.1 * d for d in range(D - 2)]
    w1 = [0.2, 0.2] + [0.45] * (D - 3) + [0.8]
    y, init, probe, R = A.tie_data(D, [w0, w1])
    grads, inputs, m = _m_step_grads(y, init, None, None, R, probe=probe, covariance_norm=norm)
    lam = m['eigenvalues'].numpy()[0]
    assert lam[0, 0] == lam[0, 1] and lam[1, 0] == lam[1, 1] and np.all(lam > 1e-10)
    _check_mp(grads, inputs, np.random.RandomState(D), 1e-11, n_dirs=3, covariance_norm=norm, R=R, probe=probe)


@pytest.mark.parametrize('gap', [1e-2, 1e-4, 1e-6, 1e-8, 1e-10, 1e-12])
@pytest.mark.parametrize('norm', ['eigenvalue', False])
def test_near_ties_match_mpmath(gap, norm):
    """a relative gap between two unfloored eigenvalues: the closed form has no cancellation, so the error stays far
    below u D / gap (the loss of a divided difference of computed eigenvalues)"""
    D = 4
    y, init, probe, R = A.tie_data(D, [[0.3, 0.3 * (1 + gap), 0.5, 0.9], [0.7, 0.2, 0.2 * (1 + gap), 0.4]], seed=1)
    grads, inputs, _ = _m_step_grads(y, init, None, None, R, probe=probe, covariance_norm=norm)
    rng = np.random.RandomState(2)
    worst = _check_mp(grads, inputs, rng, max(1e-11, U * D / gap), n_dirs=2, covariance_norm=norm, R=R, probe=probe)
    # and the closed form is accurate to ~1e-11 at every gap, not only within u D / gap
    _check_mp(grads, inputs, rng, 1e-11, n_dirs=1, covariance_norm=norm, R=R, probe=probe)
    print(f'\nnear tie gap {gap:.0e} {norm}: worst err / (u D / gap) {worst:.2e}')


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('rank', [1, 2, 3])
def test_floored_blocks_match_mpmath(norm, rank):
    """observations in a rank-r subspace of D = 4: D - r floored eigenvalues (multiplicity 3, 2, 1), whose block of
    B^-1 is 1 / floor and passes no gradient through the floor"""
    F, T, D, K = 1, 10, 4, 2
    rng = np.random.RandomState(30 + rank)
    basis = rng.randn(rank, D) + 1j * rng.randn(rank, D)
    y = ((rng.randn(T, rank) + 1j * rng.randn(T, rank)) @ basis)[None]
    init = synth.init_affiliation(F, K, T, seed=rank)
    probe = rng.randn(1, 5, D) + 1j * rng.randn(1, 5, D)
    R = rng.standard_normal((F, K, 5))
    floor = 1e-3
    grads, inputs, m = _m_step_grads(y, init, None, None, R, probe=probe, covariance_norm=norm, eigenvalue_floor=floor)
    lam = m['eigenvalues'].numpy()[0]
    assert np.sum(lam[0] == lam[0, 0]) == D - rank
    _check_mp(grads, inputs, rng, 1e-10, n_dirs=2, covariance_norm=norm, eigenvalue_floor=floor, R=R, probe=probe)


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
def test_tied_top_eigenvalue_follows_the_forwards_top_eigenvector(norm):
    """At a tie at the top, mu_max is not differentiable.  The convention: m is the Rayleigh quotient of the forward's
    top eigenvector, held fixed (the derivative of mu_max wherever the top is simple).  A floored eigenvalue makes m
    matter for every norm."""
    D = 4
    y, init, probe, R = A.tie_data(D, [[0.0, 0.4, 0.7, 0.7], [0.5, 0.0, 0.9, 0.9]], seed=3)
    grads, inputs, m = _m_step_grads(y, init, None, None, R, probe=probe, covariance_norm=norm, eigenvalue_floor=1e-3)
    lam = m['eigenvalues'].numpy()[0]
    assert lam[0, -1] == lam[0, -2] and lam[1, -1] == lam[1, -2]
    _check_mp(grads, inputs, np.random.RandomState(4), 1e-11, n_dirs=3, covariance_norm=norm, eigenvalue_floor=1e-3,
              R=R, probe=probe, top=m['eigenvectors'].numpy())


@pytest.mark.parametrize('dead', [0.0, 1e-310])
def test_dead_class_passes_no_gradient_and_no_nan(dead):
    """S_k <= tiny: exactly 0 (C_k = 0) or subnormal (C_k = D Psi_k / tiny, an O(1) covariance that depends on y)"""
    F, T, D, K = 1, 20, 4, 3
    y, _ = synth.structured_stft(F, T, D, K, seed=40)
    init = synth.init_affiliation(F, K, T, seed=41)
    init[0, 2] = dead
    probe = np.random.RandomState(42).randn(1, 5, D) + 1j * np.random.RandomState(43).randn(1, 5, D)
    R = np.random.RandomState(44).standard_normal((F, K, 5))
    q = np.random.RandomState(45).uniform(0.5, 2.0, (F, K, T))
    grads, _, m = _m_step_grads(y, init, q, None, R, probe=probe)
    assert np.all(np.isfinite(m['eigenvalues'].numpy()))
    for k, v in grads.items():
        assert np.all(np.isfinite(v)), k
    assert not np.any(grads['init'][0, 2]) and not np.any(grads['q'][0, 2])
