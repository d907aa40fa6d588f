"""The single distributions of pb_bss.distribution on the device -- ComplexAngularCentralGaussian (+ trainer),
ComplexWatson (+ trainer), ComplexCircularSymmetricGaussian (+ trainer), the samplers -- against the reference's
outputs in tests/golden/distributions.npz and the NumPy restatement (oracle/distributions_oracle.py).

Tolerances (fp64): log-pdfs and log normalisers rtol 1e-12, single steps rtol 1e-10, 10-iteration fits and kappa
through the spline rtol 1e-9 / atol 1e-12, samples rtol 1e-13.  Wider bounds carry their reason: the float64 spread
of the reference's own medium formula where its correction cancels (DO.cw_log_norm_spread), and the complex64
rounding of the reference's normalisation for complex64 input."""
import numpy as np
import pytest
import torch

from oracle import distributions_oracle as DO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold(golden):
    return golden('distributions')


def _dist():
    import pb_bss_b200.distribution as dist
    return dist


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _cov_close(model, cov, lam, rtol, atol=0.0):
    """Compare a cACG model through V diag(lambda) V^H: eigenvector phases are arbitrary."""
    scale = np.abs(lam).max()
    np.testing.assert_allclose(model.covariance_eigenvalues, lam, rtol=rtol, atol=atol + rtol * 1e-3 * scale)
    np.testing.assert_allclose(model.covariance, cov, rtol=rtol, atol=atol + rtol * 1e-3 * scale)


def _state_equal(gold, key):
    s = np.random.get_state()
    return (np.array_equal(s[1], gold[f'{key}_state_keys']) and s[2] == gold[f'{key}_state_pos']
            and s[3] == gold[f'{key}_state_has_gauss'] and s[4] == gold[f'{key}_state_gauss'])


# ---- complex angular central Gaussian -------------------------------------------------------------------------------
@pytest.mark.parametrize('tag,floor,norm', [('eig', 0.0, 'eigenvalue'), ('trace', 0.0, 'trace'), ('none', 0.0, False),
                                            ('eig_floor', 1e-2, 'eigenvalue'), ('trace_floor', 1e-2, 'trace'),
                                            ('none_floor', 1e-2, False)])
def test_from_covariance(gold, tag, floor, norm):
    CACG = _dist().ComplexAngularCentralGaussian
    c = DO.case_input('cov')
    arg = c.copy()
    m = CACG.from_covariance(arg, eigenvalue_floor=floor, covariance_norm=norm)
    assert np.array_equal(arg, c), 'the input is never changed'
    assert isinstance(m.covariance_eigenvalues, np.ndarray) and m.covariance_eigenvalues.shape == (3, 5)
    assert np.all(np.diff(m.covariance_eigenvalues, axis=-1) >= 0)
    _cov_close(m, gold[f'cov_{tag}_cov'], gold[f'cov_{tag}_lam'], rtol=1e-10)
    t = _cuda(c)
    mt = CACG.from_covariance(t, eigenvalue_floor=floor, covariance_norm=norm)
    assert mt.covariance_eigenvectors.is_cuda and torch.equal(t, _cuda(c))
    np.testing.assert_array_equal(mt.covariance_eigenvalues.cpu().numpy(), m.covariance_eigenvalues)


def test_log_pdf_broadcast_zero_frames_and_complex64(gold):
    CACG = _dist().ComplexAngularCentralGaussian
    _, y = DO.case_input('logpdf')
    m = CACG(covariance_eigenvectors=gold['logpdf_V'], covariance_eigenvalues=gold['logpdf_lam'])
    lp = m.log_pdf(y)  # model (3, 2, D, D) against y (3, 1, N, D)
    assert lp.shape == (3, 2, 50)
    np.testing.assert_allclose(lp, gold['logpdf'], rtol=1e-12)
    z = np.ascontiguousarray(np.swapaxes(DO.unit_rows(y), -1, -2))
    lp2, q = m._log_pdf(z)
    np.testing.assert_allclose(lp2, gold['logpdf_swapped'], rtol=1e-12)
    np.testing.assert_allclose(q, gold['logpdf_q'], rtol=1e-12)
    assert q[0, 0, 7] == np.finfo(np.float64).tiny
    assert m.log_pdf(y[..., :0, :]).shape == (3, 2, 0)
    # the reference normalises complex64 input in complex64: its quadratic forms carry that rounding, a few eps32
    # relative, which -D log q turns into an absolute error of a few D eps32
    lp64 = m.log_pdf(y.astype(np.complex64))
    np.testing.assert_allclose(lp64, gold['logpdf_c64'], rtol=1e-6, atol=8 * 4 * np.finfo(np.float32).eps)
    _, q64 = m._log_pdf(z.astype(np.complex64))
    assert q64[0, 0, 7] == np.float64(np.finfo(np.float32).tiny)
    mt = CACG(covariance_eigenvectors=_cuda(gold['logpdf_V']), covariance_eigenvalues=_cuda(gold['logpdf_lam']))
    lpt = mt.log_pdf(_cuda(y))
    assert lpt.is_cuda and np.array_equal(lpt.cpu().numpy(), lp)
    # a model broadcast along a leading dim that is not the last one takes the one-class path
    m2 = CACG(covariance_eigenvectors=gold['logpdf_V'][:, :1], covariance_eigenvalues=gold['logpdf_lam'][:, :1])
    np.testing.assert_allclose(m2.log_pdf(y), gold['logpdf'][:, :1], rtol=1e-12)


@pytest.mark.parametrize('D,norm,herm', [(D, 'eigenvalue', True) for D in DO.FIT_DIMS]
                         + [(4, 'trace', True), (4, False, True), (3, 'eigenvalue', False)])
def test_trainer_fit(gold, D, norm, herm):
    y = DO.case_input('fit', D)
    m = _dist().ComplexAngularCentralGaussianTrainer().fit(y, covariance_norm=norm, hermitize=herm)
    key = f'fit_d{D}_{norm}_{int(herm)}'
    _cov_close(m, gold[f'{key}_cov'], gold[f'{key}_lam'], rtol=1e-9, atol=1e-12)


def test_trainer_fits_every_leading_index(gold):
    y = DO.case_input('batch')
    m = _dist().ComplexAngularCentralGaussianTrainer().fit(y)
    assert str(gold['batch_error']) == 'TypeError'  # what the reference does with leading dims
    assert m.covariance_eigenvalues.shape == (2, 3, 4)
    _cov_close(m, gold['batch_cov'], gold['batch_lam'], rtol=1e-9, atol=1e-12)
    mt = _dist().ComplexAngularCentralGaussianTrainer().fit(_cuda(y))
    assert mt.covariance_eigenvalues.is_cuda
    np.testing.assert_array_equal(mt.covariance_eigenvalues.cpu().numpy(), m.covariance_eigenvalues)


@pytest.mark.parametrize('tag', ['none', 'sal'])
@pytest.mark.parametrize('herm', [True, False])
def test_trainer_step(gold, tag, herm):
    z, q, sal = DO.case_input('step')
    m = _dist().ComplexAngularCentralGaussianTrainer()._fit(z, sal if tag == 'sal' else None, q, hermitize=herm)
    assert m.covariance_eigenvalues.shape == (2, 4)  # y (1, D, N) against q (K, N)
    _cov_close(m, gold[f'step_{tag}_cov'], gold[f'step_{tag}_lam'], rtol=1e-10)


# ---- complex Watson -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', DO.NORM_DIMS)
@pytest.mark.parametrize('variant', DO.VARIANTS)
def test_watson_log_norms(gold, variant, D):
    CW = _dist().ComplexWatson
    fn = getattr(CW, f'log_norm_{variant}' if variant in ('1f1', 'tran_vu') else f'log_norm_{variant}_concentration')
    k = DO.kappas(D)
    got = fn(k, D)
    ref = gold[f'lognorm_{variant}_d{D}']
    assert got.shape == k.shape
    fin = np.isfinite(ref)
    spread = DO.cw_log_norm_spread(variant, k, D)
    # where 1 - S lies within the rounding of S (spread >= 1), float64 cannot resolve log(1 - S): the reference's
    # value there is rounding noise (medium formula, D = 8, at the clamp kappa = 1e-2); the port must give its own
    # value at the clamp for every kappa below it
    noise = spread >= 1.0
    chk = fin & ~noise
    tol = 1e-12 * np.abs(ref[chk]) + spread[chk]
    assert np.all(np.abs(got[chk] - ref[chk]) <= tol), (got, ref)
    if noise.any():
        assert variant == 'medium' and np.all(k[noise] <= 1e-2), (variant, k[noise])
        np.testing.assert_array_equal(got[noise], fn(np.full(int(noise.sum()), 1e-2), D))
    if variant == '1f1':
        assert np.all(np.isfinite(got)), 'finite where scipy overflows'
        np.testing.assert_allclose(got[~fin], DO.cw_log_norm('1f1', k[~fin], D), rtol=1e-12)
        assert isinstance(fn(20.1, D), np.float64)
    else:
        assert np.array_equal(np.isfinite(got[~noise]), fin[~noise])
    gt = fn(_cuda(k.reshape(2, 4)), D)
    assert gt.is_cuda and np.array_equal(gt.cpu().numpy().ravel(), got)


def test_watson_log_pdf_and_pdf(gold):
    CW = _dist().ComplexWatson
    mode, kappa, y = DO.case_input('watson')
    m = CW(mode=mode, concentration=kappa)
    ref = gold['watson_logpdf']
    np.testing.assert_allclose(m.log_pdf(y), ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    np.testing.assert_allclose(m.pdf(y), gold['watson_pdf'], rtol=1e-11)
    np.testing.assert_allclose(m.log_norm(), DO.cw_log_norm('1f1', kappa, 4), rtol=1e-12)
    # one y shared by every model, and complex64
    lp = m.log_pdf(y[0])
    np.testing.assert_allclose(lp, DO.cw_log_pdf(y[0], mode, kappa), rtol=1e-12, atol=1e-12 * np.abs(lp).max())
    np.testing.assert_allclose(m.log_pdf(y.astype(np.complex64)), DO.cw_log_pdf(y.astype(np.complex64), mode, kappa),
                               rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    mt = CW(mode=_cuda(mode), concentration=_cuda(kappa))
    out = mt.log_pdf(_cuda(y))
    assert out.is_cuda and mt.pdf(_cuda(y)).is_cuda
    np.testing.assert_array_equal(out.cpu().numpy(), m.log_pdf(y))


@pytest.mark.parametrize('D', DO.FIT_DIMS)
@pytest.mark.parametrize('sal', [True, False])
def test_watson_fit(gold, D, sal):
    dist = _dist()
    y, s = DO.case_input('wfit', D)
    s = s if sal else None
    key = f'wfit_d{D}' + ('' if sal else '_nosal')
    t = dist.ComplexWatsonTrainer()
    m = t.fit(y, saliency=s)
    assert t.dimension == D and m.mode.shape == (D,) and np.ndim(m.concentration) == 0
    assert abs(np.vdot(m.mode, gold[f'{key}_mode'])) == pytest.approx(1.0, abs=1e-10)
    np.testing.assert_allclose(m.concentration, gold[f'{key}_kappa'], rtol=1e-9, atol=1e-12)
    m2 = dist.ComplexWatsonTrainer(D)._fit(DO.unit_rows(y), s)
    assert abs(np.vdot(m2.mode, gold[f'{key}_mode'])) == pytest.approx(1.0, abs=1e-10)
    np.testing.assert_allclose(m2.concentration, gold[f'{key}_kappa'], rtol=1e-9, atol=1e-12)
    mt = dist.ComplexWatsonTrainer().fit(_cuda(y), saliency=None if s is None else _cuda(s))
    assert mt.mode.is_cuda and mt.concentration.is_cuda


# ---- complex circular-symmetric Gaussian ----------------------------------------------------------------------------
def test_ccsg_log_pdf(gold):
    CCSG = _dist().ComplexCircularSymmetricGaussian
    herm, nonherm, classes, y, yreal = DO.case_input('ccsg')
    for tag, cov, obs in (('herm', herm, y), ('nonherm', nonherm, y), ('classes', classes, y), ('real', herm, yreal)):
        got = CCSG(covariance=cov).log_pdf(obs)
        assert got.shape == gold[f'ccsg_{tag}'].shape, tag
        np.testing.assert_allclose(got, gold[f'ccsg_{tag}'], rtol=1e-12, err_msg=tag)
    # every class against its own frames, complex64 frames, zero frames, CUDA in / out
    yk = np.stack([y, 2 * y, y[::-1]])
    np.testing.assert_allclose(CCSG(covariance=classes).log_pdf(yk), DO.ccsg_log_pdf(yk, classes), rtol=1e-12)
    y64 = y.astype(np.complex64)
    np.testing.assert_allclose(CCSG(covariance=herm).log_pdf(y64), DO.ccsg_log_pdf(y64.astype(complex), herm),
                               rtol=1e-12)
    assert CCSG(covariance=classes).log_pdf(y[:0]).shape == (3, 0)
    out = CCSG(covariance=_cuda(nonherm)).log_pdf(_cuda(y))
    assert out.is_cuda
    np.testing.assert_allclose(out.cpu().numpy(), gold['ccsg_nonherm'], rtol=1e-12)


def test_ccsg_log_pdf_spreads_one_model_over_many_frames():
    CCSG = _dist().ComplexCircularSymmetricGaussian
    rng = np.random.default_rng(5)
    cov = DO.hermitian_pd(rng, D=8) + 0.3 * (rng.normal(size=(8, 8)) + 1j * rng.normal(size=(8, 8)))
    y = rng.normal(size=(300_001, 8)) + 1j * rng.normal(size=(300_001, 8))
    _, logdet = np.linalg.slogdet(cov)
    ref = -8 * np.log(np.pi) - logdet - np.einsum('nd,nd->n', y.conj(), np.linalg.solve(cov, y.T).T).real
    np.testing.assert_allclose(CCSG(covariance=cov).log_pdf(y), ref, rtol=1e-12)


def test_ccsg_singular_covariance_raises_linalg_error(gold):
    CCSG = _dist().ComplexCircularSymmetricGaussian
    assert str(gold['error_ccsg_singular']) == 'LinAlgError'
    _, _, classes, y, _ = DO.case_input('ccsg')
    sing = classes.copy()
    sing[1, 2, :] = 0  # a zero row: an exactly zero pivot
    with pytest.raises(np.linalg.LinAlgError):
        CCSG(covariance=sing).log_pdf(y)


@pytest.mark.parametrize('tag', ['none', 'sal'])
def test_ccsg_fit(gold, tag):
    y, sal = DO.case_input('ccsg_fit')
    s = sal if tag == 'sal' else None
    T = _dist().ComplexCircularSymmetricGaussianTrainer
    ref = gold[f'ccsg_fit_{tag}']
    np.testing.assert_allclose(T().fit(y, saliency=s).covariance, ref, rtol=1e-12, atol=1e-15)
    out = T().fit(_cuda(y), saliency=None if s is None else _cuda(s)).covariance
    assert out.is_cuda
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-12, atol=1e-15)


# ---- samplers -----------------------------------------------------------------------------------------------------
def test_samplers_match_reference_draws_and_leave_its_rng_state(gold):
    dist = _dist()
    from pb_bss_b200.distribution.complex_angular_central_gaussian import sample_complex_angular_central_gaussian
    cov3, _, _ = DO.sample_inputs()
    calls = {'ccsg': lambda: dist.ComplexCircularSymmetricGaussian(covariance=cov3).sample((7,)),
             'ccsg_empty': lambda: dist.ComplexCircularSymmetricGaussian(covariance=cov3).sample((0,)),
             'cacg': lambda: dist.ComplexAngularCentralGaussian.from_covariance(cov3).sample((5,)),
             'cacg_fn': lambda: sample_complex_angular_central_gaussian((6,), cov3)}
    for key, fn in calls.items():
        np.random.seed(DO.SAMPLE_SEED)
        x = fn()
        assert _state_equal(gold, f'sample_{key}'), key
        ref = gold[f'sample_{key}']
        assert x.shape == ref.shape and x.dtype == np.complex128, key
        np.testing.assert_allclose(x, ref, rtol=1e-13, atol=1e-13 * max(1.0, np.abs(ref).max(initial=0)), err_msg=key)
    np.random.seed(DO.SAMPLE_SEED)
    xt = dist.ComplexCircularSymmetricGaussian(covariance=_cuda(cov3)).sample((7,))
    assert xt.is_cuda
    np.testing.assert_allclose(xt.cpu().numpy(), gold['sample_ccsg'], rtol=1e-13, atol=1e-13)


def test_sample_cacgmm_equals_the_per_class_loop_exactly(gold):
    dist = _dist()
    _, covK, weight = DO.sample_inputs()
    np.random.seed(DO.SAMPLE_SEED)
    x, labels = dist.sample_cacgmm(20, weight, covK, return_label=True)
    assert _state_equal(gold, 'sample_cacgmm')
    np.testing.assert_array_equal(labels, gold['sample_cacgmm_labels'])
    np.testing.assert_allclose(x, gold['sample_cacgmm'], rtol=1e-13, atol=1e-13)
    assert not np.any(labels == 1)  # weight 0: a class with zero samples
    # the reference's test_sample_cacgmm: the same as drawing the labels and sampling class by class
    np.random.seed(DO.SAMPLE_SEED)
    labels2 = np.random.choice(range(3), size=20, p=weight)
    x2 = np.zeros((20, 3), dtype=np.complex128)
    for k in range(3):
        x2[labels2 == k] = dist.ComplexAngularCentralGaussian.from_covariance(covK[k]).sample(
            (int(np.sum(labels2 == k)),))
    np.testing.assert_array_equal(x, x2)
    np.random.seed(DO.SAMPLE_SEED)
    np.testing.assert_array_equal(dist.sample_cacgmm(20, weight, covK), x)
    np.random.seed(DO.SAMPLE_SEED)
    xt = dist.sample_cacgmm(20, weight, _cuda(covK))
    assert xt.is_cuda and np.array_equal(xt.cpu().numpy(), x)


# ---- errors ---------------------------------------------------------------------------------------------------------
def test_error_types(gold):
    dist = _dist()
    CACG, CACGT = dist.ComplexAngularCentralGaussian, dist.ComplexAngularCentralGaussianTrainer
    CCSG, CCSGT = dist.ComplexCircularSymmetricGaussian, dist.ComplexCircularSymmetricGaussianTrainer
    CWT = dist.ComplexWatsonTrainer
    c = DO.case_input('cov')
    yf = DO.case_input('fit', 4)
    z, q, _ = DO.case_input('step')
    herm, _, classes, y, _ = DO.case_input('ccsg')
    _, covK, weight = DO.sample_inputs()
    cases = {
        'from_covariance_norm': lambda: CACG.from_covariance(c.copy(), covariance_norm='frobenius'),
        'from_covariance_nonfinite': lambda: CACG.from_covariance(np.full((3, 3), np.inf + 0j)),
        'cacg_fit_saliency': lambda: CACGT().fit(yf, saliency=np.ones(yf.shape[0])),
        'cacg_fit_real': lambda: CACGT().fit(yf.real),
        'cacg_fit_d1': lambda: CACGT().fit(yf[:, :1]),
        'cacg_step_real': lambda: CACGT()._fit(z.real, None, q),
        'ccsg_sample_ndim': lambda: CCSG(covariance=classes).sample((3,)),
        'ccsg_sample_int': lambda: CCSG(covariance=herm).sample(3),
        'ccsg_sample_2d': lambda: CCSG(covariance=herm).sample((2, 3)),
        'ccsg_sample_not_pd': lambda: CCSG(covariance=-herm).sample((3,)),
        'ccsg_fit_type': lambda: CCSGT().fit(y, covariance_type='diagonal'),
        'ccsg_fit_real': lambda: CCSGT().fit(y.real),
        'cw_fit_real': lambda: CWT().fit(yf.real),
        'cw_fit_dim': lambda: CWT(3).fit(yf),
        'sample_cacgmm_size': lambda: dist.sample_cacgmm((3,), weight, covK),
        'sample_cacgmm_weight': lambda: dist.sample_cacgmm(3, weight[None], covK),
        'sample_cacgmm_cov': lambda: dist.sample_cacgmm(3, weight, covK[0]),
    }
    for key, fn in cases.items():
        want = str(gold[f'error_{key}'])
        with pytest.raises(Exception) as info:
            fn()
        assert type(info.value).__name__ == want, (key, info.value)
    with pytest.raises(np.linalg.LinAlgError):
        CACG.from_covariance(np.full((3, 3), np.inf + 0j), eigenvalue_floor=1e-10)
    # a size of two or more dims raises before any draw
    state = np.random.get_state()
    with pytest.raises(ValueError):
        CACG.from_covariance(herm).sample((4, 4))
    assert np.array_equal(np.random.get_state()[1], state[1]) and np.random.get_state()[2] == state[2]


# ---- the whole dimension domain, zero frames, the dtype's floor -----------------------------------------------------
@pytest.mark.parametrize('D', [59, 60, 64])
def test_ccsg_log_pdf_and_samplers_up_to_d64(D):
    """Up to D = 64 the factorisations of one warp each fit the CTA's shared memory."""
    dist = _dist()
    rng = np.random.default_rng(D)
    classes = DO.hermitian_pd(rng, 3, D=D)
    nonherm = classes + 0.1 * (rng.normal(size=(3, D, D)) + 1j * rng.normal(size=(3, D, D)))
    y = rng.normal(size=(3, 40, D)) + 1j * rng.normal(size=(3, 40, D))
    np.testing.assert_allclose(dist.ComplexCircularSymmetricGaussian(covariance=nonherm).log_pdf(y),
                               DO.ccsg_log_pdf(y, nonherm), rtol=1e-12)
    # the Cholesky factor of a D = 64 matrix sums up to 64 rounded products per entry, on the device and in LAPACK
    # alike: samples agree to a few D eps of their scale
    tol = dict(rtol=1e-12, atol=1e-12)
    np.random.seed(D)
    x = dist.ComplexCircularSymmetricGaussian(covariance=classes[0]).sample((9,))
    np.random.seed(D)
    np.testing.assert_allclose(x, DO.ccsg_sample((9,), classes[0]), **tol)
    np.random.seed(D)
    x = dist.ComplexAngularCentralGaussian.from_covariance(classes[1]).sample((9,))
    np.random.seed(D)
    V, lam = DO.cacg_from_covariance(classes[1])
    np.testing.assert_allclose(x, DO.ccsg_sample((9,), DO.covariance(V, lam), True), **tol)
    np.random.seed(D)
    x, labels = dist.sample_cacgmm(30, np.array([0.2, 0.3, 0.5]), classes, return_label=True)
    np.random.seed(D)
    ox, ol = DO.sample_cacgmm(30, np.array([0.2, 0.3, 0.5]), classes)
    np.testing.assert_array_equal(labels, ol)
    np.testing.assert_allclose(x, ox, **tol)


def test_trainers_without_frames():
    """As the reference: the cACG scatter of no frames is zero (identity eigenvectors, floored eigenvalues), the
    Watson scatter 0 / 0 raises LinAlgError, the Gaussian's covariance is 0 / 0 = NaN, or 0 with a saliency."""
    dist = _dist()
    y = np.zeros((2, 0, 4), dtype=np.complex128)
    m = dist.ComplexAngularCentralGaussianTrainer().fit(y)
    np.testing.assert_array_equal(m.covariance_eigenvalues, np.full((2, 4), 1e-10))
    np.testing.assert_array_equal(m.covariance_eigenvectors, np.broadcast_to(np.eye(4), (2, 4, 4)))
    m = dist.ComplexAngularCentralGaussianTrainer().fit(_cuda(y), covariance_norm=False)
    assert m.covariance_eigenvalues.is_cuda and not m.covariance_eigenvalues.cpu().numpy().any()
    m = dist.ComplexAngularCentralGaussianTrainer()._fit(np.zeros((1, 4, 0), complex), None, np.ones((3, 0)))
    np.testing.assert_array_equal(m.covariance_eigenvalues, np.full((3, 4), 1e-10))
    with pytest.raises(np.linalg.LinAlgError):
        dist.ComplexWatsonTrainer().fit(y)
    T = dist.ComplexCircularSymmetricGaussianTrainer
    assert np.isnan(T().fit(y).covariance).all()
    np.testing.assert_array_equal(T().fit(y, saliency=np.zeros((2, 0))).covariance, np.zeros((2, 4, 4)))


def test_ccsg_fit_floors_the_saliency_sum_at_the_tiny_of_y():
    """complex64 y: the reference floors sum_n s at the float32 tiny, above a saliency sum of 1e-298."""
    y, _ = DO.case_input('ccsg_fit')
    y64 = y.astype(np.complex64)
    sal = np.full(y.shape[:-1], 1e-300)
    got = _dist().ComplexCircularSymmetricGaussianTrainer().fit(y64, saliency=sal).covariance
    y64 = y64.astype(np.complex128)
    want = np.einsum('...n,...nd,...ne->...de', sal, y64, y64.conj()) * (1.0 / np.finfo(np.float32).tiny)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
