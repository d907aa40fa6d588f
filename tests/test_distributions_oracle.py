"""The NumPy restatement of the single distributions (oracle/distributions_oracle.py) against the fixture the
unmodified reference wrote (tests/golden/distributions.npz), and the reference's exported names.  CPU only."""
import importlib
import os

import numpy as np
import pytest

from oracle import distributions_oracle as DO

GOLD = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'distributions.npz'))


def _state_equal(key):
    s = np.random.get_state()
    return (np.array_equal(s[1], GOLD[f'{key}_state_keys']) and s[2] == GOLD[f'{key}_state_pos']
            and s[3] == GOLD[f'{key}_state_has_gauss'] and s[4] == GOLD[f'{key}_state_gauss'])


def test_every_exported_name_of_the_reference_imports():
    pkg = importlib.import_module('pb_bss_b200.distribution')
    names = [str(n) for n in GOLD['names']]
    assert {'ComplexAngularCentralGaussianTrainer', 'ComplexCircularSymmetricGaussian',
            'ComplexCircularSymmetricGaussianTrainer', 'sample_cacgmm'} <= set(names)
    missing = [n for n in names if not hasattr(pkg, n)]
    assert not missing, missing


@pytest.mark.parametrize('tag,floor,norm', [('eig', 0.0, 'eigenvalue'), ('trace', 0.0, 'trace'), ('none', 0.0, False),
                                            ('eig_floor', 1e-2, 'eigenvalue'), ('trace_floor', 1e-2, 'trace'),
                                            ('none_floor', 1e-2, False)])
def test_from_covariance(tag, floor, norm):
    V, lam = DO.cacg_from_covariance(DO.case_input('cov'), floor, norm)
    np.testing.assert_allclose(lam, GOLD[f'cov_{tag}_lam'], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(DO.covariance(V, lam), GOLD[f'cov_{tag}_cov'], rtol=1e-12, atol=1e-15)


def test_log_pdf_and_quadratic_form():
    _, y = DO.case_input('logpdf')
    V, lam = GOLD['logpdf_V'], GOLD['logpdf_lam']
    lp, q = DO.cacg_log_pdf(np.swapaxes(DO.unit_rows(y), -1, -2), V, lam)
    np.testing.assert_allclose(lp, GOLD['logpdf'], rtol=1e-12)
    np.testing.assert_allclose(lp, GOLD['logpdf_swapped'], rtol=1e-12)
    np.testing.assert_allclose(q, GOLD['logpdf_q'], rtol=1e-12)
    assert q[0, 0, 7] == DO.TINY


@pytest.mark.parametrize('D,norm,herm', [(D, 'eigenvalue', 1) for D in DO.FIT_DIMS]
                         + [(4, 'trace', 1), (4, 'False', 1), (3, 'eigenvalue', 0)])
def test_trainer_fit(D, norm, herm):
    V, lam = DO.cacg_fit(DO.case_input('fit', D), norm=False if norm == 'False' else norm)
    key = f'fit_d{D}_{norm}_{herm}'
    np.testing.assert_allclose(lam, GOLD[f'{key}_lam'], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(DO.covariance(V, lam), GOLD[f'{key}_cov'], rtol=1e-9, atol=1e-12)


def test_batched_fit_is_the_per_slice_fit():
    assert str(GOLD['batch_error']) == 'TypeError'
    V, lam = DO.cacg_fit(DO.case_input('batch'))
    np.testing.assert_allclose(lam, GOLD['batch_lam'], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(DO.covariance(V, lam), GOLD['batch_cov'], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize('tag', ['none', 'sal'])
def test_trainer_step(tag):
    z, q, sal = DO.case_input('step')
    V, lam = DO.cacg_step(z, q, sal if tag == 'sal' else None)
    np.testing.assert_allclose(lam, GOLD[f'step_{tag}_lam'], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(DO.covariance(V, lam), GOLD[f'step_{tag}_cov'], rtol=1e-10, atol=1e-13)


@pytest.mark.parametrize('D', DO.NORM_DIMS)
@pytest.mark.parametrize('variant', DO.VARIANTS)
def test_watson_log_norms(variant, D):
    k = DO.kappas(D)
    ref = GOLD[f'lognorm_{variant}_d{D}']
    o = DO.cw_log_norm(variant, k, D)
    fin = np.isfinite(ref)
    tol = 1e-12 * np.abs(ref[fin]) + DO.cw_log_norm_spread(variant, k, D)[fin]
    assert np.all(np.abs(o[fin] - ref[fin]) <= tol)
    if variant == '1f1':
        # scipy's hyp1f1 overflows beyond kappa ~ 710; the restatement stays finite and equals the closed form
        assert np.array_equal(fin, k < 700) and np.all(np.isfinite(o))
        np.testing.assert_allclose(o[k >= 700], DO.cw_log_norm('high', k[k >= 700], D), rtol=1e-12)
    else:
        assert np.array_equal(np.isfinite(o), fin)


def test_watson_normalisers_need_asfarray_under_numpy2():
    assert str(GOLD['lognorm_numpy2_error']) == ('AttributeError' if not hasattr(np, 'asfarray') else 'none')


def test_watson_log_pdf():
    mode, kappa, y = DO.case_input('watson')
    np.testing.assert_allclose(DO.cw_log_pdf(y, mode, kappa), GOLD['watson_logpdf'], rtol=1e-12)
    np.testing.assert_allclose(np.exp(DO.cw_log_pdf(y, mode, kappa)), GOLD['watson_pdf'], rtol=1e-11)


@pytest.mark.parametrize('D', DO.FIT_DIMS)
@pytest.mark.parametrize('sal', [True, False])
def test_watson_fit(D, sal):
    from pb_bss_b200.distribution import ComplexWatsonTrainer
    y, s = DO.case_input('wfit', D)
    lam, V = np.linalg.eigh(DO.cw_scatter(DO.unit_rows(y), s if sal else None))
    kappa = ComplexWatsonTrainer(D).hypergeometric_ratio_inverse(lam[-1])
    key = f'wfit_d{D}' + ('' if sal else '_nosal')
    assert abs(np.vdot(V[:, -1], GOLD[f'{key}_mode'])) == pytest.approx(1.0, abs=1e-12)
    np.testing.assert_allclose(kappa, GOLD[f'{key}_kappa'], rtol=1e-9, atol=1e-12)


def test_ccsg_log_pdf_and_fit():
    herm, nonherm, classes, y, yreal = DO.case_input('ccsg')
    for tag, cov, obs in (('herm', herm, y), ('nonherm', nonherm, y), ('classes', classes, y), ('real', herm, yreal)):
        np.testing.assert_allclose(DO.ccsg_log_pdf(obs, cov), GOLD[f'ccsg_{tag}'], rtol=1e-12)
    y, sal = DO.case_input('ccsg_fit')
    np.testing.assert_allclose(DO.ccsg_fit(y), GOLD['ccsg_fit_none'], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(DO.ccsg_fit(y, sal), GOLD['ccsg_fit_sal'], rtol=1e-12, atol=1e-15)


def test_samplers_reproduce_draws_and_rng_state():
    cov3, covK, weight = DO.sample_inputs()
    calls = {'ccsg': lambda: DO.ccsg_sample((7,), cov3), 'ccsg_empty': lambda: DO.ccsg_sample((0,), cov3),
             'cacg': lambda: DO.ccsg_sample((5,), DO.covariance(*DO.cacg_from_covariance(cov3)), True),
             'cacg_fn': lambda: DO.ccsg_sample((6,), cov3, True)}
    for key, fn in calls.items():
        np.random.seed(DO.SAMPLE_SEED)
        x = fn()
        assert _state_equal(f'sample_{key}'), key
        np.testing.assert_allclose(x, GOLD[f'sample_{key}'], rtol=1e-13, atol=1e-14)
    np.random.seed(DO.SAMPLE_SEED)
    x, labels = DO.sample_cacgmm(20, weight, covK)
    assert _state_equal('sample_cacgmm')
    assert np.array_equal(labels, GOLD['sample_cacgmm_labels'])
    np.testing.assert_allclose(x, GOLD['sample_cacgmm'], rtol=1e-13, atol=1e-14)
