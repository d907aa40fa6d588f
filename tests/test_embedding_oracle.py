"""Pins the NumPy restatements of the embedding mixture models (oracle/embedding_oracle.py: Gaussian, GMM, von
Mises-Fisher, VMFMM) to fixtures made by the unmodified reference (oracle/make_golden_embedding.py).  CPU only."""
import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import embedding_oracle as O
from conftest import load_golden

RT = dict(rtol=1e-12, atol=1e-14)

GMM_CASES = {
    'full': ('y0', 'init0', dict()),
    'full_b3': ('yb', 'initb', dict()),
    'diagonal': ('y0', 'init0', dict(covariance_type='diagonal')),
    'spherical': ('y0', 'init0', dict(covariance_type='spherical')),
    'full_fixed': ('y0', 'init0', dict(fixed_covariance='fixed_covariance')),
    'full_sal': ('y0', 'init0', dict(saliency='saliency')),
    'w_m2': ('y0', 'init0', dict(weight_constant_axis=-2)),
    'w_t2_sal': ('yb', 'initb', dict(weight_constant_axis=(-2,), saliency='saliency_b')),
}

VMF_CASES = {
    'vmf': ('y0', 'init0', dict()),
    'vmf_b2_maxc': ('yb', 'initb', dict(max_concentration=3.)),
    'vmf_sal_t2': ('y0', 'init0', dict(saliency='saliency', weight_constant_axis=(-2,))),
}


def resolve(g, kw):
    out = {}
    for k, v in kw.items():
        if v == 'saliency_b':
            v = np.broadcast_to(g['saliency'], g['yb'].shape[:-1]).copy()
        elif k in ('saliency', 'fixed_covariance'):
            v = g[v]
        out[k] = v
    return out


@pytest.mark.parametrize('name', list(GMM_CASES))
def test_gmm_oracle_matches_reference(name):
    g = load_golden('gmm')
    y, init, kw = GMM_CASES[name]
    model = O.gmm_fit(g[y], g[init], int(g['iterations']), **resolve(g, kw))
    np.testing.assert_allclose(model['weight'], g[f'{name}_weight'], **RT)
    np.testing.assert_allclose(model['gaussian']['mean'], g[f'{name}_mean'], **RT)
    np.testing.assert_allclose(model['gaussian']['covariance'], g[f'{name}_covariance'], **RT)
    np.testing.assert_allclose(O.gmm_predict(g[y], model), g[f'{name}_affiliation'], **RT)


def test_zero_saliency_observations_get_no_affiliation():
    """weight_constant_axis=(-2,): the reference's (..., 1, N) weight is 0 where the saliency is 0."""
    g = load_golden('gmm')
    zero = g['saliency'] == 0
    assert zero.any() and g['w_t2_sal_weight'].shape == (3, 1, g['y0'].shape[0])
    assert (g['w_t2_sal_weight'][..., zero] == 0).all() and (g['w_t2_sal_weight'][..., ~zero] == 1).all()
    assert (g['w_t2_sal_affiliation'][..., zero] == 0).all()


def test_gaussian_oracle_log_pdf_and_fit():
    g = load_golden('gmm')
    model = O.gaussian_model(g['full_b3_mean'], g['full_b3_covariance'], 'full')
    np.testing.assert_allclose(O.gaussian_model_log_pdf(model, g['logpdf_y']), g['logpdf'], **RT)
    sal = np.broadcast_to(g['saliency'], g['yb'].shape[:-1])
    for ct in ('full', 'diagonal', 'spherical'):
        fit = O.gaussian_fit(g['yb'], sal, ct)
        np.testing.assert_allclose(fit['mean'], g[f'fit_{ct}_mean'], **RT)
        np.testing.assert_allclose(fit['covariance'], g[f'fit_{ct}_covariance'], **RT)
    fit = O.gaussian_fit(g['y0'], None, 'full')
    np.testing.assert_allclose(fit['mean'], g['fit_nosal_mean'], **RT)
    np.testing.assert_allclose(fit['covariance'], g['fit_nosal_covariance'], **RT)


def test_full_log_pdf_is_the_density_only_for_a_diagonal_covariance():
    """The reference contracts U (upper triangular) as U d, not U^T d: equal to the Gaussian density for a diagonal
    covariance, different otherwise."""
    rng = np.random.RandomState(0)
    E = 4
    y = rng.randn(50, E)
    mean = rng.randn(E)
    diag = np.diag(rng.uniform(0.5, 2.0, E))
    m = O.gaussian_model(mean, diag, 'full')
    np.testing.assert_allclose(O.gaussian_model_log_pdf(m, y), multivariate_normal.logpdf(y, mean, diag),
                               rtol=1e-12)
    a = rng.randn(E, E)
    full = a @ a.T + 0.5 * np.eye(E)
    m = O.gaussian_model(mean, full, 'full')
    diff = np.abs(O.gaussian_model_log_pdf(m, y) - multivariate_normal.logpdf(y, mean, full))
    assert diff.max() > 1e-3


@pytest.mark.parametrize('name', list(VMF_CASES))
def test_vmfmm_oracle_matches_reference(name):
    g = load_golden('vmfmm')
    y, init, kw = VMF_CASES[name]
    model = O.vmfmm_fit(g[y], g[init], int(g['iterations']), **resolve(g, kw))
    np.testing.assert_allclose(model['weight'], g[f'{name}_weight'], **RT)
    np.testing.assert_allclose(model['mean'], g[f'{name}_mean'], **RT)
    np.testing.assert_allclose(model['concentration'], g[f'{name}_concentration'], **RT)
    np.testing.assert_allclose(O.vmfmm_predict(g[y], model), g[f'{name}_affiliation'], **RT)
    if name == 'vmf_b2_maxc':
        assert (model['concentration'] == 3.).any()


def test_vmf_oracle_fit():
    g = load_golden('vmfmm')
    yb = O._unit_rows(load_golden('gmm')['yb'])
    mean, conc = O.vmf_fit(yb, np.broadcast_to(g['saliency'], yb.shape[:-1]))
    np.testing.assert_allclose(mean, g['fit_mean'], **RT)
    np.testing.assert_allclose(conc, g['fit_concentration'], **RT)
