"""The NumPy restatement of the complex Bingham mixture model (oracle/bingham_oracle.py) against the fixtures the
unmodified reference wrote (oracle/make_golden_bingham.py).  CPU only.

The reference's parameter solve stops at residuals of ~1e-7 (scipy least squares with default tolerances), the
oracle solves the same equations to 1e-12: parameters agree to 5e-4 relative, and everything computed from given
parameters (normaliser, log pdf, posterior, scatter) agrees to rounding."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import bingham_oracle as B
from oracle import synth


def test_known_answers():
    g = load_golden('cbmm_steps')
    np.testing.assert_allclose(B.find_eigenvalues_v3(g['known_s2']), g['known_lam2'], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(B.find_eigenvalues_v3(g['known_s6']), g['known_lam6'], rtol=5e-7)
    np.testing.assert_allclose(B.find_eigenvalues_v3(g['known_s6'], max_concentration=500), g['known_lam6_mc500'],
                               rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(np.exp(B.log_norm(g['known_norm_lam'])), g['known_norm'], rtol=1e-13)
    assert abs(g['known_norm'] - 84.71169626134224) < 1e-10
    # exact value at a repeated eigenvalue, complex_bingham.py:120-122
    exact = 2 * np.pi ** 3 * (np.exp(1) / 0.9 ** 2 - np.exp(0.1) / 0.9 ** 2 + np.exp(0.1) / (0.1 - 1))
    np.testing.assert_allclose(np.exp(B.log_norm(np.array([1, .1, .1]), eps=0)), exact, rtol=1e-14)


@pytest.mark.parametrize('D', [2, 3, 4, 5, 6])
def test_single_m_step_matches_reference(D):
    g = load_golden('cbmm_steps')
    p = f'mstep_d{D}_'
    z = B.normalize_observation_cw(g[p + 'y'])
    aff = g[p + 'aff']
    np.testing.assert_allclose(np.linalg.eigvalsh(B.scatter(z[:, None], aff)), g[p + 'scatter_eig'], rtol=1e-12)
    model = B.cbmm_m_step(z, aff, np.ones_like(aff[:, 0]))
    np.testing.assert_allclose(model['weight'], g[p + 'weight'], rtol=1e-13)
    s = g[p + 'scatter_eig']
    np.testing.assert_allclose(B.model_covariance(model['V'], s), B.model_covariance(g[p + 'V'], s), atol=1e-13)
    np.testing.assert_allclose(model['lam'], g[p + 'lam'], rtol=5e-4, atol=1e-9)
    for idx in np.ndindex(s.shape[:-1]):
        assert B.residual_norm(model['lam'][idx], s[idx]) <= 1e-12
    # E-step quantities from the REFERENCE's model
    lp = B.log_pdf(z[:, None], g[p + 'V'], g[p + 'lam'])
    np.testing.assert_allclose(lp, g[p + 'log_pdf'], rtol=1e-10)
    post = B.log_pdf_to_affiliation(g[p + 'weight'], lp)
    np.testing.assert_allclose(post, g[p + 'posterior'], rtol=1e-10, atol=1e-14)


def test_predict_and_fits_match_reference():
    g = load_golden('cbmm_fit')
    y, init = g['y'], g['init']
    for it in (2, 5):
        ref = dict(weight=g[f'fit{it}_weight'], V=g[f'fit{it}_V'], lam=g[f'fit{it}_lam'])
        np.testing.assert_allclose(B.cbmm_predict(y, ref), g[f'fit{it}_affiliation'], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(B.cbmm_predict(y, ref, 1e-3), g[f'fit{it}_affiliation_eps'], rtol=1e-9, atol=1e-12)
    ref = B.cbmm_fit(y, init, 2)
    np.testing.assert_allclose(B.cbmm_predict(y, ref), g['fit2_affiliation'], atol=1e-3)
    np.testing.assert_allclose(ref['lam'], g['fit2_lam'], rtol=5e-3)
    for name, kw in (('sal', dict(saliency=g['saliency'])), ('mc5', dict(max_concentration=5.)),
                     ('eps', dict(affiliation_eps=1e-2))):
        m = B.cbmm_fit(y, init, 2, **kw)
        np.testing.assert_allclose(m['weight'], g[f'{name}_weight'], atol=2e-3)
        if name == 'mc5':
            # the clamp at -max_concentration leaves eigenvalues 1e-8 apart, where the reference's term-by-term
            # normaliser cancels catastrophically (its posteriors are off by ~0.07): compare the parameters only
            np.testing.assert_allclose(m['lam'], g['mc5_lam'], rtol=5e-3, atol=1e-7)
            continue
        np.testing.assert_allclose(B.cbmm_predict(y, m), g[f'{name}_affiliation'], atol=1e-3)


def test_error_types():
    with pytest.raises(ValueError):
        B.find_eigenvalues_v3([0, .5, .5])          # x0 = -inf (complex_bingham.py:378)
    with pytest.raises(ValueError):
        B.find_eigenvalues_v3([-1e-3, .5, .5])      # x0 above the upper bound
    y = synth.noise_stft(1, 3, 4, seed=1)         # T < D: rank-deficient scatter
    with pytest.raises(AssertionError):
        B.bingham_fit(B.normalize_observation_cw(y), np.ones((1, 3)))


def test_divided_differences_against_closed_form():
    rng = np.random.RandomState(0)
    for D in range(2, 7):
        lam = np.sort(-rng.uniform(0, 50, size=D))
        lam[-1] = 0
        c = sum(np.exp(l) / np.prod([l - m for m in lam if m != l]) for l in lam)
        np.testing.assert_allclose(B.dd_exp(lam)[0, -1], c, rtol=1e-11)
        g, H = B.derivatives(lam)
        np.testing.assert_allclose(g.sum(), 1, atol=1e-13)
        np.testing.assert_allclose(H.sum(0), 0, atol=1e-12)
        h = 1e-6
        for k in range(D):
            e = np.zeros(D)
            e[k] = h
            fd = (B.log_norm(lam + e, 0) - B.log_norm(lam - e, 0)) / (2 * h)
            np.testing.assert_allclose(g[k], fd, rtol=1e-6, atol=1e-9)
