"""CPU checks of oracle/em_oracle.py: the float64 oracle against the mpmath references on well-conditioned inputs,
where the two disagree (large condition numbers), the Watson normaliser over its whole domain, the input generators
and the softmax switch formulas."""
import numpy as np
import pytest

from oracle import em_oracle as E
from oracle import pb_bss_oracle as O

EPS = np.finfo(np.float64).eps


def _model(D, K, cond, seed):
    rng = np.random.default_rng(seed)
    from oracle import linalg_oracle as L
    V = np.stack([L.unitary(D, rng) for _ in range(K)])[None]
    lam = np.logspace(-np.log10(cond), 0, D)
    lam = np.broadcast_to(lam, (1, K, D)).copy()
    return dict(weight=np.full((1, K, 1), 1 / K), eigenvectors=V, eigenvalues=lam)


@pytest.mark.parametrize('D', [2, 5, 8, 17])
def test_quadratic_form_and_log_det_against_mpmath(D):
    """Well conditioned: the oracle's q and log det agree with 40 digits to a few eps of the error scale."""
    model = _model(D, 2, 10.0, seed=D)
    y = (np.random.default_rng(1).standard_normal((1, 20, D)) + 1j * np.random.default_rng(2).standard_normal((1, 20, D)))
    _, q = O.cacgmm_predict(y, model, return_quadratic_form=True)
    scale = E.q_error_scale(y, model)
    z = O.normalize_observation_cacg(y)[0]
    for k in range(2):
        qm = E.mp_quadratic_form(z, model['eigenvectors'][0, k], model['eigenvalues'][0, k])
        assert np.all(np.abs(q[0, k] - qm) <= 4 * D * EPS * scale[0, k])
        assert abs(np.sum(np.log(model['eigenvalues'][0, k])) - E.mp_log_det(model['eigenvalues'][0, k])) <= 4 * D * EPS


def test_oracle_q_error_grows_with_the_condition_number():
    """At cond 1e12 the float64 q of frames on the small eigenvector still agrees with mpmath within the error scale
    zᴴ|B⁻¹|z, which is then far above q itself for other frames -- the reason the device tests scale their bounds."""
    D = 6
    model = _model(D, 1, 1e12, seed=3)
    y = np.random.default_rng(4).standard_normal((1, 30, D)) + 0j
    _, q = O.cacgmm_predict(y, model, return_quadratic_form=True)
    scale = E.q_error_scale(y, model)
    qm = E.mp_quadratic_form(O.normalize_observation_cacg(y)[0], model['eigenvectors'][0, 0],
                             model['eigenvalues'][0, 0])
    err = np.abs(q[0, 0] - qm)
    assert np.all(err <= 4 * D * EPS * scale[0, 0])
    assert np.max(scale[0, 0] / q[0, 0]) > 10.0


def test_posterior_bound_covers_a_perturbation():
    rng = np.random.default_rng(0)
    q = rng.uniform(0.5, 5, size=(2, 3, 50))
    lp = -4 * np.log(q)
    w = np.full((2, 3, 1), 1 / 3)
    a = O.log_pdf_to_affiliation(w, lp)
    dq = 1e-6 * q
    a2 = O.log_pdf_to_affiliation(w, -4 * np.log(q * (1 + rng.uniform(-1e-6, 1e-6, q.shape))))
    assert np.all(np.abs(a2 - a) <= E.posterior_bound(a, q, 4 * dq))


@pytest.mark.parametrize('D', [2, 3, 4, 5, 8, 12, 17, 23, 34])
def test_watson_normaliser_scipy_matches_mpmath(D):
    """scipy.special.hyp1f1 (the reference's normaliser) against mpmath at D = 2..34 and kappa in [0, 500],
    including both sides of the device's series / closed-form switch at kappa = 20: they agree to 1e-13 in the log,
    so the oracle only falls back to mpmath where scipy's value is not finite."""
    kappa = np.r_[0.0, 1e-3, 0.5, 5.0, 10.0, 19.999, 20.0, 20.001, 50.0, 100.0, 250.0, 499.0, 500.0]
    m = E.mp_cw_log_norm(kappa, D)
    s = O.cw_log_norm(kappa, D)
    assert np.all(np.abs(s - m) <= 1e-13 * (1 + np.abs(m))), np.abs(s - m)
    assert np.all(np.abs(E.cw_log_norm(kappa, D) - m) <= 1e-13 * (1 + np.abs(m)))
    # kappa = 0: log(2 pi^D / (D-1)!)
    assert abs(m[0] - (np.log(2) + D * np.log(np.pi) - sum(np.log(np.arange(1, D))))) < 1e-13 * (1 + abs(m[0]))


def test_m_step_against_mpmath_on_graded_data():
    """One cACG M-step at cond 1e4 (float64 exact to eps lambda_max) and 1e11 (the smallest eigenvalue below the
    floor: float64 and mpmath both floor it)."""
    D, K, T = 4, 2, 40
    rng = np.random.default_rng(5)
    for cond in (1e4, 1e11):
        y, _ = E.graded_stft(1, T, D, K, cond, seed=7)
        a = rng.uniform(0.1, 1, size=(1, K, T))
        a /= a.sum(1, keepdims=True)
        q = rng.uniform(0.5, 2, size=(1, K, T))
        z = O.normalize_observation_cacg(y)
        ref = O.cacgmm_m_step(z, q, a)
        lam_f, lam_raw = E.mp_cacg_m_step(z[0], q[0], a[0])
        np.testing.assert_allclose(ref['eigenvalues'][0], lam_f, rtol=0, atol=16 * D * EPS)
        if cond == 1e11:
            assert np.all(lam_f[:, 0] == 1e-10) and np.all(lam_raw[:, 0] < 1e-10)


def test_graded_stft_conditions():
    """The class scatter matrices of graded data have lambda_min / lambda_max ~ 2^k / cond for any affiliation;
    rank-deficient data are exactly singular; zero frames are zero."""
    D, K, T = 6, 3, 400
    for cond in (1e4, 1e9):
        y, lab = E.graded_stft(2, T, D, K, cond, seed=1)
        for f in range(2):
            for k in range(K):
                x = y[f, lab[f] == k]
                x = x / np.linalg.norm(x, axis=-1, keepdims=True)
                w = np.linalg.eigvalsh(x.T @ x.conj())
                assert 0.1 / cond < w[0] / w[-1] < 100 * 2 ** k / cond
    y, _ = E.graded_stft(1, T, D, K, 1.0, seed=1, rank=D - 2, zero_frames=3)
    assert np.all(y[:, :3] == 0)
    s = np.linalg.svd(y[0, 3:], compute_uv=False)
    assert s[-2] < 1e-12 * s[0] and s[-3] > 1e-3 * s[0]


def test_extreme_model_structure():
    D, K, floor = 8, 4, 1e-11
    m = E.extreme_model(2, D, K, floor, seed=0)
    V, lam = m['eigenvectors'], m['eigenvalues']
    np.testing.assert_allclose(np.einsum('fkde,fkdg->fkeg', V.conj(), V), np.broadcast_to(np.eye(D), V.shape),
                               atol=1e-13)
    assert np.all(lam[..., -1] == 1) and np.all(lam[:, 0, :-1] == floor)
    np.testing.assert_allclose(np.abs(np.einsum('fd,fd->f', V[:, 0, :, 0].conj(), V[:, 1, :, -1])), 1, atol=1e-14)
    np.testing.assert_allclose(m['weight'][0, :, 0] / m['weight'][0, 0, 0], np.logspace(0, -12, K), rtol=1e-12)
    y, _ = E.extreme_stft(2, 30, D, K, floor, seed=0)
    _, q = O.cacgmm_predict(y, m, return_quadratic_form=True)
    assert q[:, 0, :10].min() > 1e-2 / floor   # frames on class 0's floor eigenvector


def test_softmax_switch_formulas():
    """The floors at which the switches of api_cacgmm.cu flip (e.g. D = 8, K = 4: lean down to ~8.3e-12, the
    per-iteration fast softmax down to ~3.2e-18)."""
    assert E.lean_ok(8, 4, 1e-11) and not E.lean_ok(8, 4, 1e-12)
    assert E.softmax_fast_ok(8, 1e-17) and not E.softmax_fast_ok(8, 1e-18)
    for D in (4, 6, 8):
        for K in (2, 3, 4):
            t = E.lean_threshold(D, K)
            assert E.lean_ok(D, K, t * 1.01) and not E.lean_ok(D, K, t / 1.01)
            f = E.fast_threshold(D)
            assert E.softmax_fast_ok(D, f * 1.01) and not E.softmax_fast_ok(D, f / 1.01)
    assert not E.softmax_fast_ok(4, 0.0) and not E.softmax_fast_ok(4, 2.0)
