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
