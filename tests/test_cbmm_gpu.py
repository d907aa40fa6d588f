"""The device complex Bingham mixture model against the oracle (oracle/bingham_oracle.py, same equations solved
to convergence) and against the reference's fixtures (oracle/make_golden_bingham.py).  Eigenvectors have an
arbitrary phase, so they are compared through V diag(s) V^H."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import bingham_oracle as B
from oracle import synth

pytestmark = pytest.mark.gpu


def _cov(V, lam):
    return B.model_covariance(V, lam)


def _assert_model(model, ref, rtol, s=None):
    cb = model.complex_bingham
    np.testing.assert_allclose(cb.covariance_eigenvalues, ref['lam'], rtol=rtol, atol=rtol * 1e-3)
    s = np.broadcast_to(np.arange(1, ref['lam'].shape[-1] + 1, dtype=float), ref['lam'].shape) if s is None else s
    np.testing.assert_allclose(_cov(cb.covariance_eigenvectors, s), _cov(ref['V'], s), atol=1e-9)
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=rtol, atol=1e-12)


@pytest.mark.parametrize('D', [2, 3, 4, 5, 6])
def test_single_m_step(D):
    from pb_bss_b200.distribution import CBMMTrainer
    g = load_golden('cbmm_steps')
    p = f'mstep_d{D}_'
    y, aff = g[p + 'y'], g[p + 'aff']
    model = CBMMTrainer().fit(y, initialization=aff, iterations=1)
    ref = B.cbmm_m_step(B.normalize_observation_cw(y), aff, np.ones_like(aff[:, 0]))
    _assert_model(model, ref, 1e-9)
    # against the reference: its parameter solve stops early (5e-4 relative)
    np.testing.assert_allclose(model.complex_bingham.covariance_eigenvalues, g[p + 'lam'], rtol=5e-4, atol=1e-9)
    np.testing.assert_allclose(model.weight, g[p + 'weight'], rtol=1e-12)


def test_known_answers_and_log_norm():
    from pb_bss_b200.distribution import ComplexBingham, ComplexBinghamTrainer
    g = load_golden('cbmm_steps')
    T = ComplexBinghamTrainer
    np.testing.assert_allclose(T.find_eigenvalues_v3(g['known_s2']), g['known_lam2'], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(T.find_eigenvalues_v3(g['known_s6']), g['known_lam6'], rtol=5e-7)
    np.testing.assert_allclose(T.find_eigenvalues_v3(g['known_s6'], max_concentration=500),
                               g['known_lam6_mc500'], rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(ComplexBingham(None, g['known_norm_lam']).norm(), g['known_norm'], rtol=1e-13)
    lam = np.array([[1, .1, .1], [1, .1, 0.]])
    np.testing.assert_allclose(ComplexBingham(None, lam).log_norm(), B.log_norm(lam), rtol=1e-13)
    np.testing.assert_allclose(ComplexBingham(None, lam).norm(remove_duplicate_eigenvalues=False),
                               np.exp(B.log_norm(lam, 0)), rtol=1e-13)


def test_batched_parameters_match_oracle():
    from pb_bss_b200.distribution import ComplexBinghamTrainer
    rng = np.random.RandomState(3)
    for D in range(2, 7):
        a = rng.randn(40, D, 3 * D) + 1j * rng.randn(40, D, 3 * D)
        s = np.linalg.eigvalsh(a @ a.conj().swapaxes(-1, -2))
        s /= s.sum(-1, keepdims=True)
        s = s.reshape(4, 10, D)
        for mc in (np.inf, 20.):
            lam = ComplexBinghamTrainer.find_eigenvalues_v3(s, max_concentration=mc)
            ref = np.array([B.find_eigenvalues_v3(v, max_concentration=mc) for v in s.reshape(-1, D)])
            np.testing.assert_allclose(lam.reshape(-1, D), ref, rtol=1e-9, atol=1e-12)
            if np.isinf(mc):
                assert max(B.residual_norm(l, v) for l, v in zip(lam.reshape(-1, D), s.reshape(-1, D))) <= 1e-12


def test_predict_and_log_pdf_from_reference_model():
    from pb_bss_b200.distribution import CBMM, ComplexBingham
    g = load_golden('cbmm_fit')
    y = g['y']
    for it in (2, 5):
        m = CBMM(weight=g[f'fit{it}_weight'],
                 complex_bingham=ComplexBingham(g[f'fit{it}_V'], g[f'fit{it}_lam']))
        np.testing.assert_allclose(m.predict(y), g[f'fit{it}_affiliation'], atol=1e-10)
        np.testing.assert_allclose(m.predict(y, affiliation_eps=1e-3), g[f'fit{it}_affiliation_eps'], atol=1e-10)
    s = load_golden('cbmm_steps')
    z = B.normalize_observation_cw(s['mstep_d5_y'])
    cb = ComplexBingham(s['mstep_d5_V'], s['mstep_d5_lam'])
    np.testing.assert_allclose(cb.log_pdf(z[:, None]), s['mstep_d5_log_pdf'], rtol=1e-10)


@pytest.mark.parametrize('F,T,D,K,I', [(5, 150, 4, 2, 20), (3, 120, 6, 3, 10), (4, 90, 3, 2, 8), (3, 80, 5, 4, 6),
                                       (4, 70, 2, 3, 8)])
def test_fit_matches_oracle(F, T, D, K, I):
    from pb_bss_b200.distribution import CBMMTrainer
    y, _ = synth.structured_stft(F, T, D, K, seed=F * T + D)
    init = synth.init_affiliation(F, K, T, seed=K)
    ref = B.cbmm_fit(y, init, I)
    model = CBMMTrainer().fit(y, initialization=init, iterations=I)
    _assert_model(model, ref, 1e-6)
    np.testing.assert_allclose(model.predict(y), B.cbmm_predict(y, ref), atol=1e-8)


def test_fits_match_reference_golden():
    from pb_bss_b200.distribution import CBMMTrainer
    g = load_golden('cbmm_fit')
    y, init = g['y'], g['init']
    m = CBMMTrainer().fit(y, initialization=init, iterations=2)
    np.testing.assert_allclose(m.predict(y), g['fit2_affiliation'], atol=1e-3)
    for name, kw in (('sal', dict(saliency=g['saliency'])), ('eps', dict(affiliation_eps=1e-2))):
        m = CBMMTrainer().fit(y, initialization=init, iterations=2, **kw)
        np.testing.assert_allclose(m.predict(y), g[f'{name}_affiliation'], atol=1e-3)
        ref = B.cbmm_fit(y, init, 2, **kw)
        _assert_model(m, ref, 1e-6)
    m = CBMMTrainer(max_concentration=5.).fit(y, initialization=init, iterations=2)
    _assert_model(m, B.cbmm_fit(y, init, 2, max_concentration=5.), 1e-6)
    np.testing.assert_allclose(m.complex_bingham.covariance_eigenvalues, g['mc5_lam'], rtol=5e-3, atol=1e-7)
    m = CBMMTrainer().fit(g['yb'], initialization=g['initb'], iterations=2)
    assert m.weight.shape == (2, 2, 2, 1) and m.complex_bingham.covariance_eigenvectors.shape == (2, 2, 2, 4, 4)
    np.testing.assert_allclose(m.predict(g['yb']), g['batch_affiliation'], atol=1e-3)


@pytest.mark.parametrize('name,axis', [('tied_time', (-3,)), ('tied', (-3, -1)), ('inline_pa', (-3,))])
def test_coupled_fit_matches_reference_golden(name, axis):
    from pb_bss_b200.distribution import CBMMTrainer
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    g = load_golden('cbmm_coupled')
    al = None
    if name == 'inline_pa':
        al = DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                      main_iterations=5, sub_iterations=2)
        assert al.alignment_plan == g['plan'].tolist()
    m = CBMMTrainer().fit(g['y'], initialization=g['init'], iterations=2, weight_constant_axis=axis,
                          inline_permutation_aligner=al)
    assert m.weight.shape == g[f'{name}_weight'].shape
    np.testing.assert_allclose(m.weight, g[f'{name}_weight'], atol=1e-3)
    np.testing.assert_allclose(m.predict(g['y']), g[f'{name}_affiliation'], atol=1e-3)


def test_complex64_storage_and_tensor_io():
    import torch
    from pb_bss_b200.distribution import CBMMTrainer
    y, _ = synth.structured_stft(4, 100, 4, 2, seed=9)
    init = synth.init_affiliation(4, 2, 100, seed=1)
    ref = CBMMTrainer().fit(y, initialization=init, iterations=5)
    m = CBMMTrainer().fit(y.astype(np.complex64), initialization=init, iterations=5)
    np.testing.assert_allclose(m.predict(y), ref.predict(y), atol=1e-3)
    yt = torch.from_numpy(y).cuda()
    mt = CBMMTrainer().fit(yt, initialization=init, iterations=5)
    assert isinstance(mt.complex_bingham.covariance_eigenvalues, torch.Tensor)
    aff = mt.predict(yt)
    assert isinstance(aff, torch.Tensor) and aff.is_cuda
    np.testing.assert_array_equal(aff.cpu().numpy(), ref.predict(y))


def test_num_classes_leading_dims_and_reruns():
    from pb_bss_b200.distribution import CBMMTrainer
    y = synth.structured_stft(6, 60, 4, 2, seed=2)[0].reshape(2, 3, 60, 4)
    np.random.seed(3)
    m = CBMMTrainer().fit(y, num_classes=2, iterations=4)
    assert m.weight.shape == (2, 3, 2, 1)
    assert m.complex_bingham.covariance_eigenvectors.shape == (2, 3, 2, 4, 4)
    np.random.seed(3)
    init = np.random.uniform(size=(2, 3, 2, 60))
    init /= np.einsum('...kn->...n', init)[..., None, :]
    ref = B.cbmm_fit(y, init, 4)
    np.testing.assert_allclose(m.complex_bingham.covariance_eigenvalues, ref['lam'], rtol=1e-6)
    again = CBMMTrainer().fit(y, initialization=init, iterations=4)
    assert np.array_equal(again.complex_bingham.covariance_eigenvalues, m.complex_bingham.covariance_eigenvalues)
    assert np.array_equal(again.complex_bingham.covariance_eigenvectors, m.complex_bingham.covariance_eigenvectors)
    aff = CBMMTrainer().fit_predict(y, initialization=init, iterations=4)
    np.testing.assert_array_equal(aff, m.predict(y))


def test_error_types():
    from pb_bss_b200.distribution import CBMMTrainer, ComplexBinghamTrainer
    y = synth.noise_stft(2, 3, 4, seed=1)                      # T < D: rank-deficient scatter
    with pytest.raises(AssertionError, match='numerically zero'):
        CBMMTrainer().fit(y, initialization=synth.init_affiliation(2, 2, 3), iterations=2)
    y7 = synth.noise_stft(2, 30, 7, seed=1)
    with pytest.raises(KeyError):
        CBMMTrainer().fit(y7, initialization=synth.init_affiliation(2, 2, 30), iterations=2)
    with pytest.raises(ValueError):
        ComplexBinghamTrainer.find_eigenvalues_v3([0, .5, .5])
    with pytest.raises(ValueError, match='problem 1'):
        ComplexBinghamTrainer.find_eigenvalues_v3([[.2, .3, .5], [-1e-3, .5, .5]])
