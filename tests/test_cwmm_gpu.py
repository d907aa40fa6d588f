"""Parity of the CUDA complex-Watson mixture model against the reference's
golden fixtures and the oracle.  The Watson mode has an arbitrary phase
(eigenvector), so modes are compared through |<a, b>| (cos similarity)."""
import numpy as np
import pytest

from conftest import load_golden, cos_similarity
from oracle import pb_bss_oracle as O
from oracle import synth
from test_em_kernels_gpu import last_plan

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', ['cwmm_d6k4', 'cwmm_d4k2'])
def test_fit_matches_reference_golden(name):
    from pb_bss_b200.distribution import CWMMTrainer
    g = load_golden(name)
    model = CWMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']))
    assert model.weight.shape == g['weight'].shape
    assert model.complex_watson.mode.shape == g['mode'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.complex_watson.concentration, g['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(model.complex_watson.mode, g['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(np.linalg.norm(model.complex_watson.mode, axis=-1), 1, atol=1e-12)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize('name,axis', [('cwmm_tied_time', (-3,)), ('cwmm_tied', (-3, -1)), ('cwmm_inline_pa', (-3,))])
def test_coupled_fit_matches_reference_golden(name, axis):
    """Frequency-tied weights (weight_constant_axis (-3,) / (-3, -1)) and the inline permutation alignment
    (cwmm.py:152-184): per-iteration loop of device kernels, fixtures from the unmodified reference."""
    from pb_bss_b200.distribution import CWMMTrainer
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    g = load_golden(name)
    al = None
    if 'plan' in g:
        al = DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                      main_iterations=5, sub_iterations=2)
        assert al.alignment_plan == g['plan'].tolist()
    model = CWMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']),
                              weight_constant_axis=axis, inline_permutation_aligner=al)
    assert model.weight.shape == g['weight'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.complex_watson.concentration, g['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(model.complex_watson.mode, g['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-5, atol=1e-8)
    if al is not None:
        with pytest.raises(AssertionError):  # needs frequency-tied weights, like the reference
            CWMMTrainer().fit(g['y'], initialization=g['init'], iterations=2, inline_permutation_aligner=al)


@pytest.mark.parametrize('F,T,D,K,I', [(9, 150, 6, 4, 6), (5, 64, 8, 3, 5), (4, 100, 3, 2, 5), (3, 90, 5, 3, 4)])
def test_fit_matches_oracle(F, T, D, K, I):
    from pb_bss_b200.distribution import CWMMTrainer
    y, _ = synth.structured_stft(F, T, D, K, seed=F * T)
    init = synth.init_affiliation(F, K, T, seed=K)
    ref = O.cwmm_fit(y, init, I)
    model = CWMMTrainer().fit(y, initialization=init, iterations=I)
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.complex_watson.concentration, ref['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(model.complex_watson.mode, ref['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(model.predict(y), O.cwmm_predict(y, ref), rtol=1e-5, atol=1e-8)


# the T at which the library splits one bin-iteration of the complex Watson fit into S = 1, 2, 4 parts
CW_SPLIT_T = {(6, 4): {1: 200, 2: 400, 4: 600}, (8, 3): {1: 150, 2: 300, 4: 515}, (4, 2): {1: 300, 2: 1200, 4: 2100}}


@pytest.mark.parametrize('S', [1, 2, 4])
@pytest.mark.parametrize('F,D,K,I', [(5, 6, 4, 6), (3, 8, 3, 5), (4, 4, 2, 5)])
def test_frame_split_matches_oracle(F, D, K, I, S):
    """One EM iteration of a bin split over the S CTAs the library picks (em_persistent.cuh, "frame split"): same
    model as the oracle, and deterministic."""
    from pb_bss_b200.distribution import CWMMTrainer
    T = CW_SPLIT_T[D, K][S]
    y, _ = synth.structured_stft(F, T, D, K, seed=F * T)
    init = synth.init_affiliation(F, K, T, seed=K)
    ref = O.cwmm_fit(y, init, I)
    model = CWMMTrainer().fit(y, initialization=init, iterations=I)
    assert last_plan() == (2, S, 3), (T, last_plan())
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.complex_watson.concentration, ref['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(model.complex_watson.mode, ref['mode']), 1, atol=1e-9)
    again = CWMMTrainer().fit(y, initialization=init, iterations=I)
    assert np.array_equal(model.complex_watson.mode, again.complex_watson.mode)


@pytest.mark.parametrize('D', [4, 6, 8])
def test_spline_table_reproduces_reference_inverse(D):
    """The device evaluates the B-spline the trainer exports; the exported
    table must be the reference's interpolant."""
    from pb_bss_b200.distribution import ComplexWatsonTrainer
    from scipy.interpolate import BSpline
    g = load_golden(f'cw_spline_d{D}')
    tr = ComplexWatsonTrainer(D)
    t, c = tr.spline_table
    lam = g['lam']
    inside = (lam >= t[0]) & (lam <= t[-1])
    np.testing.assert_allclose(BSpline(t, c, 2)(lam[inside]), g['kappa'][inside], rtol=1e-12)
    np.testing.assert_allclose(tr.hypergeometric_ratio_inverse(lam), g['kappa'], rtol=1e-12)


def test_tied_weights_with_saliency_match_reference_golden():
    from pb_bss_b200.distribution import CWMMTrainer
    g = load_golden('cwmm_tied_time_saliency')
    model = CWMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']),
                              weight_constant_axis=(-3,), saliency=g['saliency'])
    assert model.weight.shape == g['weight'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.complex_watson.concentration, g['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(model.complex_watson.mode, g['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-5, atol=1e-8)


def test_full_size_config4_properties():
    """BASELINE.json config 4 (F=257, T=1000, D=6, K=4, 50 iterations)."""
    from pb_bss_b200.distribution import CWMMTrainer
    F, T, D, K = 257, 1000, 6, 4
    y = synth.noise_stft(F, T, D, seed=4)
    init = synth.init_affiliation(F, K, T, seed=7)
    model = CWMMTrainer().fit(y, initialization=init, iterations=50)
    np.testing.assert_allclose(model.weight.sum(-2), 1, atol=1e-12)
    kap = model.complex_watson.concentration
    assert np.all(kap >= 0) and np.all(kap <= 500)
    aff = model.predict(y)
    np.testing.assert_allclose(aff.sum(-2), 1, atol=1e-12)
    sel = [0, 128, 256]
    ref = O.cwmm_fit(y[sel], init[sel], 50)
    np.testing.assert_allclose(model.weight[sel], ref['weight'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(aff[sel], O.cwmm_predict(y[sel], ref), atol=1e-5)


def test_num_classes_and_leading_dims():
    from pb_bss_b200.distribution import CWMMTrainer
    y = synth.noise_stft(6, 40, 4, seed=2).reshape(2, 3, 40, 4)
    np.random.seed(3)
    m = CWMMTrainer().fit(y, num_classes=2, iterations=3)
    assert m.weight.shape == (2, 3, 2, 1)
    assert m.complex_watson.mode.shape == (2, 3, 2, 4)
    assert m.complex_watson.concentration.shape == (2, 3, 2)
    np.random.seed(3)
    init = np.random.uniform(size=(2, 3, 2, 40))
    init /= np.einsum('...kn->...n', init)[..., None, :]
    ref = O.cwmm_fit(y, init, 3)
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-7)
    aff = CWMMTrainer().fit_predict(y, initialization=init, iterations=3)
    np.testing.assert_allclose(aff, O.cwmm_predict(y, ref), rtol=1e-6, atol=1e-9)
