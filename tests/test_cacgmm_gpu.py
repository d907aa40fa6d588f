"""Parity of the CUDA cACGMM path (through the Python API -> C ABI) against
the golden fixtures produced by the reference and against the oracle.

Tolerances (fp64 everywhere; only the summation order differs from NumPy):
single E/M steps rtol 1e-10; models after <= 10 EM iterations rtol 1e-6 /
atol 1e-9 (near-singular covariances amplify rounding through 1/lambda)."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import pb_bss_oracle as O
from oracle import synth
from test_em_kernels_gpu import device_fit, last_plan

pytestmark = pytest.mark.gpu

CASES = [
    'cacgmm_d4k2', 'cacgmm_d8k3', 'cacgmm_d8k3_structured',
    'cacgmm_opt_saliency', 'cacgmm_opt_mask', 'cacgmm_opt_trace',
    'cacgmm_opt_nonorm', 'cacgmm_opt_w2', 'cacgmm_opt_eps0',
    'cacgmm_opt_bcast',
]


def _kwargs(g):
    kw = {}
    for k, v in g.items():
        if not k.startswith('kw_'):
            continue
        name = k[3:]
        if name == 'covariance_norm':
            v = str(v) if v.dtype.kind in 'US' else False
        elif name == 'weight_constant_axis':
            v = int(v)
        elif name in ('affiliation_eps', 'eigenvalue_floor'):
            v = float(v)
        kw[name] = v
    return kw


def _cov(model):
    return model.cacg.covariance


@pytest.mark.parametrize('name', CASES)
def test_fit_matches_reference_golden(name):
    from pb_bss_b200.distribution import CACGMMTrainer
    g = load_golden(name)
    kw = _kwargs(g)
    model = CACGMMTrainer().fit(g['y'], initialization=g['init'],
                                iterations=int(g['iterations']), **kw)
    assert model.weight.shape == g['weight'].shape
    assert model.cacg.covariance_eigenvectors.shape == g['eigenvectors'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.cacg.covariance_eigenvalues, g['eigenvalues'], rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose(_cov(model), g['covariance'], rtol=1e-6, atol=1e-9)
    aff, q = model.predict(g['y'], return_quadratic_form=True,
                           source_activity_mask=kw.get('source_activity_mask'))
    np.testing.assert_allclose(aff, g['affiliation'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(q, g['quadratic_form'], rtol=1e-6)
    np.testing.assert_allclose(model.log_likelihood(g['y']), g['log_likelihood'], rtol=1e-8)
    # eigenvectors: unitary, and they reproduce the covariance with the eigenvalues
    V = model.cacg.covariance_eigenvectors
    eye = np.eye(V.shape[-1])
    np.testing.assert_allclose(np.einsum('...de,...df->...ef', V.conj(), V), np.broadcast_to(eye, V.shape), atol=1e-12)
    assert np.all(np.diff(model.cacg.covariance_eigenvalues, axis=-1) >= 0)


def test_warm_start_matches_reference():
    from pb_bss_b200.distribution import CACGMM, CACGMMTrainer
    from pb_bss_b200.distribution import ComplexAngularCentralGaussian as CACG
    g = load_golden('cacgmm_warm')
    m3 = CACGMM(weight=g['w3'], cacg=CACG(covariance_eigenvectors=g['V3'], covariance_eigenvalues=g['l3']))
    m5 = CACGMMTrainer().fit(g['y'], initialization=m3, iterations=2)
    np.testing.assert_allclose(m5.weight, g['w5'], rtol=1e-7)
    np.testing.assert_allclose(m5.cacg.covariance_eigenvalues, g['l5'], rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose(_cov(m5), g['cov5'], rtol=1e-6, atol=1e-9)
    # 3 + 2 iterations == 5 iterations in one go
    m5b = CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=5)
    np.testing.assert_allclose(_cov(m5b), g['cov5'], rtol=1e-6, atol=1e-9)


def test_single_e_and_m_step():
    from pb_bss_b200.distribution import CACGMM
    from pb_bss_b200.distribution import ComplexAngularCentralGaussian as CACG
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    g = load_golden('cacg_steps')
    model = CACGMM(weight=g['w'], cacg=CACG(covariance_eigenvectors=g['V'], covariance_eigenvalues=g['lam']))
    aff, q = model.predict(g['y'], return_quadratic_form=True)
    np.testing.assert_allclose(q, g['q'], rtol=1e-10)
    aff_ref = O.log_pdf_to_affiliation(g['w'], g['log_pdf'], None, 0.)
    np.testing.assert_allclose(aff, aff_ref, rtol=1e-9, atol=1e-300)
    m2 = cacgmm_m_step(g['y'], g['q'], g['aff'])
    np.testing.assert_allclose(m2.cacg.covariance_eigenvalues, g['fit_lam'], rtol=1e-9)
    np.testing.assert_allclose(m2.cacg.covariance, g['fit_cov'], rtol=1e-9, atol=1e-12)


def test_normalize_observation():
    from pb_bss_b200.distribution import normalize_observation
    y = synth.noise_stft(5, 77, 6, seed=3)
    y[2, 5] = 0  # zero vectors stay zero (utils.py:242-244)
    z = normalize_observation(y)
    np.testing.assert_allclose(z, O.normalize_observation_cacg(y), rtol=1e-15)
    assert np.all(z[2, :, 5] == 0)
    z32 = normalize_observation(y.astype(np.complex64))
    assert z32.dtype == np.complex64
    np.testing.assert_allclose(z32, O.normalize_observation_cacg(y), rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize('F,T,D,K,I', [
    (129, 200, 4, 2, 20),   # BASELINE.json config 1
    (7, 33, 8, 3, 5), (3, 31, 6, 4, 4), (2, 500, 8, 2, 6), (1, 7, 4, 3, 3),
    (4, 64, 3, 2, 5), (3, 130, 5, 5, 4), (2, 40, 2, 2, 6), (2, 50, 9, 3, 3),  # generic kernel
])
def test_fit_matches_oracle(F, T, D, K, I):
    from pb_bss_b200.distribution import CACGMMTrainer
    y, _ = synth.structured_stft(F, T, D, K, seed=F + T)
    init = synth.init_affiliation(F, K, T, seed=D)
    ref = O.cacgmm_fit(y, init, I)
    model = CACGMMTrainer().fit(y, initialization=init, iterations=I)
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), O.cacg_covariance_from_eig(ref['eigenvectors'], ref['eigenvalues']),
                               rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.predict(y), O.cacgmm_predict(y, ref), rtol=1e-6, atol=1e-9)


def test_leading_independent_dims_and_fit_predict():
    from pb_bss_b200.distribution import CACGMMTrainer
    y, _ = synth.structured_stft(6, 48, 4, 2, seed=4)
    init = synth.init_affiliation(6, 2, 48, seed=2)
    y4, init4 = y.reshape(2, 3, 48, 4), init.reshape(2, 3, 2, 48)
    m = CACGMMTrainer().fit(y4, initialization=init4, iterations=4)
    assert m.weight.shape == (2, 3, 2, 1)
    assert m.cacg.covariance_eigenvectors.shape == (2, 3, 2, 4, 4)
    ref = O.cacgmm_fit(y, init, 4)
    np.testing.assert_allclose(m.weight.reshape(6, 2, 1), ref['weight'], rtol=1e-7)
    aff = CACGMMTrainer().fit_predict(y4, initialization=init4, iterations=4)
    assert aff.shape == (2, 3, 2, 48)
    np.testing.assert_allclose(aff.reshape(6, 2, 48), O.cacgmm_predict(y, ref), rtol=1e-6, atol=1e-9)


def test_num_classes_uses_global_numpy_rng():
    """fit(num_classes=K) draws its init like cacgmm.py:206-209."""
    from pb_bss_b200.distribution import CACGMMTrainer
    y = synth.noise_stft(3, 40, 4, seed=1)
    np.random.seed(5)
    m = CACGMMTrainer().fit(y, num_classes=2, iterations=3)
    np.random.seed(5)
    init = np.random.uniform(size=(3, 2, 40))
    init /= np.einsum('...kn->...n', init)[..., None, :]
    ref = O.cacgmm_fit(y, init, 3)
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-8)


def test_complex64_storage():
    """complex64 observations are stored as float2 and accumulated in fp64."""
    from pb_bss_b200.distribution import CACGMMTrainer
    y, _ = synth.structured_stft(5, 120, 8, 3, seed=9)
    init = synth.init_affiliation(5, 3, 120, seed=1)
    y32 = y.astype(np.complex64)
    ref = O.cacgmm_fit(y32.astype(np.complex128), init, 6)
    m = CACGMMTrainer().fit(y32, initialization=init, iterations=6)
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(m.predict(y32), O.cacgmm_predict(y32.astype(np.complex128), ref), atol=1e-3)


def test_device_tensors_stay_on_device_and_are_deterministic():
    import torch
    from pb_bss_b200.distribution import CACGMMTrainer
    y = torch.from_numpy(synth.noise_stft(9, 100, 8, seed=2)).cuda()
    init = torch.from_numpy(synth.init_affiliation(9, 3, 100)).cuda()
    m1 = CACGMMTrainer().fit(y, initialization=init, iterations=5)
    m2 = CACGMMTrainer().fit(y, initialization=init, iterations=5)
    assert m1.weight.is_cuda and m1.cacg.covariance_eigenvectors.is_cuda
    assert torch.equal(m1.weight, m2.weight)
    assert torch.equal(m1.cacg.covariance_eigenvalues, m2.cacg.covariance_eigenvalues)
    aff = m1.predict(y)
    assert aff.is_cuda and aff.shape == (9, 3, 100)
    torch.testing.assert_close(aff.sum(-2), torch.ones_like(aff[:, 0]), rtol=0, atol=1e-12)


def test_full_size_properties():
    """BASELINE.json config 2 (F=513, T=500, D=8, K=3, 100 iterations):
    size-independent properties instead of an oracle run."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, D, K = 513, 500, 8, 3
    y = synth.noise_stft(F, T, D, seed=0)
    init = synth.init_affiliation(F, K, T, seed=7)
    tr = CACGMMTrainer()
    m2 = tr.fit(y, initialization=init, iterations=2)
    m3 = tr.fit(y, initialization=m2, iterations=1)
    m100 = tr.fit(y, initialization=init, iterations=100)
    ll2, ll3, ll100 = m2.log_likelihood(y), m3.log_likelihood(y), m100.log_likelihood(y)
    assert ll3 > ll2 and ll100 > ll3, (ll2, ll3, ll100)  # cacgmm.py:100-107 doctest
    np.testing.assert_allclose(m100.weight.sum(-2), 1, atol=1e-12)
    lam = m100.cacg.covariance_eigenvalues
    np.testing.assert_allclose(lam[..., -1], 1, rtol=1e-14)
    assert np.all(lam >= 1e-10) and np.all(np.diff(lam, axis=-1) >= 0)
    aff = m100.predict(y)
    np.testing.assert_allclose(aff.sum(-2), 1, atol=1e-12)
    # spot-check 3 bins of the 100-iteration model against the oracle
    sel = [0, 256, 512]
    ref = O.cacgmm_fit(y[sel], init[sel], 100)
    np.testing.assert_allclose(m100.weight[sel], ref['weight'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(aff[sel], O.cacgmm_predict(y[sel], ref), atol=1e-5)


@pytest.mark.parametrize('D,K', [(8, 3), (6, 4), (4, 2)])
def test_persistent_and_multi_kernel_paths_agree(D, K):
    """The persistent kernel (Gauss-Jordan update on intermediate iterations)
    and the kernel-pair-per-iteration path (Jacobi every iteration) must agree."""
    from pb_bss_b200.distribution import CACGMMTrainer
    y, _ = synth.structured_stft(40, 300, D, K, seed=3)
    init = synth.init_affiliation(40, K, 300, seed=5)
    a = CACGMMTrainer().fit(y, initialization=init, iterations=15)
    b = CACGMMTrainer().fit(y, initialization=init, iterations=15, multi_kernel=True)
    np.testing.assert_allclose(a.weight, b.weight, rtol=1e-8, atol=1e-11)
    np.testing.assert_allclose(_cov(a), _cov(b), rtol=1e-7, atol=1e-10)


def test_rank_deficient_observation_takes_the_floor_path():
    """Observations confined to a 2-dim subspace: the scatter matrices are
    singular, every update must take the eigendecomposition + floor path."""
    from pb_bss_b200.distribution import CACGMMTrainer
    rng = np.random.RandomState(0)
    F, T, D, K = 6, 96, 8, 2
    basis = rng.randn(F, 2, D) + 1j * rng.randn(F, 2, D)
    coeff = rng.randn(F, T, 2) + 1j * rng.randn(F, T, 2)
    y = np.einsum('ftr,frd->ftd', coeff, basis)
    init = synth.init_affiliation(F, K, T, seed=2)
    ref = O.cacgmm_fit(y, init, 4)
    m = CACGMMTrainer().fit(y, initialization=init, iterations=4)
    np.testing.assert_allclose(m.cacg.covariance_eigenvalues[..., :6], 1e-10, rtol=1e-6)
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(m.predict(y), O.cacgmm_predict(y, ref), atol=1e-4)


@pytest.mark.parametrize('D,K', [(8, 3), (4, 2), (6, 4)])
@pytest.mark.parametrize('variant', ['saliency', 'mask', 'trace', 'nonorm', 'w2', 'eps0', 'warm', 'floor0'])
def test_persistent_full_variant_options(D, K, variant):
    """Options on the template shapes (D in {4,6,8}) run through the FULL variant of the
    persistent kernel (saliency / activity mask / log-domain softmax / user model)."""
    from pb_bss_b200.distribution import CACGMM, CACGMMTrainer
    from pb_bss_b200.distribution import ComplexAngularCentralGaussian as CACG
    F, T, I = 5, 200, 6
    y, _ = synth.structured_stft(F, T, D, K, seed=D * K)
    init = synth.init_affiliation(F, K, T, seed=1)
    rng = np.random.RandomState(D)
    kw = {}
    if variant == 'saliency':
        kw['saliency'] = rng.uniform(0.1, 1.0, size=(F, T))
    elif variant == 'mask':
        sam = rng.uniform(size=(F, K, T)) > 0.25
        sam[:, 0, :] |= ~sam.any(axis=1)
        kw['source_activity_mask'] = sam
    elif variant == 'trace':
        kw['covariance_norm'] = 'trace'
    elif variant == 'nonorm':
        kw['covariance_norm'] = False
    elif variant == 'w2':
        kw['weight_constant_axis'] = -2
    elif variant == 'eps0':
        kw.update(affiliation_eps=0., eigenvalue_floor=1e-6)
    elif variant == 'floor0':
        kw.update(eigenvalue_floor=0.)
    if variant == 'warm':
        m0 = O.cacgmm_fit(y, init, 2)
        ref = O.cacgmm_fit(y, m0, I)
        start = CACGMM(weight=m0['weight'], cacg=CACG(covariance_eigenvectors=m0['eigenvectors'],
                                                       covariance_eigenvalues=m0['eigenvalues']))
        model = CACGMMTrainer().fit(y, initialization=start, iterations=I)
    else:
        ref = O.cacgmm_fit(y, init, I, **kw)
        model = CACGMMTrainer().fit(y, initialization=init, iterations=I, **kw)
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.cacg.covariance_eigenvalues, ref['eigenvalues'], rtol=1e-5, atol=1e-11)
    np.testing.assert_allclose(_cov(model), O.cacg_covariance_from_eig(ref['eigenvectors'], ref['eigenvalues']),
                               rtol=1e-5, atol=1e-9)


def test_zero_observation_frames():
    """All-zero STFT frames (digital silence): the reference floors their quadratic form at
    `tiny` (cacg.py:198), i.e. every class sees the same q; they still count in the weights."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, D, K, I = 6, 160, 8, 3, 6
    y, _ = synth.structured_stft(F, T, D, K, seed=31)
    y[:, 10:14] = 0
    y[2, 100:131] = 0
    init = synth.init_affiliation(F, K, T, seed=2)
    ref = O.cacgmm_fit(y, init, I)
    model = CACGMMTrainer().fit(y, initialization=init, iterations=I)
    np.testing.assert_allclose(model.weight, ref['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), O.cacg_covariance_from_eig(ref['eigenvectors'], ref['eigenvalues']),
                               rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(model.predict(y), O.cacgmm_predict(y, ref), rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('name,axis', [('cacgmm_tied_time', (-3,)), ('cacgmm_tied', (-3, -1))])
def test_frequency_tied_weights_match_reference_golden(name, axis):
    """weight_constant_axis (-3,) / (-3, -1): one weight per (class, frame) / per class shared by
    all bins (mixture_model_utils.py:187-190) -- couples the bins in every iteration."""
    from pb_bss_b200.distribution import CACGMMTrainer
    g = load_golden(name)
    model = CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']),
                                weight_constant_axis=axis)
    assert model.weight.shape == g['weight'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), g['covariance'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('name,axis', [('cacgmm_tied_time_saliency', (-3,)), ('cacgmm_tied_saliency', (-3, -1))])
def test_tied_weights_with_saliency_match_reference_golden(name, axis):
    """estimate_mixture_weight with a saliency (mixture_model_utils.py:192-203) and frequency-tied weights."""
    from pb_bss_b200.distribution import CACGMMTrainer
    g = load_golden(name)
    model = CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']),
                                weight_constant_axis=axis, saliency=g['kw_saliency'])
    assert model.weight.shape == g['weight'].shape
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), g['covariance'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-6, atol=1e-9)


def test_tied_weights_with_a_batch_dim_match_reference_golden():
    """(B, F, T, D) with weight_constant_axis=(-3,): the weights are tied over the bins of every batch element
    separately (mean over axis -3, keepdims), the reference's shape (B, 1, K, T)."""
    from pb_bss_b200.distribution import CACGMMTrainer
    g = load_golden('cacgmm_tied_batch')
    model = CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=int(g['iterations']),
                                weight_constant_axis=(-3,))
    assert model.weight.shape == g['weight'].shape, (model.weight.shape, g['weight'].shape)
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), g['covariance'], rtol=1e-6, atol=1e-9)


def test_inline_permutation_alignment_matches_reference_golden():
    """inline_permutation_aligner (cacgmm.py:260-267, mixture_model_utils.py:264-306)."""
    from pb_bss_b200.distribution import CACGMMTrainer
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    g = load_golden('cacgmm_inline_pa')
    al = DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                  main_iterations=5, sub_iterations=2)
    assert al.alignment_plan == g['plan'].tolist()
    model = CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=5, weight_constant_axis=(-3,),
                                inline_permutation_aligner=al)
    np.testing.assert_allclose(model.weight, g['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(_cov(model), g['covariance'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.predict(g['y']), g['affiliation'], rtol=1e-6, atol=1e-9)
    with pytest.raises(AssertionError):  # needs frequency-tied weights, like the reference
        CACGMMTrainer().fit(g['y'], initialization=g['init'], iterations=2, inline_permutation_aligner=al)


@pytest.mark.parametrize('shape', [(129, 200, 4, 2, 20), (40, 333, 8, 3, 12), (7, 130, 6, 4, 5), (3, 50, 8, 2, 3),
                                   (65, 257, 8, 4, 1)])
@pytest.mark.parametrize('cdtype', ['complex128', 'complex64'])
def test_pinned_host_inputs_match_device_inputs(shape, cdtype):
    """y / initialization in pinned host memory are read in place over PCIe by a loader kernel that
    overlaps the EM kernel (wave task order).  Every task computes exactly what it computes with
    device-resident inputs, so the models must be bit-identical."""
    import torch
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, D, K, iters = shape
    y, _ = synth.structured_stft(F, T, D, K, seed=3)
    y[2, 5] = 0  # an all-zero frame: that bin takes the reference-normalisation path
    y = y.astype(cdtype)
    init = synth.init_affiliation(F, K, T, seed=7)
    y_pin, init_pin = torch.from_numpy(y).pin_memory(), torch.from_numpy(init).pin_memory()
    ref = CACGMMTrainer().fit(y_pin.cuda(), initialization=init_pin.cuda(), iterations=iters)
    got = CACGMMTrainer().fit(y_pin, initialization=init_pin, iterations=iters)
    # pinned observation in -> the model is written to pinned host memory as well
    assert not got.weight.is_cuda and got.weight.is_pinned()
    assert torch.equal(got.weight, ref.weight.cpu())
    assert torch.equal(got.cacg.covariance_eigenvalues, ref.cacg.covariance_eigenvalues.cpu())
    assert torch.equal(got.cacg.covariance_eigenvectors, ref.cacg.covariance_eigenvectors.cpu())
    # pinned observation, device initialisation; and a warm start from pinned memory
    got = CACGMMTrainer().fit(y_pin, initialization=init_pin.cuda(), iterations=iters)
    assert torch.equal(got.cacg.covariance_eigenvalues, ref.cacg.covariance_eigenvalues.cpu())
    warm_dev = CACGMMTrainer().fit(y_pin.cuda(), initialization=ref, iterations=2)
    warm_pin = CACGMMTrainer().fit(y_pin, initialization=ref, iterations=2)
    assert torch.equal(warm_pin.cacg.covariance_eigenvalues.cpu(), warm_dev.cacg.covariance_eigenvalues.cpu())
    # the model fitted from pinned memory predicts like any other
    np.testing.assert_array_equal(got.predict(y_pin.cuda()).cpu().numpy(), ref.predict(y_pin.cuda()).cpu().numpy())


def _check_fit(m, ref):
    cov_ref = np.einsum('...de,...e,...fe->...df', ref['eigenvectors'], ref['eigenvalues'], ref['eigenvectors'].conj())
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=0, atol=1e-9)
    np.testing.assert_allclose(m.cacg.covariance, cov_ref, rtol=0, atol=1e-8)


def _same_model(a, b):
    return (np.array_equal(a.cacg.covariance_eigenvectors, b.cacg.covariance_eigenvectors)
            and np.array_equal(a.cacg.covariance_eigenvalues, b.cacg.covariance_eigenvalues)
            and np.array_equal(a.weight, b.weight))


# D = 8, lean: (F, T, K, I, pinned host input) for which em_ws_kernel runs with the frame split S
WS_SPLIT_CASES = {
    1: [(300, 200, 3, 6, False), (300, 129, 2, 4, False), (2, 129, 3, 4, True)],
    2: [(9, 290, 2, 7, True), (5, 350, 3, 12, True)],
    4: [(5, 500, 3, 12, True), (3, 1100, 4, 5, True), (1, 512, 3, 6, True)],
}


@pytest.mark.parametrize('S', [1, 2, 4])
def test_ws_kernel_frame_split_picked_by_the_library(S):
    """em_ws_kernel: one EM iteration of a bin is split over the S CTAs the library picks, by ring stage (em_ws.cuh,
    "frame split").  S = 1 runs device-resident input with more bins than sticky-bins clusters fit, and pinned host
    input with a short sweep; S = 2 and 4 run pinned host input with few bins (the streamed upload never runs the
    sticky-bins kernel).  Whatever S, the result matches the oracle; and it is deterministic (partial sums added in
    part order)."""
    for F, T, K, I, pinned in WS_SPLIT_CASES[S]:
        y, _ = synth.structured_stft(F, T, 8, K, seed=11)
        init = synth.init_affiliation(F, K, T, seed=5)
        m = device_fit(y, init, I, pinned=pinned)
        assert last_plan() == (0, S, 0), (F, T, last_plan())
        _check_fit(m, O.cacgmm_fit(y, init, I))
        assert _same_model(m, device_fit(y, init, I, pinned=pinned))


# the single-role kernel (em_persistent_kernel) at F = 4: the T at which the library splits a bin-iteration into
# S = 1, 2, 4 parts (the sweep T D^2 (K + 1) must pay for each part, choose_frame_split)
SINGLE_ROLE_T = {(6, 4): {1: 200, 2: 385, 4: 600}, (4, 2): {1: 530, 2: 1500, 4: 2100},
                 (4, 3): {1: 530, 2: 1000, 4: 1600}, (8, 3): {1: 150, 2: 300, 4: 530}}


@pytest.mark.parametrize('S', [1, 2, 4])
@pytest.mark.parametrize('D,K,variant', [(6, 4, 'lean'), (4, 2, 'lean'), (4, 3, 'lean'), (6, 4, 'saliency'),
                                         (4, 2, 'saliency'), (4, 3, 'saliency'), (8, 3, 'saliency')])
def test_frame_split_on_the_single_role_kernel(S, D, K, variant):
    """Frame split in em_persistent_kernel (lean D = 4 / 6, and the full variant with saliency at any D), at each split
    the library picks."""
    F, I = 4, 6
    T = SINGLE_ROLE_T[D, K][S]
    y, _ = synth.structured_stft(F, T, D, K, seed=21)
    init = synth.init_affiliation(F, K, T, seed=3)
    sal = None
    if variant == 'saliency':
        sal = np.random.default_rng(4).uniform(0.2, 1.0, size=(F, T))
    m = device_fit(y, init, I, saliency=sal)
    assert last_plan() == (2, S, 0 if sal is None else 1), (T, last_plan())
    _check_fit(m, O.cacgmm_fit(y, init, I, saliency=sal))
    assert _same_model(m, device_fit(y, init, I, saliency=sal))


def test_time_varying_weight_needs_matching_frame_count():
    """weight_constant_axis=(-3,) gives a weight per frame; predicting an observation with another number of frames
    fails in the reference (broadcast error) and must not read past the weight buffer here."""
    from pb_bss_b200.distribution import CACGMMTrainer
    y, _ = synth.structured_stft(6, 80, 4, 2, seed=2)
    m = CACGMMTrainer().fit(y, initialization=synth.init_affiliation(6, 2, 80, seed=1), iterations=3,
                            weight_constant_axis=(-3,))
    assert m.predict(y).shape == (6, 2, 80)
    y2, _ = synth.structured_stft(6, 96, 4, 2, seed=2)
    with pytest.raises(ValueError, match='frames'):
        m.predict(y2)


# D = 8, lean, few bins: (F, T, K, I) for which device-resident input runs em_sticky_kernel with clusters of S CTAs
STICKY_CASES = {
    1: [(5, 100, 3, 12), (3, 128, 2, 6), (7, 97, 4, 5)],
    2: [(5, 350, 3, 12), (3, 256, 2, 6), (7, 300, 4, 5), (2, 383, 3, 1)],
    4: [(5, 500, 3, 12), (3, 512, 2, 6), (7, 1000, 4, 5), (2, 1100, 3, 1)],
}


@pytest.mark.parametrize('S', [1, 2, 4])
def test_sticky_bins_kernel_matches_the_task_kernel_bit_for_bit(S):
    """em_sticky_kernel (one cluster of S CTAs per bin for the whole fit, few bins) sums the parts in the same order
    as em_ws_kernel with the frame split S, which the same fit from pinned host memory runs: identical models; and
    both match the oracle."""
    for F, T, K, I in STICKY_CASES[S]:
        y, _ = synth.structured_stft(F, T, 8, K, seed=31)
        init = synth.init_affiliation(F, K, T, seed=9)
        m = device_fit(y, init, I)
        assert last_plan() == (1, S, 0), (F, T, last_plan())
        mt = device_fit(y, init, I, pinned=True)
        assert last_plan() == (0, S, 0), (F, T, last_plan())
        assert _same_model(m, mt)
        _check_fit(m, O.cacgmm_fit(y, init, I))


def test_argument_errors():
    from pb_bss_b200.distribution import CACGMMTrainer
    y = synth.noise_stft(2, 20, 4)
    with pytest.raises(AssertionError):
        CACGMMTrainer().fit(y)  # neither initialization nor num_classes
    with pytest.raises(AssertionError):
        CACGMMTrainer().fit(y.real, num_classes=2)
    with pytest.raises(TypeError):
        CACGMMTrainer().fit(y, initialization='nope')
    with pytest.raises(AssertionError):
        CACGMMTrainer().fit(y, num_classes=2, iterations=0)
    with pytest.raises(NotImplementedError):
        CACGMMTrainer().fit(y.reshape(1, 2, 20, 4), num_classes=2, weight_constant_axis=(-4,))


def test_nonfinite_input_raises():
    from pb_bss_b200.distribution import CACGMMTrainer
    y = synth.noise_stft(3, 40, 4)
    y[1, 3, 2] = np.nan
    with pytest.raises(AssertionError):
        CACGMMTrainer().fit(y, num_classes=2, iterations=2)


def test_heig_batched():
    from pb_bss_b200.extraction.linalg import eigh
    for D in (2, 3, 6, 8, 13):
        a = synth.pos_def_hermitian(50, D, D, seed=D)
        a[3] = np.eye(D)          # degenerate spectrum
        a[4] = np.diag(np.arange(D, 0, -1.0))  # needs sorting
        w, v = eigh(a)
        w0 = np.linalg.eigvalsh(a)
        np.testing.assert_allclose(w, w0, rtol=1e-12, atol=1e-14)
        rec = np.einsum('nde,ne,nfe->ndf', v, w, v.conj())
        np.testing.assert_allclose(rec, a, rtol=1e-12, atol=1e-13)
