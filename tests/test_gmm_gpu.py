"""GMM / Gaussian and VMFMM / von Mises-Fisher over embeddings on the device: parity with the reference's fixtures
(oracle/make_golden_embedding.py), the reference's own unit tests (tests/test_distribution/test_gmm.py,
test_gaussian.py, test_vmfmm.py) with a fixed seed, error paths, reproducibility and I/O types."""
import itertools

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_embedding_oracle import GMM_CASES, VMF_CASES, resolve

pytestmark = pytest.mark.gpu

MODEL = dict(rtol=1e-7, atol=1e-10)
AFF = dict(rtol=1e-6, atol=1e-9)


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')


@pytest.mark.parametrize('name', list(GMM_CASES))
def test_gmm_fixture_parity(name):
    from pb_bss_b200.distribution import GMMTrainer
    g = load_golden('gmm')
    y, init, kw = GMM_CASES[name]
    model = GMMTrainer().fit(g[y], initialization=g[init], iterations=int(g['iterations']), **resolve(g, kw))
    np.testing.assert_allclose(np.asarray(model.weight), g[f'{name}_weight'], **MODEL)
    np.testing.assert_allclose(model.gaussian.mean, g[f'{name}_mean'], **MODEL)
    np.testing.assert_allclose(model.gaussian.covariance, g[f'{name}_covariance'], **MODEL)
    np.testing.assert_allclose(model.predict(g[y]), g[f'{name}_affiliation'], **AFF)


def test_gmm_fit_predict_default_weight_axis():
    """fit_predict defaults to weight_constant_axis=(-2,) (a (..., 1, N) weight of ones)."""
    from pb_bss_b200.distribution import GMMTrainer
    g = load_golden('gmm')
    sal = np.broadcast_to(g['saliency'], g['yb'].shape[:-1]).copy()
    aff = GMMTrainer().fit_predict(g['yb'], initialization=g['initb'], iterations=int(g['iterations']), saliency=sal)
    np.testing.assert_allclose(aff, g['w_t2_sal_affiliation'], **AFF)


def test_gaussian_log_pdf_and_trainer_parity():
    from pb_bss_b200.distribution import Gaussian, GaussianTrainer
    g = load_golden('gmm')
    model = Gaussian(mean=g['full_b3_mean'], covariance=g['full_b3_covariance'])
    np.testing.assert_allclose(model.log_pdf(g['logpdf_y']), g['logpdf'], rtol=1e-10)
    sal = np.broadcast_to(g['saliency'], g['yb'].shape[:-1]).copy()
    for ct in ('full', 'diagonal', 'spherical'):
        fit = GaussianTrainer().fit(g['yb'], saliency=sal, covariance_type=ct)
        np.testing.assert_allclose(fit.mean, g[f'fit_{ct}_mean'], rtol=1e-10)
        np.testing.assert_allclose(fit.covariance, g[f'fit_{ct}_covariance'], rtol=1e-10)
    fit = GaussianTrainer().fit(g['y0'])
    np.testing.assert_allclose(fit.mean, g['fit_nosal_mean'], rtol=1e-10)
    np.testing.assert_allclose(fit.covariance, g['fit_nosal_covariance'], rtol=1e-10)


@pytest.mark.parametrize('name', list(VMF_CASES))
def test_vmfmm_fixture_parity(name):
    from pb_bss_b200.distribution import VMFMMTrainer
    g = load_golden('vmfmm')
    y, init, kw = VMF_CASES[name]
    model = VMFMMTrainer().fit(g[y], initialization=g[init], iterations=int(g['iterations']), **resolve(g, kw))
    np.testing.assert_allclose(np.asarray(model.weight), g[f'{name}_weight'], **MODEL)
    np.testing.assert_allclose(model.vmf.mean, g[f'{name}_mean'], **MODEL)
    np.testing.assert_allclose(model.vmf.concentration, g[f'{name}_concentration'], **MODEL)
    np.testing.assert_allclose(model.predict(g[y]), g[f'{name}_affiliation'], **AFF)


def test_vmf_trainer_parity():
    from pb_bss_b200.distribution import VonMisesFisherTrainer
    g = load_golden('vmfmm')
    yb = load_golden('gmm')['yb']
    fit = VonMisesFisherTrainer().fit(yb, saliency=np.broadcast_to(g['saliency'], yb.shape[:-1]).copy())
    np.testing.assert_allclose(fit.mean, g['fit_mean'], rtol=1e-10)
    np.testing.assert_allclose(fit.concentration, g['fit_concentration'], rtol=1e-10)


# ---- the reference's unit tests, fixed seed ----

def _two_clouds(rng, samples=1000):
    weight = np.array([0.3, 0.7])
    labels = rng.choice(range(2), size=(samples,), p=weight)
    mean = np.array([[-1, -1], [1, 1]])
    covariance = np.tile(0.25 * np.eye(2), (2, 1, 1))
    x = np.zeros((samples, 2))
    for k in range(2):
        x[labels == k, :] = rng.multivariate_normal(mean[k], covariance[0], size=(np.sum(labels == k),))
    return x, mean, covariance


def _best(model_mean, mean):
    return min(itertools.permutations(range(2)), key=lambda p: np.sum((model_mean[p, :] - mean) ** 2))


def test_reference_gmm():
    from pb_bss_b200.distribution import GMMTrainer
    np.random.seed(0)
    x, mean, covariance = _two_clouds(np.random)
    model = GMMTrainer().fit(x, num_classes=2)
    p = list(_best(model.gaussian.mean, mean))
    np.testing.assert_allclose(model.gaussian.mean[p, :], mean, atol=0.2)
    np.testing.assert_allclose(model.gaussian.covariance[p, :], covariance, atol=0.2)


def test_reference_gmm_independent_dimension():
    from pb_bss_b200.distribution import GMMTrainer
    np.random.seed(1)
    x, mean, covariance = _two_clouds(np.random)
    x = np.concatenate((x[None, ...], x[None, ...]), axis=0)
    model = GMMTrainer().fit(x, num_classes=2)
    p = list(_best(model.gaussian.mean[0], mean))
    np.testing.assert_allclose(model.gaussian.mean[0, p, :], mean, atol=0.2)
    np.testing.assert_allclose(model.gaussian.covariance[0, p, :], covariance, atol=0.2)


@pytest.mark.parametrize('covariance_type', ['full', 'diagonal', 'spherical'])
def test_reference_gaussian(covariance_type):
    from pb_bss_b200.distribution import GaussianTrainer
    np.random.seed(2)
    mean, covariance = np.ones((3,)), 2 * np.eye(3)
    x = np.random.multivariate_normal(mean, covariance, size=(10000,))
    model = GaussianTrainer().fit(x, covariance_type=covariance_type)
    np.testing.assert_allclose(model.mean, mean, atol=0.1)
    expected = {'full': covariance, 'diagonal': np.diag(covariance),
                'spherical': np.mean(np.diag(covariance))}[covariance_type]
    np.testing.assert_allclose(model.covariance, expected, atol=0.1)


def test_reference_vmfmm_shapes():
    from pb_bss_b200.distribution import VMFMMTrainer
    np.random.seed(3)
    x, mean, _ = _two_clouds(np.random)
    model = VMFMMTrainer().fit(x, num_classes=2)
    assert model.vmf.mean.shape == mean.shape
    assert model.vmf.concentration.shape == (2,)


def test_random_initialisation_follows_the_global_stream():
    """num_classes draws np.random.uniform((..., K, N)) exactly like the reference: the same fit as with that draw."""
    from pb_bss_b200.distribution import GMMTrainer
    g = load_golden('gmm')
    np.random.seed(5)
    a = GMMTrainer().fit(g['yb'], num_classes=3, iterations=3)
    np.random.seed(5)
    init = np.random.uniform(size=(3, 3, g['yb'].shape[1]))
    init /= init.sum(-2, keepdims=True)
    b = GMMTrainer().fit(g['yb'], initialization=init, iterations=3)
    np.testing.assert_array_equal(a.gaussian.mean, b.gaussian.mean)


# ---- error paths ----

def test_error_paths():
    from pb_bss_b200.distribution import GMMTrainer, VMFMMTrainer
    g = load_golden('gmm')
    y, init = g['y0'], g['init0']
    with pytest.raises(AssertionError):
        GMMTrainer().fit(y, initialization=init, num_classes=3)
    with pytest.raises(AssertionError):
        GMMTrainer().fit(y)
    with pytest.raises(AssertionError):
        VMFMMTrainer().fit(y, initialization=init, num_classes=3)
    with pytest.raises(AssertionError):
        GMMTrainer().fit(y.astype(np.complex128), initialization=init)
    with pytest.raises(AssertionError):
        VMFMMTrainer().fit(y.astype(np.complex128), initialization=init)
    # a singular fixed covariance
    with pytest.raises(ValueError, match='ill-defined empirical covariance'):
        GMMTrainer().fit(y, initialization=init, iterations=2, fixed_covariance=np.zeros((3, 5, 5)))
    # a collapsed class: every observation the same
    with pytest.raises(ValueError, match='ill-defined empirical covariance'):
        GMMTrainer().fit(np.ones((50, 4)), initialization=np.full((2, 50), 0.5), iterations=2)
    for ct in ('diagonal', 'spherical'):
        with pytest.raises(ValueError):
            GMMTrainer().fit(g['yb'][:2], initialization=g['initb'][:2], iterations=2, covariance_type=ct)
    with pytest.raises(ValueError):
        GMMTrainer().fit(np.random.RandomState(0).randn(40, 65), num_classes=2, iterations=1)
    with pytest.raises(NotImplementedError):
        GMMTrainer().fit(y, num_classes=7, iterations=1)
    with pytest.raises(NotImplementedError):
        GMMTrainer().fit(y, initialization=init, iterations=1, weight_constant_axis=(-3,))
    with pytest.raises(NotImplementedError):
        VMFMMTrainer().fit(y, num_classes=7, iterations=1)
    with pytest.raises(ValueError):
        GMMTrainer().fit(y, initialization=init, iterations=1, covariance_type='banana')


# ---- reproducibility and I/O types ----

def test_bit_reproducible():
    from pb_bss_b200.distribution import GMMTrainer, VMFMMTrainer
    rng = np.random.RandomState(7)
    y = rng.randn(4, 3000, 20)
    init = rng.uniform(size=(4, 4, 3000))
    init /= init.sum(-2, keepdims=True)
    a = GMMTrainer().fit(y, initialization=init, iterations=4)
    b = GMMTrainer().fit(y, initialization=init, iterations=4)
    np.testing.assert_array_equal(a.gaussian.covariance, b.gaussian.covariance)
    np.testing.assert_array_equal(a.predict(y), b.predict(y))
    a = VMFMMTrainer().fit(y, initialization=init, iterations=4)
    b = VMFMMTrainer().fit(y, initialization=init, iterations=4)
    np.testing.assert_array_equal(a.vmf.mean, b.vmf.mean)
    np.testing.assert_array_equal(a.predict(y), b.predict(y))


def test_io_types():
    from pb_bss_b200.distribution import GMMTrainer, VMFMMTrainer
    g = load_golden('gmm')
    y, init = g['yb'], g['initb']
    model = GMMTrainer().fit(y, initialization=init, iterations=3)
    assert isinstance(model.gaussian.mean, np.ndarray) and isinstance(model.weight, np.ndarray)
    assert isinstance(model.predict(y), np.ndarray)
    yt, it = torch.from_numpy(y).cuda(), torch.from_numpy(init).cuda()
    tmodel = GMMTrainer().fit(yt, initialization=it, iterations=3)
    assert torch.is_tensor(tmodel.gaussian.mean) and tmodel.gaussian.mean.is_cuda
    assert torch.is_tensor(tmodel.weight) and tmodel.weight.is_cuda
    aff = tmodel.predict(yt)
    assert torch.is_tensor(aff) and aff.is_cuda
    np.testing.assert_array_equal(aff.cpu().numpy(), model.predict(y))
    aff = GMMTrainer().fit_predict(yt, initialization=it, iterations=3)
    assert torch.is_tensor(aff) and aff.is_cuda
    vmodel = VMFMMTrainer().fit(yt, initialization=it, iterations=3)
    assert torch.is_tensor(vmodel.vmf.mean) and vmodel.vmf.mean.is_cuda
    aff = vmodel.predict(yt)
    assert torch.is_tensor(aff) and aff.is_cuda
    assert isinstance(VMFMMTrainer().fit_predict(y, initialization=init, iterations=3), np.ndarray)
