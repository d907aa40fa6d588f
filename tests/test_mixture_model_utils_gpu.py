"""The EM plumbing shared by the cACGMM, CWMM and CBMM trainers (pb_bss_b200/distribution/mixture_model_utils.py):
frequency-tied weights with a batch dim, the predict-side weight checks, and the dataclass walks that move models to
NumPy and stack them."""
import numpy as np
import pytest

from oracle import synth

TRAINERS = ['CACGMMTrainer', 'CWMMTrainer', 'CBMMTrainer']


def _trainer(name):
    from pb_bss_b200 import distribution
    return getattr(distribution, name)()


def _leaves(model):
    """{dotted field name: value} of a model and its sub-models."""
    out = {}
    for k, v in model.to_dict().items():
        if isinstance(v, dict):
            out.update({f'{k}.{kk}': vv for kk, vv in v.items()})
        else:
            out[k] = v
    return out


def test_weight_axis_mapping():
    from pb_bss_b200 import _lib
    from pb_bss_b200.distribution.mixture_model_utils import weight_mode as _weight_mode
    assert _weight_mode((-1,), 3) == _lib.WEIGHT_TIME
    assert _weight_mode([-1], 3) == _lib.WEIGHT_TIME
    assert _weight_mode(2, 3) == _lib.WEIGHT_TIME
    assert _weight_mode(-2, 3) == _lib.WEIGHT_CONST
    assert _weight_mode(1, 3) == _lib.WEIGHT_CONST
    assert _weight_mode((-3,), 3) == _lib.WEIGHT_TIED_TIME
    assert _weight_mode((-3, -1), 3) == _lib.WEIGHT_TIED
    assert _weight_mode((-1, -3), 3) == _lib.WEIGHT_TIED
    # more than one independent dim: the bins (axis -3) are tied, the dims in front stay independent fits
    assert _weight_mode((-3,), 4) == _lib.WEIGHT_TIED_TIME
    assert _weight_mode((-3, -1), 5) == _lib.WEIGHT_TIED
    with pytest.raises(NotImplementedError):
        _weight_mode((-4, -1), 4)


@pytest.mark.gpu
@pytest.mark.parametrize('with_saliency', [False, True])
@pytest.mark.parametrize('axis', [(-3,), (-3, -1)])
@pytest.mark.parametrize('name', TRAINERS)
def test_tied_weights_with_a_batch_dim_are_one_fit_per_leading_index(name, axis, with_saliency):
    """y (B, F, T, D) with weight_constant_axis (-3,) / (-3, -1): the weights are tied over the bins of each batch
    element (the reference's mean over axis -3 keeps the batch apart), so the fit is the B single fits stacked, bit for
    bit, and the weight has the reference's shape (B, 1, K, T) / (B, 1, K, 1)."""
    B, F, T, D, K = 2, 5, 64, 4, 2
    ys = [synth.structured_stft(F, T, D, K, seed=3 + b)[0] for b in range(B)]
    inits = [synth.init_affiliation(F, K, T, seed=11 + b) for b in range(B)]
    sals = [np.random.default_rng(b).uniform(0.2, 1.0, size=(F, T)) if with_saliency else None for b in range(B)]
    kw = dict(iterations=4, weight_constant_axis=axis)
    batch = _trainer(name).fit(np.stack(ys), initialization=np.stack(inits),
                               saliency=np.stack(sals) if with_saliency else None, **kw)
    singles = [_trainer(name).fit(y, initialization=init, saliency=sal, **kw) for y, init, sal in zip(ys, inits, sals)]
    assert batch.weight.shape == (B, 1, K, T if axis == (-3,) else 1)
    got, want = _leaves(batch), [_leaves(m) for m in singles]
    assert got.keys() == want[0].keys()
    for k, v in got.items():
        assert isinstance(v, np.ndarray), k
        assert np.array_equal(v, np.stack([w[k] for w in want])), k


@pytest.mark.gpu
@pytest.mark.parametrize('name', TRAINERS)
def test_time_varying_weight_needs_matching_frame_count(name):
    """A weight per frame (weight_constant_axis=(-3,)) cannot predict an observation with another frame count: the
    reference's broadcast fails with ValueError, and so does every model here."""
    y, _ = synth.structured_stft(6, 80, 4, 2, seed=2)
    m = _trainer(name).fit(y, initialization=synth.init_affiliation(6, 2, 80, seed=1), iterations=3,
                           weight_constant_axis=(-3,))
    assert m.predict(y).shape == (6, 2, 80)
    y2, _ = synth.structured_stft(6, 96, 4, 2, seed=2)
    with pytest.raises(ValueError, match='frames'):
        m.predict(y2)


def test_model_to_host_walks_nested_models():
    """Every tensor field, also of sub-models and fields without an init argument, comes back as NumPy; other fields
    (the integrated models' weight 1 / K, their axes and stream weights) stay as they are; the input is not changed."""
    import torch
    from pb_bss_b200.distribution import (CACGMM, CBMM, GCACGMM, GMM, ComplexAngularCentralGaussian, ComplexBingham,
                                          Gaussian, SphericalGaussian)
    from pb_bss_b200.distribution.mixture_model_utils import model_to_host
    rng = np.random.default_rng(0)
    V = torch.from_numpy(rng.normal(size=(3, 2, 4, 4)) + 1j * rng.normal(size=(3, 2, 4, 4)))
    lam = torch.from_numpy(rng.uniform(size=(3, 2, 4)))
    w = torch.from_numpy(rng.uniform(size=(3, 2, 1)))
    cacg = ComplexAngularCentralGaussian(covariance_eigenvectors=V, covariance_eigenvalues=lam)
    models = [
        CACGMM(weight=w, cacg=cacg),
        CBMM(weight=w, complex_bingham=ComplexBingham(V, lam)),
        GCACGMM(weight=1 / 2, weight_constant_axis=(-2,), cacg=cacg, spatial_weight=0.5,
                gaussian=SphericalGaussian(mean=rng.normal(size=(2, 3)), covariance=np.array([1., 2.]))),
        GMM(weight=w, gaussian=Gaussian._from_device(torch.zeros(3, 2, 3), torch.eye(3).expand(3, 2, 3, 3),
                                                     torch.eye(3).expand(3, 2, 3, 3), torch.zeros(3, 2), False)),
    ]
    for model in models:
        before = _leaves(model)
        host = model_to_host(model)
        assert type(host) is type(model)
        for k, v in _leaves(host).items():
            if isinstance(before[k], torch.Tensor):
                assert isinstance(v, np.ndarray), k
                np.testing.assert_array_equal(v, before[k].numpy())
            else:
                assert v is before[k], k
        assert all(v is before[k] for k, v in _leaves(model).items())
    assert model_to_host(models[2]).weight == 0.5 and model_to_host(models[3]).gaussian.precision_cholesky.shape == (
        3, 2, 3, 3)


def test_fit_tied_leading_picks_every_leading_index_and_stacks():
    """The array arguments are picked at each leading index (trailing dims: y 3, initialization 3, saliency 2,
    source_activity_mask 3; singleton and missing leading dims broadcast) and the models stack to (*lead, ...)."""
    from pb_bss_b200.distribution import CACGMM, ComplexAngularCentralGaussian
    from pb_bss_b200.distribution.mixture_model_utils import fit_tied_leading
    lead, F, N, D, K = (2, 3), 4, 5, 2, 2
    rng = np.random.default_rng(1)
    y = rng.normal(size=lead + (F, N, D))
    init = rng.uniform(size=(1, 3, F, K, N))
    sal = rng.uniform(size=(2, 1, F, N))
    mask = rng.uniform(size=(F, K, N)) > 0.5
    calls = []

    def fit(y, initialization, saliency, source_activity_mask, iterations):
        assert y.shape == (F, N, D) and initialization.shape == (F, K, N) and saliency.shape == (F, N)
        calls.append(iterations)
        return CACGMM(weight=y, cacg=ComplexAngularCentralGaussian(
            covariance_eigenvectors=np.stack([initialization, source_activity_mask]),
            covariance_eigenvalues=saliency))

    m = fit_tied_leading(fit, lead, y=y, initialization=init, saliency=sal, source_activity_mask=mask, iterations=7)
    assert calls == [7] * 6
    np.testing.assert_array_equal(m.weight, y)
    np.testing.assert_array_equal(m.cacg.covariance_eigenvalues, np.broadcast_to(sal, lead + (F, N)))
    np.testing.assert_array_equal(m.cacg.covariance_eigenvectors[:, :, 0], np.broadcast_to(init, lead + (F, K, N)))
    np.testing.assert_array_equal(m.cacg.covariance_eigenvectors[:, :, 1], np.broadcast_to(mask, lead + (F, K, N)))
