"""Pins the NumPy restatement of the integrated models (oracle/integration_oracle.py: GCACGMM, VMFCACGMM, the inline
pairing of spatial and spectral classes) to fixtures made by the unmodified reference: tests/golden/gcacgmm.npz,
vmfcacgmm.npz (oracle/make_golden.py: make_gcacgmm) and integration_shapes.npz (oracle/make_golden_integration.py).
CPU only."""
import itertools
import warnings

import numpy as np
import pytest

from conftest import load_golden
from oracle import integration_oracle as IO
from oracle import pb_bss_oracle as PO
from oracle.make_golden_integration import CASES, ERROR_AXES, PROBLEMS, embedding_of, fixture_inputs, resolve

RT = dict(rtol=1e-12, atol=1e-14)

# the cases of make_golden.make_gcacgmm: name -> (fixture, spectral model, keyword arguments)
OLD_CASES = {
    'spherical': ('gcacgmm', 'gaussian', dict()),
    'diagonal_kt': ('gcacgmm', 'gaussian', dict(covariance_type='diagonal', weight_constant_axis=(-3,))),
    'spherical_k_inline': ('gcacgmm', 'gaussian', dict(weight_constant_axis=(-3, -1),
                                                       inline_permutation_alignment=True)),
    'spherical_sal_weights': ('gcacgmm', 'gaussian', dict(saliency='saliency', spatial_weight=0.7,
                                                          spectral_weight=1.3)),
    'vmf': ('vmfcacgmm', 'vmf', dict()),
    'vmf_kt_inline': ('vmfcacgmm', 'vmf', dict(weight_constant_axis=(-3,), inline_permutation_alignment=True,
                                               max_concentration=50)),
    'vmf_sal': ('vmfcacgmm', 'vmf', dict(saliency='saliency', spatial_weight=0.6, spectral_weight=1.2,
                                         weight_constant_axis=(-3, -1))),
}


def assert_model_matches(model, g, name, spectral, **tol):
    np.testing.assert_allclose(np.asarray(model['weight']), g[f'{name}_weight'], **tol)
    np.testing.assert_allclose(model['spectral']['mean'], g[f'{name}_mean'], **tol)
    if spectral == 'vmf':
        np.testing.assert_allclose(model['spectral']['concentration'], g[f'{name}_concentration'], **tol)
    else:
        np.testing.assert_allclose(model['spectral']['covariance'], g[f'{name}_gcov'], **tol)
    np.testing.assert_allclose(model['eigenvalues'], g[f'{name}_eigenvalues'], **tol)
    np.testing.assert_allclose(PO.cacg_covariance_from_eig(model['eigenvectors'], model['eigenvalues']),
                               g[f'{name}_covariance'], **tol)


@pytest.mark.parametrize('name', list(OLD_CASES))
def test_oracle_matches_the_original_integration_fixtures(name):
    fixture, spectral, kw = OLD_CASES[name]
    g = load_golden(fixture)
    kw = {k: g[v] if k == 'saliency' else v for k, v in kw.items()}
    model = IO.integrated_fit(g['y'], g['embedding'], g['init'], 4, spectral, **kw)
    assert_model_matches(model, g, name, spectral, **RT)
    np.testing.assert_allclose(IO.integrated_predict(g['y'], g['embedding'], model), g[f'{name}_affiliation'], **RT)


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_matches_the_shape_sweep_fixture(name):
    g = load_golden('integration_shapes')
    problem, spectral, kw = CASES[name]
    d = fixture_inputs(g, problem)
    emb = embedding_of(d, spectral)
    model = IO.integrated_fit(d['y'], emb, d['init'], int(g['iterations']), spectral, **resolve(d, kw))
    assert_model_matches(model, g, name, spectral, **RT)
    np.testing.assert_allclose(IO.integrated_predict(d['y'], emb, model), g[f'{name}_affiliation'], **RT)
    if kw.get('inline_permutation_alignment'):
        assert model['min_margin'] > 1e-6


def test_shape_sweep_fixture_covers_the_shapes():
    g = load_golden('integration_shapes')
    for problem, (F, T, D, E, K) in PROBLEMS.items():
        d = fixture_inputs(g, problem)
        assert d['y'].shape == (F, T, D) and d['embedding'].shape == (F, T, E)
        assert d['init'].shape == (F, K, T)
        assert (d['saliency'] == 0).any()
    assert {K for *_, K in PROBLEMS.values()} == {1, 2, 4, 6}
    assert {E for *_, E, _ in PROBLEMS.values()} == {1, 16, 33, 64}


def test_reference_rejects_a_constant_weight_it_cannot_unsqueeze():
    """weight_constant_axis (-2,) and (-3, -2): the scalar 1 / K cannot be unsqueezed to that many dims."""
    g = load_golden('integration_shapes')
    assert str(g['error_axes_m2']) == 'IndexError' and str(g['error_axes_m3m2']) == 'IndexError'
    assert str(g['error_axes_m2m1']) == ''
    assert set(ERROR_AXES) == {k for k in g if k.startswith('error_axes_')}
    for key, axes in ERROR_AXES.items():
        expected = str(g[key])
        try:
            IO.unsqueeze(1 / 3, axes)
            got = ''
        except IndexError:
            got = 'IndexError'
        assert got == expected, (axes, got, expected)


def test_unsqueeze_and_class_weight_layouts():
    rng = np.random.RandomState(0)
    m = rng.uniform(size=(3, 4, 5))
    for axes, shape in (((-1,), (3, 4)), ((-3,), (4, 5)), ((-3, -1), (4,))):
        w = IO.class_weight(m.copy(), axes)
        assert w.shape == shape
        np.testing.assert_allclose(IO.unsqueeze(w, axes).sum(-2), 1, rtol=1e-14)
    assert IO.class_weight(m, (-3, -2, -1)) == 1 / 4
    assert IO.unsqueeze(1 / 4, (-3, -2, -1)).shape == (1, 1, 1)


@pytest.mark.parametrize('K', [1, 2, 3, 4, 5, 6])
def test_inline_pairing_oracle_is_the_first_argmax_over_itertools_permutations(K):
    """Brute force over itertools.permutations with the reference's auxiliary function, margin and choice."""
    rng = np.random.RandomState(K)
    F, T = 3, 40
    a, b = rng.randn(F, K, T) * 3, rng.randn(F, K, T) * 3
    weight = rng.uniform(0.1, 1, size=(F, K, 1))
    aff, chosen, margin = IO.inline_pa_affiliation(weight, a, b)
    perms = list(itertools.permutations(range(K)))
    for f in range(F):
        aux = []
        for p in perms:
            lp = a[f, list(p)] + b[f]
            s = np.exp(lp - lp.max(0))
            s /= s.sum(0)
            aux.append(np.sum(s * lp))
        best = int(np.argmax(aux))
        assert tuple(chosen[f]) == perms[best]
        if K > 1:
            gap = aux[best] - sorted(aux)[-2]
            np.testing.assert_allclose(margin[f], gap / np.max(np.abs(aux)), rtol=1e-10)
        np.testing.assert_allclose(
            aff[f], PO.log_pdf_to_affiliation(weight[f], a[f, list(chosen[f])] + b[f]), rtol=1e-14)
    # a tie keeps the first permutation, like the reference's strict '>'
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        _, chosen, margin = IO.inline_pa_affiliation(1., np.zeros((1, K, 4)), b[:1, :, :4])
    assert tuple(chosen[0]) == tuple(range(K))
