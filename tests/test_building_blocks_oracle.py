"""CPU: the NumPy restatement of oracle/building_blocks_oracle.py reproduces every case of
tests/golden/building_blocks.npz (made from the unmodified reference), and every public name of every module of the
reference resolves under the mirrored pb_bss_b200 module path -- importing the package needs no GPU."""
import importlib
import os

import numpy as np
import pytest

from oracle import building_blocks_oracle as BO

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'building_blocks.npz'))

# Out of scope: test helpers and a network dataset loader (pb_bss.testing), PESQ (evaluation.module_pesq, and the
# `pesq` name pb_bss.evaluation re-exports), the Cython seam (extraction.cythonized) and the sympy-generated Bingham
# normaliser gradients (distribution.complex_bingham_utils).
EXCLUDED_MODULES = {'pb_bss.testing', 'pb_bss.testing.dummy_data', 'pb_bss.testing.module_asserts',
                    'pb_bss.testing.random_utils', 'pb_bss.evaluation.module_pesq', 'pb_bss.extraction.cythonized',
                    'pb_bss.distribution.complex_bingham_utils'}
EXCLUDED_NAMES = {('pb_bss.evaluation', 'pesq')}


def _names():
    return sorted((k[len('names__'):], str(n)) for k in G.files if k.startswith('names__') for n in G[k])


def test_every_public_name_resolves():
    missing = []
    modules = {}
    for mod, name in _names():
        if mod in EXCLUDED_MODULES or (mod, name) in EXCLUDED_NAMES:
            continue
        target = 'pb_bss_b200' + mod[len('pb_bss'):]
        if target not in modules:
            modules[target] = importlib.import_module(target)
        if not hasattr(modules[target], name):
            missing.append(f'{target}.{name}')
    assert not missing, missing
    assert len(_names()) > 150


@pytest.mark.parametrize('case', BO.AFF_CASES, ids=[c[0] for c in BO.AFF_CASES])
def test_affiliation_oracle(case):
    if case[0] not in G:
        pytest.skip('not stored (larger than STORE_MAX)')
    w, lp, m, eps = BO.aff_input(case)
    ref = G[case[0]]
    got = BO.log_pdf_to_affiliation(w, lp, m, eps)
    assert got.dtype == ref.dtype
    rtol = 1e-5 if ref.dtype == np.float32 else 1e-12
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=1e-7 if ref.dtype == np.float32 else 0)


def test_error_types_recorded():
    assert str(G['aff_err_bcast']) == 'ValueError'
    assert str(G['aff_err_mask']) == 'AssertionError'
    assert str(G['un_err_style']) == 'AssertionError'
    assert str(G['oh_err_range']) == 'IndexError' and str(G['oh_err_neg']) == 'IndexError'
    assert str(G['oh_err_keep']) == 'AssertionError'
    assert str(G['snr_err_int']) == 'UFuncTypeError'


@pytest.mark.parametrize('tag,K', BO.INT_CASES)
def test_integration_oracle(tag, K):
    w, a, b = BO.int_input(K)
    np.testing.assert_allclose(BO.integration_affiliation(w, a, b), G[tag], rtol=1e-12, atol=0)


@pytest.mark.parametrize('tag,axis,sal', BO.EMW_CASES)
def test_mixture_weight_oracle(tag, axis, sal):
    aff, s = BO.emw_input(sal)
    np.testing.assert_allclose(BO.estimate_mixture_weight(aff, s, axis), G[tag], rtol=1e-13, atol=1e-15)


def test_doctest_values():
    np.testing.assert_allclose(G['emw_doc0'], [[0.6], [0.4]])
    np.testing.assert_allclose(G['emw_doc1'], [[0.5], [0.5]])
    np.testing.assert_allclose(G['emw_doc4'], [[[0.4, 1., 0.4], [0.6, 0., 0.6]]])
    np.testing.assert_allclose(G['un_doc_plus'][0], [7.07056785e-01] * 2, rtol=1e-8)
    np.testing.assert_allclose(G['un_doc_where'][1], [0.70710678] * 2, rtol=1e-8)
    np.testing.assert_array_equal(G['fh_doc'], [[1, 5 - 3j], [5 + 3j, 13]])


@pytest.mark.parametrize('tag,ordv,style,dtype', BO.UNIT_CASES)
def test_unit_norm_oracle(tag, ordv, style, dtype):
    x = BO.unit_input(dtype)
    got = BO.unit_norm(x, -1, 1e-4, style, ordv)
    np.testing.assert_allclose(got, G[tag], rtol=1e-5 if dtype == 'float32' else 1e-12, atol=0)


def test_small_functions_oracle():
    np.testing.assert_allclose(BO.force_hermitian(BO.hermitian_input()), G['fh'], rtol=0, atol=0)
    for tag, lab, C, ax, kd, dt in BO.ONE_HOT_CASES:
        np.testing.assert_array_equal(BO.labels_to_one_hot(lab, C, ax, kd, np.dtype(dt)), G[tag])
        assert G[tag].dtype == np.dtype(dt)
    X, N = BO.snr_input()
    Xc = X + 1j * N[::-1]
    np.testing.assert_allclose(BO.get_energy(Xc, -1), G['energy_ax1'], rtol=1e-13)
    np.testing.assert_allclose(N * BO.set_snr_factor(X, N, 5.0, -1), G['snr_inplace_ax'], rtol=1e-13)
    vec, val = BO.get_pca(BO.pca_input())
    np.testing.assert_allclose(val, G['pca_val_0'], rtol=1e-12)
    np.testing.assert_allclose(np.broadcast_to(val.reshape(-1)[-1], val.shape), G['pca_val_1'], rtol=1e-12)
