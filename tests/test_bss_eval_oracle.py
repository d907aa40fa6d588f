"""CPU checks of BSS Eval: the NumPy restatement (oracle/bss_eval_oracle.py) reproduces the mir_eval numbers the
reference publishes (tests/golden/bss_eval.npz) and the structural cases of the reference's test_mir_eval.py, and
the public entry point raises the reference's errors for bad shapes before it touches the device."""
import numpy as np
import pytest

from oracle import bss_eval_oracle as O
from oracle.make_golden_bss_eval import input_signals


def test_oracle_input_metrics_anchor(golden):
    g = golden('bss_eval')
    ref, est = input_signals(g)
    assert ref.shape == est.shape == (2, 3, 10000)
    sdr, sir, sar = O.mir_eval_sources(ref, est, compute_permutation=False)
    for name, v in (('sdr', sdr), ('sir', sir), ('sar', sar)):
        np.testing.assert_allclose(v, g['input_' + name], rtol=float(g['input_rtol']))


def test_oracle_output_metrics_anchor(golden):
    g = golden('bss_eval')
    out = O.mir_eval_sources(g['output_reference'], g['output_estimation'], return_dict=True)
    for name in ('sdr', 'sir', 'sar'):
        np.testing.assert_allclose(out[name], g['output_' + name], rtol=float(g['output_rtol']))
    np.testing.assert_array_equal(out['selection'], g['output_selection'])


def test_oracle_doctest_anchor(golden):
    """Periodic signals: kappa(G) is about 5.8e19, and LU with partial pivoting still gives the printed 4 decimals."""
    g = golden('bss_eval')
    sdr, sir, sar, sel = O.mir_eval_sources(g['doctest_reference'], g['doctest_estimation'])
    for name, v in (('sdr', sdr), ('sir', sir), ('sar', sar)):
        np.testing.assert_array_equal(np.round(v, 4), g['doctest_' + name])
    np.testing.assert_array_equal(sel, g['doctest_selection'])


def structural_cases(seed=0, T=8000):
    """The cases of the reference's tests/test_evaluation/test_mir_eval.py with seeded signals: name -> (reference,
    estimation, expected selection)."""
    rng = np.random.default_rng(seed)
    s1, s2, n = rng.standard_normal((3, T))
    return {
        'identical': (np.stack([s1, s2]), np.stack([s1, s2]), [0, 1]),
        'swapped': (np.stack([s1, s2]), np.stack([s2, s1]), [1, 0]),
        'noise_class': (np.stack([s1, s2]), np.stack([s2, n, s1]), [2, 0]),
        'with_channel': (np.array([[s1] * 4, [s2] * 4]), np.array([[s2, n, n, n], [n, s2, s2, s2], [s1] * 4]),
                         np.array([[2, 2, 2, 2], [0, 1, 1, 1]])),
    }


@pytest.mark.parametrize('case', sorted(structural_cases()))
def test_oracle_structural_cases(case):
    ref, est, selection = structural_cases()[case]
    sdr, sir, sar, sel = O.mir_eval_sources(ref, est)
    for v in (sdr, sir, sar):
        assert v.shape == ref.shape[:-1] and np.all(v > 100), v
    assert sel.shape == ref.shape[:-1] and sel.dtype == np.int64
    np.testing.assert_array_equal(sel, selection)


def test_oracle_permutation_rules():
    """np.mean / np.argmax: +inf wins, the first of equal means wins, and the first NaN mean wins."""
    inf = np.inf
    z = np.zeros((3, 2))
    sir = np.array([[1.0, 2.0], [inf, 0.0], [3.0, 4.0]])
    assert list(O.select(z, sir, z)[3]) == [1, 0]
    sir = np.array([[1.0, 1.0], [1.0, 1.0], [1.0, 1.0]])
    assert list(O.select(z, sir, z)[3]) == [0, 1]
    sir = np.array([[1.0, inf], [-inf, 0.0], [2.0, 2.0]])   # mean of (1, 0) is nan, of (2, 0) inf
    assert list(O.select(z, sir, z)[3]) == [1, 0]


@pytest.mark.parametrize('ref_shape, est_shape, kwargs, exc', [
    ((2, 100), (2, 101), {}, AssertionError),
    ((2, 100), (2, 3, 100), {}, AssertionError),
    ((2, 3, 100), (2, 4, 100), {}, AssertionError),
    ((2, 100), (4, 100), {}, ValueError),
    ((2, 3, 100), (1, 3, 100), {}, ValueError),
    ((100,), (100,), {}, ValueError),
    ((), (), {}, ValueError),
    ((2, 100), (3, 100), {'compute_permutation': False}, NotImplementedError),
    ((2, 3, 100), (3, 3, 100), {'compute_permutation': False}, NotImplementedError),
    ((9, 100), (9, 100), {}, ValueError),
    ((2, 0), (2, 0), {}, ValueError),
    ((2, 0, 100), (2, 0, 100), {}, ValueError),
])
def test_shape_errors_are_raised_before_the_device(ref_shape, est_shape, kwargs, exc):
    from pb_bss_b200.evaluation import mir_eval_sources
    with pytest.raises(exc):
        mir_eval_sources(np.ones(ref_shape), np.ones(est_shape), **kwargs)


def test_complex_input_raises_type_error():
    from pb_bss_b200.evaluation import mir_eval_sources
    with pytest.raises(TypeError):
        mir_eval_sources(np.ones((2, 100), np.complex128), np.ones((2, 100)))
    with pytest.raises(TypeError):
        mir_eval_sources(np.ones((2, 100)), np.ones((3, 100), np.complex64))
