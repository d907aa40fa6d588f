"""The building blocks on the device -- mixture_model_utils, distribution.utils, pb_bss_b200.utils and the sxr_module
completions -- against tests/golden/building_blocks.npz (the unmodified reference) and the NumPy restatement of
oracle/building_blocks_oracle.py.  fp64 results are held to rtol 1e-13 where the computation is the reference's
order of operations, and to the bound of a reordered sum where the device sums in another order than NumPy's pairwise
sum; float32 results to 2 ulp of the fp64 result rounded once.  Every function: NumPy in gives NumPy out, CUDA in gives
CUDA out, and two calls give the same bits."""
import os

import numpy as np
import pytest
import torch

from oracle import building_blocks_oracle as BO

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'building_blocks.npz'))


def _cuda(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda() if isinstance(x, np.ndarray) else x


def _same_both_ways(fn, *args, **kwargs):
    """fn on NumPy and on CUDA tensors (same values): NumPy out / CUDA out, bit-identical, and reproducible."""
    a = fn(*args, **kwargs)
    b = fn(*args, **kwargs)
    assert isinstance(a, np.ndarray), type(a)
    np.testing.assert_array_equal(a, b)
    c = fn(*[_cuda(x) if isinstance(x, np.ndarray) else x for x in args], **kwargs)
    assert isinstance(c, torch.Tensor) and c.is_cuda
    np.testing.assert_array_equal(c.cpu().numpy(), a)
    return a


def _f32_close(got, want64):
    np.testing.assert_array_max_ulp(got, want64.astype(np.float32), maxulp=2)


# ---- log_pdf_to_affiliation ----------------------------------------------------------------------------------------

@pytest.mark.parametrize('case', BO.AFF_CASES, ids=[c[0] for c in BO.AFF_CASES])
def test_log_pdf_to_affiliation(case):
    from pb_bss_b200.distribution.mixture_model_utils import log_pdf_to_affiliation
    w, lp, m, eps = BO.aff_input(case)
    got = _same_both_ways(log_pdf_to_affiliation, w, lp, m, eps)
    assert got.dtype == lp.dtype and got.shape == lp.shape
    want = BO.log_pdf_to_affiliation(w, lp.astype(np.float64), m, eps)
    if lp.dtype == np.float32:
        _f32_close(got, want)
    else:
        np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-300)
        if case[0] in G:
            np.testing.assert_allclose(got, G[case[0]], rtol=1e-13, atol=1e-300)
    if case[7] == 'neginf':
        assert np.isnan(got[..., 3]).all()
    if case[7] == 'masked_out':
        assert (got[..., 5] == 0).all()


def test_log_pdf_to_affiliation_errors():
    from pb_bss_b200.distribution.mixture_model_utils import log_pdf_to_affiliation
    w, lp, m = BO.aff_error_input('bcast')
    with pytest.raises(ValueError):
        log_pdf_to_affiliation(w, lp, m)
    w, lp, m = BO.aff_error_input('mask_dtype')
    with pytest.raises(AssertionError):
        log_pdf_to_affiliation(w, lp, m)
    assert str(G['aff_err_bcast']) == 'ValueError' and str(G['aff_err_mask']) == 'AssertionError'


def test_log_pdf_to_affiliation_leaves_inputs_alone():
    from pb_bss_b200.distribution.mixture_model_utils import log_pdf_to_affiliation
    w, lp, m, eps = BO.aff_input(BO.AFF_CASES[10])
    lp0 = lp.copy()
    t = torch.from_numpy(lp).cuda()
    log_pdf_to_affiliation(w, lp, m, eps)
    log_pdf_to_affiliation(w, t, m, eps)
    np.testing.assert_array_equal(lp, lp0)
    np.testing.assert_array_equal(t.cpu().numpy(), lp0)


@pytest.mark.parametrize('tag,K', BO.INT_CASES)
def test_integration_inline_pa(tag, K):
    from pb_bss_b200.distribution.mixture_model_utils import \
        log_pdf_to_affiliation_for_integration_models_with_inline_pa as f
    w, a, b = BO.int_input(K)
    got = _same_both_ways(f, w, a, b)
    assert got.dtype == np.float64
    np.testing.assert_allclose(got, G[tag], rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(got, f(np.broadcast_to(w, a.shape).copy(), a, b), rtol=0, atol=0)


def test_integration_inline_pa_k7():
    from pb_bss_b200.distribution.mixture_model_utils import \
        log_pdf_to_affiliation_for_integration_models_with_inline_pa as f
    a = np.zeros((2, 7, 5))
    with pytest.raises(NotImplementedError, match='K <= 6'):
        f(np.ones((7, 1)), a, a)


# ---- estimate_mixture_weight ---------------------------------------------------------------------------------------

@pytest.mark.parametrize('tag,axis,sal', BO.EMW_CASES)
def test_estimate_mixture_weight(tag, axis, sal):
    from pb_bss_b200.distribution.mixture_model_utils import estimate_mixture_weight
    aff, s = BO.emw_input(sal)
    got = _same_both_ways(estimate_mixture_weight, aff, s, axis)
    want = G[tag]
    assert got.shape == want.shape and got.dtype == want.dtype
    # a reordered sum of at most n = 4 * 3 * 41 terms in [0, 1]: |error| <= n eps sum
    n = aff.size
    np.testing.assert_allclose(got, want, rtol=n * np.finfo(float).eps, atol=1e-15)


def test_estimate_mixture_weight_doctest():
    from pb_bss_b200.distribution.mixture_model_utils import estimate_mixture_weight
    doc = [[0.4, 1, 0.4], [0.6, 0, 0.6]]
    for i, (a, ax) in enumerate([(doc, -1), (doc, -2), ([doc, doc], -1), ([doc, doc], -2), ([doc, doc], -3)]):
        np.testing.assert_allclose(estimate_mixture_weight(a, weight_constant_axis=ax), G[f'emw_doc{i}'], rtol=1e-15)


def test_apply_inline_permutation_alignment():
    from pb_bss_b200.distribution.mixture_model_utils import apply_inline_permutation_alignment
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    r = np.random.default_rng(3)
    F, K, T = 257, 3, 60
    aff = r.random((F, K, T))
    aff /= aff.sum(1, keepdims=True)
    q = r.random((F, K, T))
    aligner = DHTVPermutationAlignment.from_stft_size(512)
    got_a, got_q = apply_inline_permutation_alignment(aff, quadratic_form=q, weight_constant_axis=(-3, -1),
                                                      aligner=aligner)
    mapping = aligner.calculate_mapping(aff.transpose(1, 0, 2))
    want_a = aligner.apply_mapping(aff.transpose(1, 0, 2), mapping).transpose(1, 0, 2)
    np.testing.assert_array_equal(got_a, want_a)
    np.testing.assert_array_equal(got_q, aligner.apply_mapping(q.transpose(1, 0, 2), mapping).transpose(1, 0, 2))
    only = apply_inline_permutation_alignment(aff, weight_constant_axis=-3, aligner=aligner)
    np.testing.assert_array_equal(only, want_a)
    with pytest.raises(AssertionError, match='Inline permutation alignment'):
        apply_inline_permutation_alignment(aff, weight_constant_axis=-1, aligner=aligner)


# ---- distribution.utils ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('tag,ordv,style,dtype', BO.UNIT_CASES)
def test_unit_norm(tag, ordv, style, dtype):
    from pb_bss_b200.distribution.utils import _unit_norm
    x = BO.unit_input(dtype)
    got = _same_both_ways(_unit_norm, x, eps_style=style, ord=ordv)
    assert got.dtype == x.dtype
    want = BO.unit_norm(x.astype(np.complex128 if x.dtype.kind == 'c' else np.float64), -1, 1e-4, style, ordv)
    if dtype == 'float32':
        _f32_close(got, want)
    else:
        # n = 5 terms summed in another order than NumPy's, then pow / sqrt: a few ulp
        np.testing.assert_allclose(got, want, rtol=1e-14, atol=1e-300)
        np.testing.assert_allclose(got, G[tag], rtol=1e-14, atol=1e-300)


def test_unit_norm_doctest_and_errors():
    from pb_bss_b200.distribution.utils import _unit_norm
    sig = np.array([[1, 1], [1e-20, 1e-20], [0, 0]])
    for st in ('plus', 'max', 'where'):
        np.testing.assert_allclose(_unit_norm(sig, eps_style=st), G[f'un_doc_{st}'], rtol=1e-15, atol=0)
    with pytest.raises(AssertionError):
        _unit_norm(sig, eps_style='other')


def test_force_hermitian():
    from pb_bss_b200.distribution.utils import force_hermitian
    from pb_bss_b200.distribution import complex_bingham
    assert complex_bingham.force_hermitian is force_hermitian
    np.testing.assert_array_equal(_same_both_ways(force_hermitian, BO.hermitian_input()), G['fh'])
    real = _same_both_ways(force_hermitian, BO.hermitian_input().real)
    assert real.dtype == np.float64
    np.testing.assert_array_equal(real, G['fh_real'])
    A = np.array([[1 + 2j, 3 + 5j], [7 + 11j, 13 + 17j]])
    np.testing.assert_array_equal(force_hermitian(A), G['fh_doc'])
    np.testing.assert_array_equal(force_hermitian(force_hermitian(A)), G['fh_doc'])


def test_normalize_observation_watson_bingham():
    from pb_bss_b200.distribution import complex_bingham, complex_watson
    assert complex_bingham.normalize_observation is complex_watson.normalize_observation
    r = np.random.default_rng(5)
    y = r.normal(size=(3, 20, 4)) + 1j * r.normal(size=(3, 20, 4))
    y[1, 3] = 0
    got = _same_both_ways(complex_watson.normalize_observation, y)
    want = y / np.maximum(np.linalg.norm(y, axis=-1, keepdims=True), np.finfo(y.dtype).tiny)
    np.testing.assert_allclose(got, want, rtol=1e-14, atol=0)


def test_stack_parameters_and_lookup():
    from pb_bss_b200.distribution import CACGMM, ComplexAngularCentralGaussian, ComplexAngularCentralGaussianTrainer
    from pb_bss_b200.distribution.utils import get_trainer_class_from_model, parameter_from_dict, stack_parameters
    m1 = ComplexAngularCentralGaussian.from_covariance(covariance=[[1, 0], [0, 1]])
    m2 = ComplexAngularCentralGaussian.from_covariance(covariance=[[3, 1], [1, 2]])
    s = stack_parameters([m1, m2])
    np.testing.assert_allclose(s.covariance_eigenvalues, [[1, 1], [0.38196601, 1]], rtol=1e-7)
    w = stack_parameters([CACGMM(cacg=m1, weight=np.array([6])), CACGMM(cacg=m2, weight=np.array([9]))])
    np.testing.assert_array_equal(w.weight, [[6], [9]])
    assert get_trainer_class_from_model(ComplexAngularCentralGaussian) is ComplexAngularCentralGaussianTrainer
    assert get_trainer_class_from_model(m1) is ComplexAngularCentralGaussianTrainer
    again = parameter_from_dict('ComplexAngularCentralGaussian', m1.to_dict())
    np.testing.assert_array_equal(again.covariance_eigenvalues, m1.covariance_eigenvalues)
    t = stack_parameters([CACGMM(cacg=m1, weight=torch.ones(2).cuda()), CACGMM(cacg=m2, weight=torch.ones(2).cuda())])
    assert t.weight.is_cuda and tuple(t.weight.shape) == (2, 2)


# ---- pb_bss_b200.utils ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('tag,lab,C,axis,keepdims,dtype', BO.ONE_HOT_CASES)
def test_labels_to_one_hot(tag, lab, C, axis, keepdims, dtype):
    from pb_bss_b200.utils import labels_to_one_hot
    got = _same_both_ways(labels_to_one_hot, np.asarray(lab), C, axis=axis, keepdims=keepdims, dtype=np.dtype(dtype))
    assert got.dtype == np.dtype(dtype)
    np.testing.assert_array_equal(got, G[tag])
    np.testing.assert_array_equal(labels_to_one_hot(lab, C, axis=axis, keepdims=keepdims, dtype=np.dtype(dtype)), got)


@pytest.mark.parametrize('tag,lab,C,axis,keepdims', BO.ONE_HOT_ERRORS)
def test_labels_to_one_hot_errors(tag, lab, C, axis, keepdims):
    from pb_bss_b200.utils import labels_to_one_hot
    with pytest.raises({'IndexError': IndexError, 'AssertionError': AssertionError}[str(G[tag])]):
        labels_to_one_hot(lab, C, axis=axis, keepdims=keepdims)


@pytest.mark.parametrize('use_scipy', [False, True])
def test_get_pca(use_scipy):
    from pb_bss_b200.utils import get_pca
    P = BO.pca_input()
    vec, val = get_pca(P, use_scipy=use_scipy)
    tv, tval = get_pca(torch.from_numpy(P).cuda(), use_scipy=use_scipy)
    np.testing.assert_array_equal(tv.cpu().numpy(), vec)
    np.testing.assert_array_equal(tval.cpu().numpy(), val)
    want_vec, want_val = G[f'pca_vec_{int(use_scipy)}'], G[f'pca_val_{int(use_scipy)}']
    assert vec.shape == want_vec.shape and val.shape == want_val.shape
    np.testing.assert_allclose(val, want_val, rtol=1e-12)
    # eigenvectors up to their phase: |<v, w>| = 1
    np.testing.assert_allclose(np.abs(np.sum(np.conj(vec) * want_vec, -1)), 1, rtol=0, atol=1e-10)


@pytest.mark.parametrize('dtype', ['complex128', 'complex64', 'float64', 'float32'])
def test_abs_square(dtype):
    from pb_bss_b200.utils import abs_square
    rr = BO.rng('abs')
    xs = {}
    for dt in ('complex128', 'complex64', 'float64', 'float32'):
        xs[dt] = (rr.normal(size=(7, 9)) + (1j * rr.normal(size=(7, 9)) if dt.startswith('complex') else 0)).astype(dt)
    got = _same_both_ways(abs_square, xs[dtype])
    assert got.dtype == G[f'abs_{dtype}'].dtype
    np.testing.assert_array_equal(got, G[f'abs_{dtype}'])


def test_host_helpers():
    from pb_bss_b200 import math as pmath, utils
    from pb_bss_b200.extraction import linalg
    assert pmath.solve.stable_solve is linalg.stable_solve
    assert utils.is_broadcast_compatible((2, 3), (3,)) and not utils.is_broadcast_compatible((2, 3), (2,))
    x = torch.arange(24.0, device='cuda').reshape(2, 3, 4)
    np.testing.assert_array_equal(utils.reshape(x, 'a b c -> c a*b').cpu().numpy(),
                                  utils.reshape(x.cpu().numpy(), 'a b c -> c a*b'))
    with pytest.warns(utils.DeprecatedWarning):
        utils.deprecated('use g')(lambda: 1)()


# ---- sxr_module and VonMisesFisher ----------------------------------------------------------------------------------

@pytest.mark.parametrize('tag,axis,keepdims', [('all', None, False), ('ax1', -1, False), ('ax01k', (0, 1), True)])
def test_get_energy(tag, axis, keepdims):
    from pb_bss_b200.evaluation.sxr_module import get_energy
    X, N = BO.snr_input()
    Xc = X + 1j * N[::-1]
    got = get_energy(Xc, axis=axis, keepdims=keepdims)
    assert np.shape(got) == np.shape(G[f'energy_{tag}'])
    again = get_energy(torch.from_numpy(Xc).cuda(), axis=axis, keepdims=keepdims)
    np.testing.assert_array_equal(again.cpu().numpy(), got)
    # a reordered sum of n non-negative terms: |error| <= n eps sum
    n = Xc.size
    np.testing.assert_allclose(got, G[f'energy_{tag}'], rtol=n * np.finfo(float).eps, atol=0)


@pytest.mark.parametrize('axis', [None, -1])
def test_set_snr(axis):
    from pb_bss_b200.evaluation.sxr_module import set_snr
    X, N = BO.snr_input()
    tag = 'none' if axis is None else 'ax'
    # the factor comes from two reordered sums of 300 (or 50) squares
    rtol = 1e-13
    Nn = N.copy()
    assert set_snr(X, Nn, 5.0, axis=axis) is None
    np.testing.assert_allclose(Nn, G[f'snr_inplace_{tag}'], rtol=rtol)
    Nt = torch.from_numpy(N.copy()).cuda()
    assert set_snr(torch.from_numpy(X).cuda(), Nt, 5.0, axis=axis) is None
    np.testing.assert_array_equal(Nt.cpu().numpy(), Nn)
    X2, N2 = set_snr(X, N, 5.0, axis=axis, inplace=False)
    assert X2 is X
    np.testing.assert_allclose(N2, G[f'snr_copy_{tag}'], rtol=rtol)
    with pytest.raises(TypeError):
        set_snr(X, np.ones((2, 3, 50), np.int64), 5.0)


def test_von_mises_fisher_pdf_norm_sample():
    from pb_bss_b200.distribution import VonMisesFisher
    r = np.random.default_rng(7)
    mean = r.normal(size=(3, 5))
    mean /= np.linalg.norm(mean, axis=-1, keepdims=True)
    m = VonMisesFisher(mean=mean, concentration=np.array([1.0, 5.0, 20.0]))
    y = r.normal(size=(3, 40, 5))
    pdf = m.pdf(y)
    np.testing.assert_allclose(pdf, np.exp(m.log_pdf(y)), rtol=1e-14, atol=0)
    np.testing.assert_allclose(m.norm(), np.exp(m.log_norm()), rtol=0, atol=0)
    with pytest.raises(NotImplementedError):
        m.sample(3)


# ---- strided CUDA views, long reductions over few outputs, argument order and dtypes ------------------------------

def _transposed_view(a):
    """A CUDA view of a's values whose last two axes are transposed in memory (non-contiguous, class stride 1)."""
    t = torch.from_numpy(np.ascontiguousarray(np.swapaxes(a, -1, -2))).cuda().transpose(-1, -2)
    assert not t.is_contiguous()
    return t


@pytest.mark.parametrize('case', [c for c in BO.AFF_CASES if c[7] == 'transposed' or c[4]],
                         ids=[c[0] for c in BO.AFF_CASES if c[7] == 'transposed' or c[4]])
def test_log_pdf_to_affiliation_transposed_cuda_views(case):
    """log_pdf, mask and a 3-d weight passed as transposed CUDA views reach the kernel in their own strides."""
    from pb_bss_b200.distribution.mixture_model_utils import log_pdf_to_affiliation
    w, lp, m, eps = BO.aff_input(case)
    want = log_pdf_to_affiliation(np.ascontiguousarray(w), np.ascontiguousarray(lp),
                                  None if m is None else np.ascontiguousarray(m), eps)
    wt = _transposed_view(w) if np.ndim(w) >= 2 and min(np.shape(w)[-2:]) > 1 else w
    got = log_pdf_to_affiliation(wt, _transposed_view(lp), None if m is None else _transposed_view(m), eps)
    np.testing.assert_array_equal(got.cpu().numpy(), want)


def test_log_pdf_to_affiliation_check_order():
    """A weight that broadcasts log_pdf to a larger shape raises ValueError before the mask's dtype is checked, as
    the reference's ``affiliation *= weight`` comes before its mask assert."""
    from pb_bss_b200.distribution.mixture_model_utils import log_pdf_to_affiliation
    lp = np.zeros((3, 11))
    with pytest.raises(ValueError):
        log_pdf_to_affiliation(np.ones((2, 3, 1)), lp, np.ones((3, 11), np.int64))
    with pytest.raises(AssertionError):
        log_pdf_to_affiliation(np.ones((3, 1)), lp, np.ones((3, 11), np.int64))
    with pytest.raises(ValueError):
        log_pdf_to_affiliation(np.ones((3, 1)), lp, np.ones((2, 3, 11), bool))


def _repeatable(fn, *args, **kwargs):
    a = fn(*args, **kwargs)
    np.testing.assert_array_equal(a, fn(*args, **kwargs))
    return a


@pytest.mark.parametrize('axis', [(-3, -1), (-3,), -3])
@pytest.mark.parametrize('saliency', [False, True])
def test_estimate_mixture_weight_long_reductions(axis, saliency):
    """Frequency-tied weights: K (or K * T) outputs, each a sum over F * T (or F) = 25800 (129) affiliations, which
    the reduction splits over chunks."""
    from pb_bss_b200.distribution.mixture_model_utils import estimate_mixture_weight
    r = np.random.default_rng(11)
    aff = r.random((129, 3, 200))
    aff /= aff.sum(-2, keepdims=True)
    sal = (r.random((129, 200)) < 0.6).astype(np.float64) if saliency else None
    got = _repeatable(estimate_mixture_weight, aff, sal, axis)
    t = estimate_mixture_weight(torch.from_numpy(aff).cuda(), None if sal is None else torch.from_numpy(sal).cuda(),
                                axis)
    np.testing.assert_array_equal(t.cpu().numpy(), got)
    want = BO.estimate_mixture_weight(aff, sal, axis)
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=aff.size * np.finfo(float).eps, atol=0)


def test_estimate_mixture_weight_bool_saliency_keeps_float32():
    from pb_bss_b200.distribution.mixture_model_utils import estimate_mixture_weight
    aff, sal = BO.emw_input(True)
    got = estimate_mixture_weight(aff.astype(np.float32), sal.astype(bool), -1)
    want = BO.estimate_mixture_weight(aff.astype(np.float32), sal.astype(bool), -1)
    assert got.dtype == want.dtype == np.float32


@pytest.mark.parametrize('shape,axis', [((3, 5000), None), ((3, 5000), -1), ((2, 3, 5000), (0, 2)), ((60000,), 0)])
def test_get_energy_long_reductions(shape, axis):
    from pb_bss_b200.evaluation.sxr_module import get_energy
    r = np.random.default_rng(12)
    x = r.normal(size=shape) + 1j * r.normal(size=shape)
    got = _repeatable(get_energy, x, axis=axis)
    np.testing.assert_array_equal(get_energy(torch.from_numpy(x).cuda(), axis=axis).cpu().numpy(), got)
    np.testing.assert_allclose(got, BO.get_energy(x, axis), rtol=x.size * np.finfo(float).eps, atol=0)


@pytest.mark.parametrize('ordv', [None, 1, np.inf, -np.inf, 0, 3, 0.5])
@pytest.mark.parametrize('axis', [-1, 0])
def test_unit_norm_long_vectors(ordv, axis):
    """Few long vectors (20000 elements, contiguous or 3 apart): the norms are chunked reductions."""
    from pb_bss_b200.distribution.utils import _unit_norm
    r = np.random.default_rng(13)
    x = r.normal(size=(3, 20000) if axis == -1 else (20000, 3)) + 1j * r.normal(size=(3, 20000) if axis == -1
                                                                              else (20000, 3))
    x[(0, 5) if axis == -1 else (5, 0)] = 0
    got = _repeatable(_unit_norm, x, axis=axis, ord=ordv)
    np.testing.assert_array_equal(_unit_norm(torch.from_numpy(x).cuda(), axis=axis, ord=ordv).cpu().numpy(), got)
    # 20000 terms summed in another order, then root and quotient
    np.testing.assert_allclose(got, BO.unit_norm(x, axis, 1e-4, 'plus', ordv), rtol=20000 * np.finfo(float).eps,
                               atol=0)


@pytest.mark.parametrize('values,dtype', [([True, False], 'bool'), ([0.5, -3.25, 300.0], 'float16'),
                                          ([3, 300, 65535], 'uint16'), ([3, -12, 127], 'int8'),
                                          ([7, -46341], 'int32')])
def test_abs_square_numpy_dtypes(values, dtype):
    """NumPy's result dtype and bits, integer wrap-around included."""
    from pb_bss_b200.utils import abs_square
    x = np.array(values, dtype=dtype)
    with np.errstate(over='ignore'):
        want = x ** 2
    got = abs_square(x)
    assert got.dtype == want.dtype
    np.testing.assert_array_equal(got, want)
