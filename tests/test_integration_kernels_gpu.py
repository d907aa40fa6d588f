"""The kernels of csrc/api_integration.cu (embedding Gaussians / von Mises-Fisher, the integrated posterior with the
inline pairing, the class weights) against the float64 NumPy oracles at the shapes where their code branches:
E across every template bucket, accumulator step and 32-lane loop, K = 1..6, N / T across the block and tile edges,
B * K at both ends of the chunking.  Then the integrated models (GCACGMM, VMFCACGMM) against the reference's fixtures
(tests/golden/integration_shapes.npz) and the oracle, and GMM / VMFMM at large E."""
import itertools

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import embedding_oracle as EO
from oracle import integration_oracle as IO
from oracle import pb_bss_oracle as PO
from oracle import synth
from oracle.make_golden_integration import CASES, ERROR_AXES, embedding_of, fixture_inputs, resolve

pytestmark = pytest.mark.gpu

REL = 1e-12
MODEL = dict(rtol=1e-7, atol=1e-10)
AFF = dict(rtol=1e-6, atol=1e-9)
E_SWEEP = [1, 7, 8, 9, 15, 16, 17, 22, 23, 31, 32, 33, 63, 64]
T_SWEEP = [1, 255, 256, 257, 1000]
# (B, N) per class count: B * K = 1 (one CTA row, the most chunks) up to 1200 (one chunk); N across the 32-row tiles
BN = [(1, 5000), (3, 31), (200, 32), (1, 1), (3, 300), (2, 33)]


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')


def _d(x, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(x)).to(device='cuda', dtype=dtype)


def _h(t):
    return t.cpu().numpy()


def _rows_close(out, ref, row_ndim=1, rel=REL, floor=0.):
    """|out - ref| <= rel * max(max |ref| of the row, floor); a row is the last ``row_ndim`` axes."""
    out, ref = np.asarray(out), np.asarray(ref)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    n = int(np.prod(ref.shape[ref.ndim - row_ndim:]))
    r, o = ref.reshape(-1, n), out.reshape(-1, n)
    scale = np.maximum(np.abs(r).max(axis=-1, keepdims=True), max(floor, 1e-300))
    err = np.abs(o - r) / scale
    assert (err <= rel).all(), err.max()


def _spd(rng, lead, E):
    """Covariances a a^T / E + 0.5 I (..., E, E), condition number below about 10."""
    a = rng.randn(*lead, E, E)
    return np.einsum('...ij,...kj->...ik', a, a) / E + 0.5 * np.eye(E)


# ---------------------------------------------------------------- full-covariance Gaussian, B independent models

@pytest.mark.parametrize('E', E_SWEEP)
def test_precision_cholesky_matches_oracle(E):
    from pb_bss_b200.distribution.gaussian import precision_cholesky
    rng = np.random.RandomState(E)
    cov = _spd(rng, (2, 3), E)
    pc, ld = precision_cholesky(_d(cov))
    ref_pc, ref_ld = EO.precision_cholesky_full(cov)
    cond = np.linalg.cond(cov.reshape(-1, E, E)).max()
    _rows_close(_h(pc), ref_pc, 2, rel=REL * cond)
    _rows_close(_h(ld)[..., None], ref_ld[..., None], 1, rel=REL * cond, floor=1.)


def test_precision_cholesky_several_failing_matrices():
    """Failing pivots at indices >= 32 in three matrices of one batch: the status names the smallest failing matrix,
    the failing ones are NaN, the others still match, and the wrapper raises ValueError."""
    from pb_bss_b200 import _lib
    from pb_bss_b200.distribution.gaussian import precision_cholesky
    rng = np.random.RandomState(1)
    M, E = 9, 40
    cov = _spd(rng, (M,), E)
    bad = [6, 2, 7]
    for m, j in zip(bad, (35, 39, 33)):
        cov[m, j, j] = -1.
    lib = _lib.load()
    c = _d(cov)
    pc = torch.empty_like(c)
    ld = torch.empty((M,), dtype=torch.float64, device='cuda')
    status = torch.zeros((1,), dtype=torch.int32, device='cuda')
    _lib.check(lib.pbb_precision_cholesky(c.data_ptr(), M, E, pc.data_ptr(), ld.data_ptr(), status.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), 'pbb_precision_cholesky')
    assert int(status.item()) == min(bad) + 1
    pc, ld = _h(pc), _h(ld)
    good = [m for m in range(M) if m not in bad]
    assert np.isnan(pc[bad]).all() and np.isnan(ld[bad]).all()
    ref_pc, ref_ld = EO.precision_cholesky_full(cov[good])
    _rows_close(pc[good], ref_pc, 2, rel=10 * REL)
    _rows_close(ld[good][:, None], ref_ld[:, None], 1, rel=10 * REL)
    with pytest.raises(ValueError, match='ill-defined empirical covariance'):
        precision_cholesky(c)


@pytest.mark.parametrize('E', E_SWEEP)
def test_full_log_pdf_matches_oracle(E):
    from pb_bss_b200.distribution.gaussian import full_log_pdf_bkn
    rng = np.random.RandomState(100 + E)
    for K in range(1, 7):
        B, N = BN[(K + E) % len(BN)]
        x = rng.randn(B, N, E) * 1.5 + 0.3
        mean = rng.randn(B, K, E)
        pc, ld = EO.precision_cholesky_full(_spd(rng, (B, K), E))
        pc = np.triu(pc)
        out = full_log_pdf_bkn(_d(x), _d(mean), _d(pc), _d(ld))
        _rows_close(_h(out), EO.gaussian_log_pdf(x[:, None], mean, pc, ld), 1)


def _full_moments(y, saliency):
    """The mean and covariance of GaussianTrainer._fit, 'full' (gaussian.py:152-193, the expressions of
    embedding_oracle.gaussian_fit) without the precision Cholesky factor: with N < E the scatter is singular."""
    denominator = np.maximum(np.einsum('...n->...', saliency), np.finfo(np.float64).tiny)
    mean = np.einsum('...n,...nd->...d', saliency, y) / denominator[..., None]
    difference = y - mean[..., None, :]
    cov = np.einsum('...n,...nd,...nD->...dD', saliency, difference, difference) / denominator[..., None, None]
    return mean, cov


@pytest.mark.parametrize('E', E_SWEEP)
def test_full_fit_matches_oracle(E):
    """Both passes of gaussian_full_partial_kernel (pass 1 holds up to 9 accumulators per thread at E = 64) and the
    chunk reduction, from one chunk (B * K = 1200) to 157 chunks (B * K = 1, N = 5000) and ragged last tiles."""
    from pb_bss_b200.distribution.gaussian import full_fit_bkn
    rng = np.random.RandomState(200 + E)
    for K in range(1, 7):
        B, N = BN[(K + 2 * E) % len(BN)]
        if B * N * E * E > 2e8:          # keep the oracle's einsum quick: 200 models at large E get fewer rows
            B = 20
        x = rng.randn(B, N, E) * 2.0 + rng.randn(B, 1, E)
        w = rng.uniform(size=(B, K, N))
        w[w < 0.1] = 0.
        mean, cov = full_fit_bkn(_d(x), _d(w))
        ref_mean, ref_cov = _full_moments(x[:, None], w)
        scale = np.abs(x).max()
        _rows_close(_h(mean), ref_mean, 1, floor=scale)
        _rows_close(_h(cov), ref_cov, 2, floor=scale ** 2 / 100)


@pytest.mark.parametrize('E', E_SWEEP)
def test_vmf_log_pdf_and_resultant_match_oracle(E):
    from pb_bss_b200.distribution.von_mises_fisher import vmf_fit_bkn, vmf_log_pdf_bkn
    rng = np.random.RandomState(300 + E)
    for K in range(1, 7):
        B, N = BN[(K + 3 * E) % len(BN)]
        x = rng.randn(B, N, E) + rng.randn(B, 1, E)
        mean = EO._unit_rows(rng.randn(B, K, E))
        kappa = rng.uniform(1., 20., size=(B, K))
        log_norm = EO.vmf_log_norm(kappa, E)
        out = vmf_log_pdf_bkn(_d(x), _d(mean), _d(kappa), _d(log_norm))
        _rows_close(_h(out), EO.vmf_log_pdf(x[:, None], mean, kappa), 1, floor=1.)
        w = rng.uniform(size=(B, K, N))
        m, c = vmf_fit_bkn(_d(x), _d(w), 1e-10, 500)
        ref_m, ref_c = EO.vmf_fit(EO._unit_rows(x)[:, None], w, 1e-10, 500)
        _rows_close(m, ref_m, 1, rel=1e-10)
        if N > 1 and E > 1:   # r_bar = 1 (one observation, or E = 1 with one sign): eq. 4.4 divides by 0
            np.testing.assert_allclose(c, ref_c, rtol=1e-9)


# ---------------------------------------------------------------- tied diagonal / spherical Gaussian, vMF over (F, T)

KE = list(zip(itertools.cycle(range(1, 7)), E_SWEEP))


def _fkt_inputs(rng, F, T, E, K):
    emb = rng.randn(F, T, E) * 1.5 + rng.randn(1, 1, E)
    w = rng.uniform(size=(F, K, T))
    w[:, :, rng.uniform(size=T) < 0.1] = 0.      # zero-saliency frames
    w[F - 1] = 0.                                # and a whole bin without weight
    return emb, w


def _ft_rows(emb, w):
    F, T, E = emb.shape
    K = w.shape[1]
    return emb.reshape(1, F * T, E), np.transpose(w, (1, 0, 2)).reshape(K, F * T)


@pytest.mark.parametrize('K,E', KE)
@pytest.mark.parametrize('covariance_type', ['diagonal', 'spherical'])
def test_gaussian_fit_fkt_and_log_pdf_match_oracle(K, E, covariance_type):
    """pbb_gaussian_fit and pbb_gaussian_log_pdf, including the diagonal model's contraction over the classes."""
    from pb_bss_b200.distribution.gaussian import gaussian_fit_fkt
    rng = np.random.RandomState(10 * K + E)
    F, T = 3, 257
    emb, w = _fkt_inputs(rng, F, T, E, K)
    model = gaussian_fit_fkt(_d(emb), _d(w), covariance_type)
    ref = EO.gaussian_fit(*_ft_rows(emb, w), covariance_type)
    scale = np.abs(emb).max()
    _rows_close(model.mean, ref['mean'], 1, floor=scale)
    _rows_close(np.reshape(model.covariance, (K, -1)), np.reshape(ref['covariance'], (K, -1)), 1, floor=1e-2)
    out = _h(model.log_pdf_fkt(_d(emb)))
    ref_lp = np.transpose(EO.gaussian_model_log_pdf(ref, emb.reshape(1, F * T, E)).reshape(K, F, T), (1, 0, 2))
    _rows_close(out, ref_lp, 1, rel=1e-10)


@pytest.mark.parametrize('K,E', KE)
def test_vmf_fit_fkt_and_log_pdf_match_oracle(K, E):
    from pb_bss_b200.distribution.von_mises_fisher import vmf_fit_fkt
    rng = np.random.RandomState(20 * K + E)
    F, T = 3, 256
    emb, w = _fkt_inputs(rng, F, T, E, K)
    emb = EO._unit_rows(emb)
    vmf = vmf_fit_fkt(_d(emb), _d(w), 1e-10, 500)
    ref_m, ref_c = EO.vmf_fit(*_ft_rows(emb, w), 1e-10, 500)
    _rows_close(vmf.mean, ref_m, 1, rel=1e-10)
    np.testing.assert_allclose(vmf.concentration, ref_c, rtol=1e-9)
    out = _h(vmf.log_pdf_fkt(_d(emb)))
    ref_lp = EO.vmf_log_pdf(emb.reshape(1, F * T, E), vmf.mean, vmf.concentration)
    _rows_close(out, np.transpose(ref_lp.reshape(K, F, T), (1, 0, 2)), 1, floor=1.)


def test_vmf_fit_fkt_class_without_weight_is_nan_like_the_reference():
    """A class whose weights are all zero: the reference divides the resultant's norm 0 by the raw total 0
    (von_mises_fisher.py:137), so its concentration is NaN and its mean 0."""
    from pb_bss_b200.distribution.von_mises_fisher import vmf_fit_fkt
    rng = np.random.RandomState(3)
    emb, w = _fkt_inputs(rng, 2, 100, 5, 3)
    emb = EO._unit_rows(emb)
    w[:, 1] = 0.
    with np.errstate(invalid='ignore', divide='ignore'):
        vmf = vmf_fit_fkt(_d(emb), _d(w), 1e-10, 500)
        ref_m, ref_c = EO.vmf_fit(*_ft_rows(emb, w), 1e-10, 500)
    assert np.isnan(ref_c[1]) and np.isnan(vmf.concentration[1])
    np.testing.assert_allclose(vmf.concentration, ref_c, rtol=1e-9)
    np.testing.assert_array_equal(vmf.mean[1], 0.)
    _rows_close(vmf.mean, ref_m, 1, rel=1e-10)


# ---------------------------------------------------------------- class weights and the posterior

@pytest.mark.parametrize('T', T_SWEEP)
@pytest.mark.parametrize('axes', [(-1,), (-3,), (-3, -1), (-3, -2, -1)])
def test_class_weights_match_oracle(T, axes):
    from pb_bss_b200.distribution.gcacgmm import class_weights
    rng = np.random.RandomState(T)
    for K in range(1, 7):
        m = rng.uniform(size=(4, K, T))
        m[:3, :, rng.uniform(size=T) < 0.1] = 0.     # zero frames, but no frame without weight in every bin
        m[:, :, 0] = rng.uniform(size=(4, K))        # and every bin keeps some weight
        bare = m.copy()
        bare[1] = 0.                                 # then a bin without weight: 0 / 0 in its per-bin weight
        for x in (m, bare):
            w = class_weights(_d(x), axes)
            with np.errstate(invalid='ignore'):
                ref = IO.class_weight(x.copy(), axes)
            if np.ndim(ref) == 0:
                assert w == ref
            else:
                nan = np.isnan(ref)
                np.testing.assert_array_equal(np.isnan(_h(w)), nan)
                _rows_close(np.where(nan, 0., _h(w)), np.where(nan, 0., ref), 1)


def _posterior(a, b, sa, sb, weight, mode, eps, inline):
    from pb_bss_b200 import _lib
    lib = _lib.load()
    F, K, T = a.shape
    out = torch.empty((F, K, T), dtype=torch.float64, device='cuda')
    chosen = torch.full((F, K), -1, dtype=torch.int32, device='cuda')
    ad, bd = _d(a), _d(b)
    wd = None if weight is None else _d(weight)
    _lib.check(lib.pbb_log_pdf_to_affiliation(
        ad.data_ptr(), bd.data_ptr(), sa, sb, None if wd is None else wd.data_ptr(), mode, None, eps, int(inline),
        F, K, T, out.data_ptr(), chosen.data_ptr(), torch.cuda.current_stream().cuda_stream),
        'pbb_log_pdf_to_affiliation')
    return _h(out), _h(chosen)


def _pairing_inputs(rng, F, K, T, weight, sa, sb):
    """Spatial / spectral log pdfs whose pairings differ clearly: the spectral classes are a shuffled, noisy copy of
    the spatial ones, redrawn until every bin's best pairing beats the second best by 1e-6 relative.  Ties are avoided
    on purpose: the device sums the auxiliary function in block order, the reference in NumPy's, so only a clear
    margin makes the choice well defined.  Returns (a, b, oracle affiliation, oracle choice)."""
    for _ in range(50):
        a = rng.randn(F, K, T) * 3.
        b = np.stack([a[f, rng.permutation(K)] for f in range(F)]) + rng.randn(F, K, T)
        ref, chosen, margin = IO.inline_pa_affiliation(weight[..., None], sa * a, sb * b, 1e-10)
        if margin.min() > 1e-6:
            return a, b, ref, chosen
    raise AssertionError('no input with a clear pairing')


@pytest.mark.parametrize('T', T_SWEEP)
@pytest.mark.parametrize('K', [4, 5, 6])
def test_inline_pairing_matches_oracle_argmax(K, T):
    from pb_bss_b200 import _lib
    rng = np.random.RandomState(K * 1000 + T)
    F = 5
    weight = rng.uniform(0.1, 1., size=(F, K))
    sa, sb = 0.7, 1.3
    a, b, ref, chosen = _pairing_inputs(rng, F, K, T, weight, sa, sb)
    out, got = _posterior(a, b, sa, sb, weight, _lib.WEIGHT_TIME, 1e-10, True)
    np.testing.assert_array_equal(got, chosen)
    _rows_close(out, ref, 2, rel=1e-10)


@pytest.mark.parametrize('T', T_SWEEP)
@pytest.mark.parametrize('axes', [(-1,), (-3,), (-3, -1), (-3, -2, -1)])
def test_posterior_weight_layouts_match_oracle(T, axes):
    from pb_bss_b200.distribution.gcacgmm import _weight_layout
    rng = np.random.RandomState(T + 7)
    mode = _weight_layout(axes)
    for K in range(1, 7):
        F = 3
        a, b = rng.randn(F, K, T) * 4, rng.randn(F, K, T) * 4
        m = rng.uniform(size=(F, K, T))
        weight = IO.class_weight(m, axes)
        for eps in (0., 1e-10):
            out, _ = _posterior(a, b, 0.6, 1.2, None if np.ndim(weight) == 0 else weight, mode, eps, False)
            ref = PO.log_pdf_to_affiliation(IO.unsqueeze(weight, axes), 0.6 * a + 1.2 * b, affiliation_eps=eps)
            _rows_close(out, ref, 2, rel=1e-10)


# ---------------------------------------------------------------- integrated models

def _oracle_model(model, spectral, covariance_type='spherical'):
    """Oracle model dict of a fitted device model."""
    d = dict(weight=np.asarray(model.weight), weight_constant_axis=model.weight_constant_axis,
             eigenvectors=model.cacg.covariance_eigenvectors, eigenvalues=model.cacg.covariance_eigenvalues,
             spatial_weight=model.spatial_weight, spectral_weight=model.spectral_weight)
    if spectral == 'vmf':
        d['spectral'] = dict(mean=model.vmf.mean, concentration=model.vmf.concentration)
    else:
        d['spectral'] = EO.gaussian_model(model.gaussian.mean, model.gaussian.covariance, covariance_type)
    return d


@pytest.mark.parametrize('T', T_SWEEP)
def test_integrated_posterior_matches_oracle(T):
    """GCACGMM.predict / VMFCACGMM.predict of a fitted device model against the oracle's E-step with the same
    parameters, T across the 256-thread block edges."""
    from pb_bss_b200.distribution import GCACGMMTrainer, VMFCACGMMTrainer
    F, D, E, K = 3, 4, 9, 3
    y, labels = synth.structured_stft(F, T, D, K, seed=T)
    rng = np.random.RandomState(T)
    emb = rng.randn(K, E)[labels] * 2 + 0.7 * rng.randn(F, T, E)
    init = synth.init_affiliation(F, K, T, seed=T)
    model = GCACGMMTrainer().fit(y, emb, initialization=init, iterations=2, covariance_type='diagonal',
                                 weight_constant_axis=(-3,))
    ref = IO.integrated_predict(y, emb, _oracle_model(model, 'gaussian', 'diagonal'))
    _rows_close(model.predict(y, emb), ref, 2, rel=1e-9)
    unit = EO._unit_rows(emb)
    model = VMFCACGMMTrainer().fit(y, unit, initialization=init, iterations=2, weight_constant_axis=(-3, -1))
    ref = IO.integrated_predict(y, unit, _oracle_model(model, 'vmf'))
    _rows_close(model.predict(y, unit), ref, 2, rel=1e-9)


def _check_model(model, g, name, spectral):
    np.testing.assert_allclose(np.asarray(model.weight), g[f'{name}_weight'], **MODEL)
    if spectral == 'vmf':
        np.testing.assert_allclose(model.vmf.mean, g[f'{name}_mean'], **MODEL)
        np.testing.assert_allclose(model.vmf.concentration, g[f'{name}_concentration'], **MODEL)
    else:
        np.testing.assert_allclose(model.gaussian.mean, g[f'{name}_mean'], **MODEL)
        np.testing.assert_allclose(model.gaussian.covariance, g[f'{name}_gcov'], **MODEL)
    np.testing.assert_allclose(model.cacg.covariance_eigenvalues, g[f'{name}_eigenvalues'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(model.cacg.covariance, g[f'{name}_covariance'], rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('name', list(CASES))
def test_integrated_fit_matches_reference_shape_sweep(name):
    from pb_bss_b200.distribution import GCACGMMTrainer, VMFCACGMMTrainer
    g = load_golden('integration_shapes')
    problem, spectral, kw = CASES[name]
    d = fixture_inputs(g, problem)
    emb = embedding_of(d, spectral)
    trainer = GCACGMMTrainer() if spectral == 'gaussian' else VMFCACGMMTrainer()
    model = trainer.fit(d['y'], emb, initialization=d['init'], iterations=int(g['iterations']), **resolve(d, kw))
    _check_model(model, g, name, spectral)
    aff = model.predict(d['y'], emb)
    np.testing.assert_allclose(aff, g[f'{name}_affiliation'], **AFF)


def test_constant_weight_axes_raise_like_the_reference():
    from pb_bss_b200.distribution import GCACGMMTrainer
    g = load_golden('integration_shapes')
    d = fixture_inputs(g, 'k2')
    for key, axes in ERROR_AXES.items():
        expected = str(g[key])
        try:
            GCACGMMTrainer().fit(d['y'], d['embedding'], initialization=d['init'], iterations=2,
                                 weight_constant_axis=axes)
            got = ''
        except IndexError:
            got = 'IndexError'
        assert got == expected, (axes, got, expected)


LARGE = {
    'gaussian_e64_k6': ('gaussian', (4, 1000, 6, 64, 6), dict(inline_permutation_alignment=True,
                                                             weight_constant_axis=(-3, -1))),
    'vmf_e33_k5': ('vmf', (5, 1000, 6, 33, 5), dict(inline_permutation_alignment=True, max_concentration=100)),
    'gaussian_diag_e23_k6': ('gaussian', (8, 600, 3, 23, 6), dict(covariance_type='diagonal',
                                                                  weight_constant_axis=(-3,))),
}


def _large_inputs(spectral, F, T, D, E, K):
    y, labels = synth.structured_stft(F, T, D, K, seed=E)
    rng = np.random.RandomState(E)
    emb = rng.randn(K, E)[labels] * 2 + 0.7 * rng.randn(F, T, E)
    if spectral == 'vmf':
        emb = EO._unit_rows(emb)
    return y, emb, synth.init_affiliation(F, K, T, seed=E + 1)


@pytest.mark.parametrize('name', list(LARGE))
def test_integrated_fit_matches_oracle_at_large_shapes(name):
    from pb_bss_b200.distribution import GCACGMMTrainer, VMFCACGMMTrainer
    spectral, shape, kw = LARGE[name]
    y, emb, init = _large_inputs(spectral, *shape)
    ref = IO.integrated_fit(y, emb, init, 3, spectral, **kw)
    if kw.get('inline_permutation_alignment'):
        assert ref['min_margin'] > 1e-6, ref['min_margin']
    trainer = GCACGMMTrainer() if spectral == 'gaussian' else VMFCACGMMTrainer()
    model = trainer.fit(y, emb, initialization=init, iterations=3, **kw)
    np.testing.assert_allclose(np.asarray(model.weight), np.asarray(ref['weight']), **MODEL)
    np.testing.assert_allclose(model.cacg.covariance_eigenvalues, ref['eigenvalues'], rtol=1e-6, atol=1e-9)
    if spectral == 'vmf':
        np.testing.assert_allclose(model.vmf.mean, ref['spectral']['mean'], **MODEL)
        np.testing.assert_allclose(model.vmf.concentration, ref['spectral']['concentration'], **MODEL)
    else:
        np.testing.assert_allclose(model.gaussian.mean, ref['spectral']['mean'], **MODEL)
        np.testing.assert_allclose(model.gaussian.covariance, ref['spectral']['covariance'], **MODEL)
    np.testing.assert_allclose(model.predict(y, emb), IO.integrated_predict(y, emb, ref), **AFF)


def test_integrated_fit_rejects_seven_classes():
    from pb_bss_b200.distribution import GCACGMMTrainer
    y, emb, _ = _large_inputs('gaussian', 2, 50, 3, 4, 3)
    with pytest.raises(ValueError, match='K <= 6'):
        GCACGMMTrainer().fit(y, emb, initialization=synth.init_affiliation(2, 7, 50), iterations=2)


# ---------------------------------------------------------------- GMM / VMFMM at large E

def _clouds(E, K=6, N=2000, B=2, seed=0):
    rng = np.random.RandomState(seed + E)
    centers = rng.randn(B, K, E) * 2.
    labels = rng.randint(0, K, size=(B, N))
    y = np.take_along_axis(centers, labels[..., None], axis=1) + rng.randn(B, N, E) * rng.uniform(0.5, 1., size=E)
    # a noisy copy of the labels: a random start lets full-covariance EM at large E collapse a class (singular)
    init = rng.uniform(size=(B, K, N)) + 2. * (labels[:, None, :] == np.arange(K)[:, None])
    return y, init / init.sum(-2, keepdims=True)


@pytest.mark.parametrize('E', [16, 33, 64])
def test_gmm_and_vmfmm_match_oracle_at_large_e(E):
    from pb_bss_b200.distribution import GMMTrainer, VMFMMTrainer
    y, init = _clouds(E)
    model = GMMTrainer().fit(y, initialization=init, iterations=5)
    ref = EO.gmm_fit(y, init, 5)
    np.testing.assert_allclose(np.asarray(model.weight), ref['weight'], **MODEL)
    np.testing.assert_allclose(model.gaussian.mean, ref['gaussian']['mean'], **MODEL)
    np.testing.assert_allclose(model.gaussian.covariance, ref['gaussian']['covariance'], **MODEL)
    np.testing.assert_allclose(model.predict(y), EO.gmm_predict(y, ref), **AFF)
    model = VMFMMTrainer().fit(y, initialization=init, iterations=5)
    ref = EO.vmfmm_fit(y, init, 5)
    np.testing.assert_allclose(np.asarray(model.weight), ref['weight'], **MODEL)
    np.testing.assert_allclose(model.vmf.mean, ref['mean'], **MODEL)
    np.testing.assert_allclose(model.vmf.concentration, ref['concentration'], **MODEL)
    np.testing.assert_allclose(model.predict(y), EO.vmfmm_predict(y, ref), **AFF)


def test_large_e_fit_is_bit_reproducible():
    from pb_bss_b200.distribution import GMMTrainer
    y, init = _clouds(64, N=5000, B=1, seed=9)
    a = GMMTrainer().fit(y, initialization=init, iterations=3)
    b = GMMTrainer().fit(y, initialization=init, iterations=3)
    np.testing.assert_array_equal(a.gaussian.covariance, b.gaussian.covariance)
    np.testing.assert_array_equal(a.predict(y), b.predict(y))
