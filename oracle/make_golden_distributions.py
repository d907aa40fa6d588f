"""Generate tests/golden/distributions.npz: the reference's single distributions of pb_bss.distribution --
ComplexAngularCentralGaussian (+ trainer), ComplexWatson (+ trainer), ComplexCircularSymmetricGaussian (+ trainer)
and the samplers -- on the cases of oracle/distributions_oracle.py.

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_distributions [OUT_DIR]

The unmodified reference is imported through oracle/ref_shim.py.  Inputs are regenerated from their seeds by
``distributions_oracle.case_input``, so only outputs are stored:
  - cACG models as their covariance V diag(lambda) V^H and eigenvalues (eigenvector phases are arbitrary); the model
    of the log-pdf cases as its eigenvectors and eigenvalues, so the port evaluates exactly that model;
  - the reference's TypeError for a batched fit next to its per-slice 2-D fits;
  - the Watson normalisers of every variant, D = 2..8, at kappa in KAPPAS.  NumPy 2 removed np.asfarray, which the
    reference's low / medium / high formulas call: the generator records that AttributeError, then provides
    np.asfarray as np.asarray(., float) -- the reference's source stays as it is;
  - sample values and the MT19937 state after each sampling call;
  - the exception type of every error case, and the names pb_bss.distribution exports.
The generator asserts that the NumPy restatement reproduces every case.
"""
import ast
import os
import sys
import warnings

import numpy as np

from . import distributions_oracle as DO
from . import ref_shim
from .make_golden_transform import OUT


def _state(out, key):
    s = np.random.get_state()
    out[f'{key}_state_keys'] = s[1]
    out[f'{key}_state_pos'] = np.int64(s[2])
    out[f'{key}_state_has_gauss'] = np.int64(s[3])
    out[f'{key}_state_gauss'] = np.float64(s[4])


def _error(fn):
    try:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            fn()
    except Exception as e:  # noqa: BLE001 -- the type is the record
        return type(e).__name__
    return 'none'


def _close(a, b, rtol=1e-10, atol=1e-12):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def exported_names():
    path = os.path.join(ref_shim.REF, 'pb_bss', 'distribution', '__init__.py')
    names = []
    for node in ast.parse(open(path).read()).body:
        if isinstance(node, ast.ImportFrom):
            names += [a.asname or a.name for a in node.names]
    return names


def main(out_dir=OUT):
    ref = ref_shim.load()
    dist = ref.distribution
    CACG, CACGT = dist.ComplexAngularCentralGaussian, dist.ComplexAngularCentralGaussianTrainer
    CW, CWT = dist.ComplexWatson, dist.ComplexWatsonTrainer
    CCSG, CCSGT = dist.ComplexCircularSymmetricGaussian, dist.ComplexCircularSymmetricGaussianTrainer
    out = {'names': np.array(exported_names())}

    # ---- from_covariance --------------------------------------------------------------------------------------------
    c = DO.case_input('cov')
    for tag, floor, norm in [('eig', 0.0, 'eigenvalue'), ('trace', 0.0, 'trace'), ('none', 0.0, False),
                             ('eig_floor', 1e-2, 'eigenvalue'), ('trace_floor', 1e-2, 'trace'),
                             ('none_floor', 1e-2, False)]:
        arg = c.copy()
        m = CACG.from_covariance(arg, eigenvalue_floor=floor, covariance_norm=norm)
        if norm == 'trace':
            assert not np.array_equal(arg, c), 'the reference divides the caller\'s covariance in place'
        V, lam = DO.cacg_from_covariance(c, floor, norm)
        _close(lam, m.covariance_eigenvalues)
        _close(DO.covariance(V, lam), m.covariance)
        out[f'cov_{tag}_cov'] = m.covariance
        out[f'cov_{tag}_lam'] = m.covariance_eigenvalues

    # ---- log_pdf / _log_pdf -----------------------------------------------------------------------------------------
    cov, y = DO.case_input('logpdf')
    m = CACG.from_covariance(cov)
    out['logpdf_V'], out['logpdf_lam'] = m.covariance_eigenvectors, m.covariance_eigenvalues
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        lp = m.log_pdf(y)
        z = ref.cacg.normalize_observation(y)
        lp2, q2 = m._log_pdf(z)
        lp64 = m.log_pdf(y.astype(np.complex64))
        lp0 = m.log_pdf(y[..., :0, :])
    ol, oq = DO.cacg_log_pdf(np.swapaxes(DO.unit_rows(y), -1, -2), m.covariance_eigenvectors,
                             m.covariance_eigenvalues)
    _close(ol, lp, rtol=1e-12)
    _close(oq, q2, rtol=1e-12)
    assert lp.shape == (3, 2, 50) and lp0.shape == (3, 2, 0), (lp.shape, lp0.shape)
    out.update(logpdf=lp, logpdf_swapped=lp2, logpdf_q=q2, logpdf_c64=lp64)

    # ---- trainer ------------------------------------------------------------------------------------------------------
    fits = [(D, 'eigenvalue', True) for D in DO.FIT_DIMS] + [(4, 'trace', True), (4, False, True),
                                                             (3, 'eigenvalue', False)]
    for D, norm, herm in fits:
        y = DO.case_input('fit', D)
        m = CACGT().fit(y, covariance_norm=norm, hermitize=herm)
        V, lam = DO.cacg_fit(y, norm=norm)
        _close(lam, m.covariance_eigenvalues, rtol=1e-9)
        _close(DO.covariance(V, lam), m.covariance, rtol=1e-9)
        key = f'fit_d{D}_{norm}_{int(herm)}'
        out[f'{key}_cov'], out[f'{key}_lam'] = m.covariance, m.covariance_eigenvalues
    y = DO.case_input('batch')
    out['batch_error'] = np.array(_error(lambda: CACGT().fit(y)))
    slices = [[CACGT().fit(y[i, j]) for j in range(y.shape[1])] for i in range(y.shape[0])]
    out['batch_cov'] = np.array([[s.covariance for s in row] for row in slices])
    out['batch_lam'] = np.array([[s.covariance_eigenvalues for s in row] for row in slices])
    z, q, sal = DO.case_input('step')
    for tag, s in (('none', None), ('sal', sal)):
        m = CACGT()._fit(z, s, q)
        V, lam = DO.cacg_step(z, q, s)
        _close(lam, m.covariance_eigenvalues)
        _close(DO.covariance(V, lam), m.covariance)
        out[f'step_{tag}_cov'], out[f'step_{tag}_lam'] = m.covariance, m.covariance_eigenvalues

    # ---- complex Watson ---------------------------------------------------------------------------------------------
    had_asfarray = hasattr(np, 'asfarray')
    out['lognorm_numpy2_error'] = np.array(_error(lambda: CW.log_norm_low_concentration(1.0, 3)))
    if not had_asfarray:
        np.asfarray = lambda a: np.asarray(a, dtype=float)
    try:
        for D in DO.NORM_DIMS:
            k = DO.kappas(D)
            for v in DO.VARIANTS:
                with warnings.catch_warnings():
                    warnings.simplefilter('ignore')
                    r = getattr(CW, f'log_norm_{v}' if v in ('1f1', 'tran_vu') else f'log_norm_{v}_concentration')(
                        k.copy(), D)
                    o = DO.cw_log_norm(v, k, D)
                fin = np.isfinite(r)
                if v == '1f1':
                    fin &= k < 700  # scipy's hyp1f1 overflows beyond
                tol = 1e-12 * np.abs(r[fin]) + DO.cw_log_norm_spread(v, k, D)[fin]
                assert np.all(np.abs(o[fin] - r[fin]) <= tol), (v, D, o, r)
                assert np.array_equal(np.isfinite(o), np.isfinite(r)) or v == '1f1', (v, D, o, r)
                out[f'lognorm_{v}_d{D}'] = np.asarray(r, dtype=np.float64)
    finally:
        if not had_asfarray:
            del np.asfarray
    mode, kappa, y = DO.case_input('watson')
    m = CW(mode=mode, concentration=kappa)
    out['watson_logpdf'], out['watson_pdf'] = m.log_pdf(y), m.pdf(y)
    _close(DO.cw_log_pdf(y, mode, kappa), out['watson_logpdf'], rtol=1e-12)
    for D in DO.FIT_DIMS:
        y, sal = DO.case_input('wfit', D)
        m = CWT().fit(y, saliency=sal)
        yn = y / np.linalg.norm(y, axis=-1, keepdims=True)
        m2 = CWT(D)._fit(yn, sal)
        assert np.allclose(np.abs(np.vdot(m.mode, m2.mode)), 1.0) and np.allclose(m.concentration, m2.concentration)
        out[f'wfit_d{D}_mode'], out[f'wfit_d{D}_kappa'] = m.mode, np.float64(m.concentration)
        m = CWT().fit(y)
        out[f'wfit_d{D}_nosal_mode'], out[f'wfit_d{D}_nosal_kappa'] = m.mode, np.float64(m.concentration)

    # ---- complex circular-symmetric Gaussian --------------------------------------------------------------------
    herm, nonherm, classes, y, yreal = DO.case_input('ccsg')
    for tag, cov, obs in (('herm', herm, y), ('nonherm', nonherm, y), ('classes', classes, y),
                          ('real', herm, yreal)):
        r = CCSG(covariance=cov).log_pdf(obs)
        _close(DO.ccsg_log_pdf(obs, cov), r, rtol=1e-12)
        out[f'ccsg_{tag}'] = r
    y, sal = DO.case_input('ccsg_fit')
    for tag, s in (('none', None), ('sal', sal)):
        r = CCSGT().fit(y, saliency=s).covariance
        _close(DO.ccsg_fit(y, s), r, rtol=1e-12)
        out[f'ccsg_fit_{tag}'] = r

    # ---- samplers -----------------------------------------------------------------------------------------------
    cov3, covK, weight = DO.sample_inputs()
    calls = {
        'ccsg': (lambda: CCSG(covariance=cov3).sample((7,)), lambda: DO.ccsg_sample((7,), cov3)),
        'ccsg_empty': (lambda: CCSG(covariance=cov3).sample((0,)), lambda: DO.ccsg_sample((0,), cov3)),
        'cacg': (lambda: CACG.from_covariance(cov3).sample((5,)),
                 lambda: DO.ccsg_sample((5,), DO.covariance(*DO.cacg_from_covariance(cov3)), True)),
        'cacg_fn': (lambda: ref.cacg.sample_complex_angular_central_gaussian((6,), cov3),
                    lambda: DO.ccsg_sample((6,), cov3, True)),
    }
    for key, (fn, oracle) in calls.items():
        np.random.seed(DO.SAMPLE_SEED)
        x = fn()
        _state(out, f'sample_{key}')
        np.random.seed(DO.SAMPLE_SEED)
        _close(oracle(), x, rtol=1e-13, atol=1e-14)
        out[f'sample_{key}'] = x
    np.random.seed(DO.SAMPLE_SEED)
    x, labels = dist.sample_cacgmm(20, weight, covK, return_label=True)
    _state(out, 'sample_cacgmm')
    assert not np.any(labels == 1), 'the class of weight 0 draws no sample'
    np.random.seed(DO.SAMPLE_SEED)
    ox, ol = DO.sample_cacgmm(20, weight, covK)
    assert np.array_equal(ol, labels)
    _close(ox, x, rtol=1e-13, atol=1e-14)
    out['sample_cacgmm'], out['sample_cacgmm_labels'] = x, labels.astype(np.int8)

    # ---- error types ------------------------------------------------------------------------------------------------
    yf = DO.case_input('fit', 4)
    errors = {
        'from_covariance_norm': lambda: CACG.from_covariance(c.copy(), covariance_norm='frobenius'),
        'from_covariance_nonfinite': lambda: CACG.from_covariance(np.full((3, 3), np.inf + 0j)),
        'cacg_fit_saliency': lambda: CACGT().fit(yf, saliency=np.ones(yf.shape[0])),
        'cacg_fit_real': lambda: CACGT().fit(yf.real),
        'cacg_fit_d1': lambda: CACGT().fit(yf[:, :1]),
        'cacg_step_real': lambda: CACGT()._fit(z.real, None, q),
        'ccsg_singular': lambda: CCSG(covariance=np.zeros((4, 4), complex)).log_pdf(y[0, :, :3].repeat(2, -1)[..., :4]),
        'ccsg_sample_ndim': lambda: CCSG(covariance=classes).sample((3,)),
        'ccsg_sample_int': lambda: CCSG(covariance=herm).sample(3),
        'ccsg_sample_2d': lambda: CCSG(covariance=herm).sample((2, 3)),
        'ccsg_sample_not_pd': lambda: CCSG(covariance=-herm).sample((3,)),
        'ccsg_fit_type': lambda: CCSGT().fit(y, covariance_type='diagonal'),
        'ccsg_fit_real': lambda: CCSGT().fit(y.real),
        'cw_fit_real': lambda: CWT().fit(yf.real),
        'cw_fit_dim': lambda: CWT(3).fit(yf),
        'sample_cacgmm_size': lambda: dist.sample_cacgmm((3,), weight, covK),
        'sample_cacgmm_weight': lambda: dist.sample_cacgmm(3, weight[None], covK),
        'sample_cacgmm_cov': lambda: dist.sample_cacgmm(3, weight, covK[0]),
    }
    for key, fn in errors.items():
        out[f'error_{key}'] = np.array(_error(fn))
        print(f'{key}: {out[f"error_{key}"]}')
    path = os.path.join(out_dir, 'distributions.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
