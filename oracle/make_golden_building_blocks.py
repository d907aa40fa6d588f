"""Generate tests/golden/building_blocks.npz: the reference's building blocks -- the public functions of
pb_bss.distribution.mixture_model_utils and pb_bss.distribution.utils, pb_bss.utils (labels_to_one_hot, get_pca,
abs_square) and sxr_module.get_energy / set_snr -- on the seeded cases of oracle/building_blocks_oracle.py.

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_building_blocks [OUT_DIR]

The unmodified reference is imported through oracle/ref_shim.py (its evaluation/sxr_module.py is loaded from the
checkout as oracle/make_golden_metrics.py does).  Inputs are regenerated from their seeds, so only outputs are
stored, plus the exception type of every error case and, as ``names__<module>``, the public module-level names of
every module of the reference, read with ``ast`` from its sources.  The generator asserts that the NumPy restatement
reproduces every case; affiliation outputs larger than ``STORE_MAX`` elements (K = 16 and 64 with leading dims)
are checked here but not stored -- the tests hold the device to the restatement there.
"""
import ast
import os
import sys
import warnings

import numpy as np

from . import building_blocks_oracle as BO
from . import build_ref, ref_shim
from .make_golden_metrics import _load
from .make_golden_transform import OUT


def _error(fn):
    try:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            fn()
    except Exception as e:  # noqa: BLE001 -- the type is the record
        return type(e).__name__
    return 'none'


def public_names(path):
    """The public module-level names a module defines (functions, classes, assignments) and, for a package's
    ``__init__.py``, the names it imports."""
    names = []
    for node in ast.parse(open(path).read()).body:
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef, ast.ClassDef)):
            names.append(node.name)
        elif isinstance(node, ast.Assign):
            names += [t.id for t in node.targets if isinstance(t, ast.Name)]
        elif isinstance(node, ast.AnnAssign) and isinstance(node.target, ast.Name):
            names.append(node.target.id)
        elif isinstance(node, ast.ImportFrom) and os.path.basename(path) == '__init__.py':
            names += [a.asname or a.name for a in node.names if a.name != '*']
    return [n for n in names if not n.startswith('_')]


def module_names(root):
    out = {}
    for d, dirs, files in os.walk(os.path.join(root, 'pb_bss')):
        dirs[:] = sorted(x for x in dirs if x != '__pycache__')
        for f in sorted(files):
            if f.endswith('.py'):
                rel = os.path.relpath(os.path.join(d, f), root)[:-3].replace(os.sep, '.')
                out[rel[:-len('.__init__')] if rel.endswith('.__init__') else rel] = public_names(os.path.join(d, f))
    return out


def _close(a, b, rtol=1e-12, atol=1e-300):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def main(out_dir=OUT):
    ref = ref_shim.load()
    mmu = ref.mixture_model_utils
    import pb_bss.distribution.utils as dutils
    import pb_bss.utils as putils
    sxr = _load('sxr_module')
    out = {}
    for mod, names in module_names(build_ref.SRC).items():
        out['names__' + mod] = np.array(names, dtype=str)

    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        for case in BO.AFF_CASES:
            w, lp, m, eps = BO.aff_input(case)
            r = mmu.log_pdf_to_affiliation(w, lp, m, eps)
            assert r.dtype == lp.dtype
            rtol = 1e-6 if lp.dtype == np.float32 else 1e-12
            _close(BO.log_pdf_to_affiliation(w, lp, m, eps), r, rtol=rtol, atol=1e-300 if rtol < 1e-7 else 1e-7)
            if r.size <= BO.STORE_MAX:
                out[case[0]] = r
        for tag, kind in BO.AFF_ERRORS:
            w, lp, m = BO.aff_error_input(kind)
            out[tag] = np.array(_error(lambda: mmu.log_pdf_to_affiliation(w, lp, m)))
        for tag, K in BO.INT_CASES:
            w, a, b = BO.int_input(K)
            r = mmu.log_pdf_to_affiliation_for_integration_models_with_inline_pa(w, a, b)
            _close(BO.integration_affiliation(w, a, b), r)
            out[tag] = r
        for tag, ax, s in BO.EMW_CASES:
            aff, sal = BO.emw_input(s)
            r = mmu.estimate_mixture_weight(aff, sal, ax)
            _close(BO.estimate_mixture_weight(aff, sal, ax), r, atol=1e-15)
            out[tag] = r
        doc = [[0.4, 1, 0.4], [0.6, 0, 0.6]]
        for i, (a, ax) in enumerate([(doc, -1), (doc, -2), ([doc, doc], -1), ([doc, doc], -2), ([doc, doc], -3)]):
            out[f'emw_doc{i}'] = mmu.estimate_mixture_weight(a, weight_constant_axis=ax)
        for tag, ordv, st, dt in BO.UNIT_CASES:
            x = BO.unit_input(dt)
            r = dutils._unit_norm(x, axis=-1, eps_style=st, ord=ordv)
            _close(BO.unit_norm(x, -1, 1e-4, st, ordv), r, rtol=1e-5 if dt == 'float32' else 1e-12, atol=1e-300)
            out[tag] = r
        sig = np.array([[1, 1], [1e-20, 1e-20], [0, 0]])
        for st in ('plus', 'max', 'where'):
            out[f'un_doc_{st}'] = dutils._unit_norm(sig, eps_style=st)
        out['un_err_style'] = np.array(_error(lambda: dutils._unit_norm(sig, eps_style='other')))
        out['fh'] = dutils.force_hermitian(BO.hermitian_input())
        A = np.array([[1 + 2j, 3 + 5j], [7 + 11j, 13 + 17j]])
        out['fh_doc'] = dutils.force_hermitian(A)
        out['fh_real'] = dutils.force_hermitian(BO.hermitian_input().real)
        _close(BO.force_hermitian(BO.hermitian_input()), out['fh'])
        for tag, lab, C, ax, kd, dt in BO.ONE_HOT_CASES:
            r = putils.labels_to_one_hot(lab, C, axis=ax, keepdims=kd, dtype=np.dtype(dt))
            np.testing.assert_array_equal(BO.labels_to_one_hot(lab, C, ax, kd, np.dtype(dt)), r)
            out[tag] = r
        for tag, lab, C, ax, kd in BO.ONE_HOT_ERRORS:
            out[tag] = np.array(_error(lambda: putils.labels_to_one_hot(lab, C, axis=ax, keepdims=kd)))
        P = BO.pca_input()
        for sc in (False, True):
            vec, val = putils.get_pca(P, use_scipy=sc)
            out[f'pca_vec_{int(sc)}'], out[f'pca_val_{int(sc)}'] = vec, val
        rr = BO.rng('abs')
        for dt in ('complex128', 'complex64', 'float64', 'float32'):
            x = rr.normal(size=(7, 9)) + (1j * rr.normal(size=(7, 9)) if dt.startswith('complex') else 0)
            out[f'abs_{dt}'] = putils.abs_square(x.astype(dt))
        X, N = BO.snr_input()
        Xc = X + 1j * N[::-1]
        for tag, ax, kd in [('all', None, False), ('ax1', -1, False), ('ax01k', (0, 1), True)]:
            out[f'energy_{tag}'] = sxr.get_energy(Xc, axis=ax, keepdims=kd)
            _close(BO.get_energy(Xc, ax, kd), out[f'energy_{tag}'])
        for tag, ax in [('none', None), ('ax', -1)]:
            Nc = N.copy()
            sxr.set_snr(X, Nc, 5.0, axis=ax)
            out[f'snr_inplace_{tag}'] = Nc
            _close(N * BO.set_snr_factor(X, N, 5.0, ax), Nc)
            out[f'snr_copy_{tag}'] = sxr.set_snr(X, N, 5.0, axis=ax, inplace=False)[1]
        out['snr_err_int'] = np.array(_error(lambda: sxr.set_snr(X, np.ones((2, 3, 50), np.int64), 5.0)))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'building_blocks.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)')


if __name__ == '__main__':
    main(*sys.argv[1:])
