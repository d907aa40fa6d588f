"""Generate tests/golden/bss_eval.npz: the mir_eval numbers the reference publishes, with the signals they belong to.

The reference checkout must be present (PB_BSS_REFERENCE, as for oracle/make_golden_srmr.py):

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_bss_eval [OUT_DIR]

mir_eval is not a dependency, so nothing is recomputed by it here.  Instead:
  - ``scenario()`` of the reference's tests/test_evaluation/test_wrapper_values.py builds the signals of
    test_input_metrics and test_output_metrics (its import of pb_bss.evaluation.wrapper and einops is satisfied by
    stub modules), and the expected mir_eval_* values are read with ``ast`` out of that file's assert_allclose calls;
  - the OutputMetrics doctest of pb_bss/evaluation/wrapper.py gives its signals and its printed mir_eval_* values
    (4 decimals).
Only arrays are stored: the signals, the values and each anchor's rtol.  test_input_metrics's signals are stored once
(speech_source and observation); ``input_signals`` builds the (K, channels, T) arrays InputMetrics passes.
"""
import ast
import importlib.util
import os
import re
import sys
import types

import numpy as np

from . import build_ref
from . import make_golden_transform

OUT = make_golden_transform.OUT


def _test_file():
    return os.path.join(build_ref.SRC, 'tests', 'test_evaluation', 'test_wrapper_values.py')


def _scenario():
    """scenario() of the reference's test_wrapper_values.py, imported with stub modules."""
    saved = {k: sys.modules.get(k) for k in ('pb_bss', 'pb_bss.evaluation', 'pb_bss.evaluation.wrapper', 'einops')}
    try:
        for name in ('pb_bss', 'pb_bss.evaluation'):
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
        wrapper = types.ModuleType('pb_bss.evaluation.wrapper')
        wrapper.InputMetrics = wrapper.OutputMetrics = None
        sys.modules['pb_bss.evaluation.wrapper'] = wrapper
        einops = types.ModuleType('einops')
        einops.rearrange = None
        sys.modules['einops'] = einops
        spec = importlib.util.spec_from_file_location('_reference_test_wrapper_values', _test_file())
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod.scenario()
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _expected(test_name):
    """{'sdr': array, ..., 'rtol': float} from the `if k == 'mir_eval_*':` branches of one test function."""
    tree = ast.parse(open(_test_file()).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == test_name)
    out = {}
    for node in ast.walk(fn):
        if not (isinstance(node, ast.If) and isinstance(node.test, ast.Compare)):
            continue
        key = node.test.comparators[0]
        if not (isinstance(key, ast.Constant) and str(key.value).startswith('mir_eval_')):
            continue
        name = key.value[len('mir_eval_'):]
        stmt = node.body[0]
        if name == 'selection':   # assert all(v == [0, 1])
            out[name] = np.array(ast.literal_eval(stmt.test.args[0].comparators[0]), dtype=np.int64)
            continue
        call = stmt.value
        assert call.func.attr == 'assert_allclose', ast.dump(call)
        out[name] = np.array(ast.literal_eval(call.args[1]), dtype=np.float64)
        rtol = [k.value for k in call.keywords if k.arg == 'rtol']
        out['rtol'] = float(ast.literal_eval(rtol[0])) if rtol else 1e-7   # assert_allclose's default
    return out


def _doctest():
    """Signals and printed mir_eval_* values of the OutputMetrics doctest (pb_bss/evaluation/wrapper.py)."""
    path = os.path.join(build_ref.SRC, 'pb_bss', 'evaluation', 'wrapper.py')
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'OutputMetrics')
    init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == '__init__')
    doc = ast.get_docstring(init)
    call = re.search(r'OutputMetrics\(\s*(.*?)\n\s*\.\.\.\s*\)', doc, re.S).group(1)
    call = re.sub(r'(^|\n)\s*\.\.\.\s*', ' ', call)
    kw = ast.parse(f'f({call})', mode='eval').body.keywords
    signals = {}
    for k in kw:
        if k.arg in ('speech_prediction', 'speech_source'):
            rows = []
            for row in k.value.args[0].elts:        # [a, b, ...] * n
                rows.append(np.array(ast.literal_eval(row.left) * ast.literal_eval(row.right), dtype=np.float64))
            signals[k.arg] = np.stack(rows)
    values = {}
    for name in ('sdr', 'sir', 'sar', 'selection'):
        m = re.search(rf"'mir_eval_{name}': array\(\[([^\]]*)\]\)", doc)
        values[name] = np.array([float(v) for v in m.group(1).split(',')])
    values['selection'] = values['selection'].astype(np.int64)
    return signals, values


def input_signals(g):
    """reference (K, D, T) and estimation (K, D, T) of test_input_metrics, as InputMetrics.mir_eval builds them: every
    channel's reference is the source, every source's estimate is the observation."""
    source, obs = g['input_source'], g['input_observation']
    K, (D, T) = source.shape[0], obs.shape
    return (np.ascontiguousarray(np.broadcast_to(source[:, None], (K, D, T))),
            np.ascontiguousarray(np.broadcast_to(obs[None], (K, D, T))))


def make_bss_eval(out_dir=OUT):
    ex = _scenario()
    out = {}
    # test_input_metrics: InputMetrics.mir_eval, references (sources, channels, T) and the observation per source
    out['input_source'], out['input_observation'] = ex['speech_source'], ex['observation']
    e = _expected('test_input_metrics')
    for name in ('sdr', 'sir', 'sar'):
        out['input_' + name] = e[name]
    out['input_rtol'] = np.float64(e['rtol'])
    # test_output_metrics: OutputMetrics.mir_eval with compute_permutation
    out['output_reference'] = ex['speech_source']
    out['output_estimation'] = ex['speech_image'][..., 0, :] + ex['noise_image'][..., 0, :]
    e = _expected('test_output_metrics')
    for name in ('sdr', 'sir', 'sar', 'selection'):
        out['output_' + name] = e[name]
    out['output_rtol'] = np.float64(e['rtol'])
    signals, values = _doctest()
    out['doctest_reference'] = signals['speech_source']
    out['doctest_estimation'] = signals['speech_prediction']
    for name, v in values.items():
        out['doctest_' + name] = v
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'bss_eval.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_bss_eval(*sys.argv[1:]))
