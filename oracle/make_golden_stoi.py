"""Generate tests/golden/stoi.npz: the STOI numbers the reference publishes.

The reference checkout must be present (PB_BSS_REFERENCE, as for oracle/make_golden_bss_eval.py):

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_stoi [OUT_DIR]

pystoi is not a dependency, so nothing is recomputed by it here.  The signals the values belong to are those of
tests/golden/bss_eval.npz (input_*, output_* and doctest_*), so only the values are stored:
  - input / output: the ``k == 'stoi'`` branches of test_input_metrics and test_output_metrics in the reference's
    tests/test_evaluation/test_wrapper_values.py, read with ``ast``, with their rtol;
  - doctest: the 8-decimal ``'stoi': array([...])`` that the OutputMetrics doctest of pb_bss/evaluation/wrapper.py
    prints for ``metrics['stoi']``.
All three are at 8 kHz.
"""
import ast
import os
import re
import sys

import numpy as np

from . import build_ref
from . import make_golden_bss_eval
from . import make_golden_transform

OUT = make_golden_transform.OUT
SAMPLE_RATE = 8000


def _expected(test_name, key='stoi'):
    """(values, rtol) of the ``if k == key:`` branch of one test function of test_wrapper_values.py."""
    tree = ast.parse(open(make_golden_bss_eval._test_file()).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == test_name)
    for node in ast.walk(fn):
        if (isinstance(node, ast.If) and isinstance(node.test, ast.Compare)
                and isinstance(node.test.comparators[0], ast.Constant) and node.test.comparators[0].value == key):
            call = node.body[0].value
            assert call.func.attr == 'assert_allclose', ast.dump(call)
            rtol = [k.value for k in call.keywords if k.arg == 'rtol']
            return (np.array(ast.literal_eval(call.args[1]), dtype=np.float64),
                    float(ast.literal_eval(rtol[0])) if rtol else 1e-7)   # assert_allclose's default
    raise KeyError(test_name, key)


def _doctest(key='stoi'):
    """The full-precision values the OutputMetrics doctest prints for metrics[key], and their decimals."""
    path = os.path.join(build_ref.SRC, 'pb_bss', 'evaluation', 'wrapper.py')
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'OutputMetrics')
    init = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == '__init__')
    doc = ast.get_docstring(init)
    printed = re.findall(rf"'{key}': array\(\[([^\]]*)\]\)", doc)
    text = max(printed, key=len)                  # the pprint without printoptions(precision=4)
    values = [v.strip() for v in text.split(',')]
    return np.array([float(v) for v in values]), max(len(v.split('.')[1]) for v in values)


def make_stoi(out_dir=OUT):
    out = {'sample_rate': np.int64(SAMPLE_RATE)}
    out['input_stoi'], rtol = _expected('test_input_metrics')
    out['input_rtol'] = np.float64(rtol)
    out['output_stoi'], rtol = _expected('test_output_metrics')
    out['output_rtol'] = np.float64(rtol)
    out['doctest_stoi'], decimals = _doctest()
    out['doctest_decimals'] = np.int64(decimals)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'stoi.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_stoi(*sys.argv[1:]))
