"""Generate tests/golden/metrics.npz: SI-SDR and the invasive SxR as the reference computes them, and the wrapper
anchors it publishes.

The reference checkout must be present (PB_BSS_REFERENCE, as for oracle/make_golden_bss_eval.py):

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_metrics [OUT_DIR]

The unmodified pb_bss/evaluation/module_si_sdr.py and sxr_module.py of the checkout are loaded with
spec_from_file_location (they import only NumPy, SciPy and the standard library) and run on:
  - sisdr_*: the doctest cases of module_si_sdr.py (np.random.seed(0), randn(100)), including inf, inf and nan;
  - sxr_*: seeded versions of the cases of tests/test_evaluation/test_sxr.py, random shapes with K = 1..9 and D up to
    29, K_target = K_source and K_source + 1, and ties (zero contributions give equal mutual powers).  Each case
    stores its signals, the powers S and N, and sdr / sir / snr for every average flag; output cases also store the
    selection, the first maximiser of the mutual power in itertools order, as output_sxr picks it;
  - snr_*: get_snr over several axis and keepdims choices;
  - wrapper_taps (2, 3, 4): the room impulse responses of the test_wrapper_values.py scenario.  Its sources and
    observation are in bss_eval.npz; ``wrapper_images`` rebuilds the speech and noise images from the three;
  - anchor_*: the published invasive_* and srmr values of test_input_metrics / test_output_metrics, read with ``ast``,
    each with its rtol.
Only arrays are stored.
"""
import ast
import importlib.util
import itertools
import os
import sys

import numpy as np
import scipy.signal

from . import build_ref
from . import make_golden_bss_eval
from . import make_golden_transform

OUT = make_golden_transform.OUT
INPUT_SHAPES = ((1, 1), (1, 3), (2, 1), (2, 6), (3, 4), (4, 29), (7, 2), (8, 1), (8, 8), (9, 1), (9, 29))
OUTPUT_SHAPES = ((1, 1), (1, 2), (2, 2), (2, 3), (3, 3), (3, 4), (5, 5), (5, 6), (7, 7), (7, 8), (8, 8), (8, 9),
                 (9, 9))
SNR_AXES = ((None, False), (None, True), (0, False), (-1, False), (-1, True), ((0, 2), False), ((0, 2), True),
            ((1,), False))


def wrapper_images(source, observation, taps):
    """speech_image (K, D, T) and noise_image (D, T) of the test_wrapper_values.py scenario: each source convolved with
    its taps (``fftconvolve(..., mode='same')``), and the observation less the images.  The noise is the scenario's
    to within rounding of the observation (1e-16 of it), far below the published anchors' tolerances."""
    images = np.array([[scipy.signal.fftconvolve(s, h, mode='same') for h in hk] for s, hk in zip(source, taps)])
    noise = observation
    for image in images:
        noise = noise - image
    return images, noise


def _scenario_taps(ex):
    """The scenario's taps: its np.random.seed(1) stream after the two 10000-sample sources, checked against its
    images bit for bit."""
    rs = np.random.RandomState(1)
    rs.random_sample(2 * ex['speech_source'].shape[1])
    K, D = ex['speech_image'].shape[:2]
    taps = rs.random_sample((K, D, 4))
    images, noise = wrapper_images(ex['speech_source'], ex['observation'], taps)
    np.testing.assert_array_equal(images, ex['speech_image'])
    np.testing.assert_allclose(noise, ex['noise_image'], rtol=0, atol=1e-15)
    return taps


def _load(name):
    path = os.path.join(build_ref.SRC, 'pb_bss', 'evaluation', name + '.py')
    spec = importlib.util.spec_from_file_location('_reference_' + name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _selection(sxr, contribution):
    """The selection output_sxr makes (sxr_module.py:217-237), from the reference's own powers."""
    S = sxr.get_variance_for_zero_mean_signal(contribution, axis=-1)
    Ks, Kt = S.shape
    perms = np.array(list(itertools.permutations(range(Kt), r=Ks)))
    mutual = np.array([np.sum([S[k, p[k]] for k in range(Ks)]) for p in perms])
    return perms[np.argmax(mutual)].astype(np.int64)


def _anchors(out):
    tree = ast.parse(open(make_golden_bss_eval._test_file()).read())
    for test, prefix in (('test_input_metrics', 'input'), ('test_output_metrics', 'output')):
        fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == test)
        for node in ast.walk(fn):
            if not (isinstance(node, ast.If) and isinstance(node.test, ast.Compare)):
                continue
            key = node.test.comparators[0]
            if not (isinstance(key, ast.Constant) and key.value in ('invasive_sdr', 'invasive_sir', 'invasive_snr',
                                                                    'srmr')):
                continue
            call = node.body[0].value
            assert call.func.attr == 'assert_allclose', ast.dump(call)
            value = call.args[1]
            if isinstance(value, ast.Attribute):          # np.inf
                value = np.inf
            else:
                value = ast.literal_eval(value)
            rtol = [k.value for k in call.keywords if k.arg == 'rtol']
            out[f'anchor_{prefix}_{key.value}'] = np.array(value, dtype=np.float64)
            out[f'anchor_{prefix}_{key.value}_rtol'] = np.float64(ast.literal_eval(rtol[0]) if rtol else 1e-7)


def _input_case(out, sxr, name, images, noise):
    out[name + '_images'], out[name + '_noise'] = images, noise
    out[name + '_S'] = sxr.get_variance_for_zero_mean_signal(images, axis=-1)
    out[name + '_N'] = sxr.get_variance_for_zero_mean_signal(noise, axis=-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        for avg_s, avg_c in itertools.product((False, True), repeat=2):
            r = sxr.input_sxr(images, noise, average_sources=avg_s, average_channels=avg_c)
            for key, v in zip(('sdr', 'sir', 'snr'), r):
                out[f'{name}_{key}_{int(avg_s)}{int(avg_c)}'] = np.asarray(v, dtype=np.float64)


def _output_case(out, sxr, name, contribution, noise):
    out[name + '_contribution'], out[name + '_noise'] = contribution, noise
    out[name + '_S'] = sxr.get_variance_for_zero_mean_signal(contribution, axis=-1)
    out[name + '_N'] = sxr.get_variance_for_zero_mean_signal(noise, axis=-1)
    out[name + '_selection'] = _selection(sxr, contribution)
    with np.errstate(divide='ignore', invalid='ignore'):
        for avg in (False, True):
            r = sxr.output_sxr(contribution, noise, average_sources=avg)
            for key, v in zip(('sdr', 'sir', 'snr'), r):
                out[f'{name}_{key}_{int(avg)}'] = np.asarray(v, dtype=np.float64)


def make_metrics(out_dir=OUT):
    si = _load('module_si_sdr')
    sxr = _load('sxr_module')
    out = {}
    # the doctest of module_si_sdr.py
    np.random.seed(0)
    reference = np.random.randn(100)
    cases = [(reference, reference), (reference, reference * 2), (reference, np.flip(reference)),
             (reference, reference + np.flip(reference)), (reference, reference + 0.5),
             (reference, reference * 2 + 1), (np.array([1., 0]), np.array([0., 0])),
             (np.array([reference, reference]), np.array([reference * 2 + 1, reference * 1 + 0.5]))]
    with np.errstate(divide='ignore', invalid='ignore'):
        for i, (r, e) in enumerate(cases):
            out[f'sisdr_{i}_reference'], out[f'sisdr_{i}_estimation'] = r, e
            out[f'sisdr_{i}_value'] = np.asarray(si.si_sdr(r, e), dtype=np.float64)
    # test_sxr.py's cases, seeded, at 256 instead of 8000 / 10000 samples to keep the file small
    rng = np.random.default_rng(0)
    L = 256
    s1, s2, n = (rng.standard_normal(L) for _ in range(3))
    s1, s2, n = (v / np.sqrt(np.mean(v ** 2)) for v in (s1, s2, n))
    z = 0 * n
    _input_case(out, sxr, 'sxr_in_unit', 10 * np.stack((s1, s2))[:, None], n[None])
    _output_case(out, sxr, 'sxr_out_inf', np.array([[s1, 0 * s2, z], [0 * s1, s2, z]]), np.array([z, z, n]))
    _output_case(out, sxr, 'sxr_out_more', np.array([[10 * s1, s2, z], [0 * s1, 10 * s2, z]]),
                 np.array([10 * n, z, z]))
    _output_case(out, sxr, 'sxr_out_square', np.array([[10 * s1, s2], [0 * s1, 10 * s2]]), np.array([10 * n, z]))
    x = rng.normal(0, 1, (1, 1, L))
    _input_case(out, sxr, 'sxr_in_single', x, 10 ** (-10 / 20) * rng.normal(0, 1, (1, L)))
    _output_case(out, sxr, 'sxr_out_single', x, 10 ** (-10 / 20) * rng.normal(0, 1, (1, L)))
    x = rng.normal(0, 1, (2, 1, L))
    x[0, 0, :] *= 10 ** (10 / 20)
    _input_case(out, sxr, 'sxr_in_no_noise', x, np.zeros((1, L)))
    x = rng.normal(0, 1, (2, 2, L))
    x[0, 1, :] = 10 ** (-20 / 20) * x[0, 0, :]
    x[1, 1, :] = x[0, 1, :]
    x[1, 0, :] = 10 ** (-20 / 20) * x[0, 1, :]
    _output_case(out, sxr, 'sxr_out_equal_no_noise', x, np.zeros((2, L)))
    # random shapes: powers spread over six decades
    T = 8
    for K, D in INPUT_SHAPES:
        scale = 10.0 ** rng.uniform(-3, 3, (K, D, 1))
        _input_case(out, sxr, f'sxr_in_k{K}_d{D}', rng.standard_normal((K, D, T)) * scale,
                    rng.standard_normal((D, T)) * 10.0 ** rng.uniform(-3, 3, (D, 1)))
    for Ks, Kt in OUTPUT_SHAPES:
        scale = 10.0 ** rng.uniform(-3, 3, (Ks, Kt, 1))
        _output_case(out, sxr, f'sxr_out_k{Ks}_t{Kt}', rng.standard_normal((Ks, Kt, T)) * scale,
                     rng.standard_normal((Kt, T)) * 10.0 ** rng.uniform(-3, 3, (Kt, 1)))
    # ties: all-zero contributions (every selection has mutual power 0), and equal columns
    _output_case(out, sxr, 'sxr_out_tie_zero', np.zeros((3, 4, T)), rng.standard_normal((4, T)))
    c = rng.standard_normal((3, 1, T))
    _output_case(out, sxr, 'sxr_out_tie_columns', np.repeat(c, 4, axis=1), rng.standard_normal((4, T)))
    c = np.zeros((4, 5, T))
    c[0, 1] = c[1, 3] = c[2, 0] = rng.standard_normal(T)
    _output_case(out, sxr, 'sxr_out_tie_partial', c, rng.standard_normal((5, T)))
    # get_snr
    X, N = rng.standard_normal((3, 4, 50)), 0.1 * rng.standard_normal((3, 4, 50))
    out['snr_X'], out['snr_N'] = X, N
    for i, (axis, keepdims) in enumerate(SNR_AXES):
        out[f'snr_{i}_value'] = np.asarray(sxr.get_snr(X, N, axis=axis, keepdims=keepdims), dtype=np.float64)
    # the wrapper scenario's taps, and the published anchors
    out['wrapper_taps'] = _scenario_taps(make_golden_bss_eval._scenario())
    _anchors(out)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'metrics.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_metrics(*sys.argv[1:]))
