"""Generate tests/golden/gammatone.npz: the UNMODIFIED reference pb_bss/transform/gammatone.py on seeded signals.

pb_bss/transform is not part of the hot-path copy under oracle/_ref, so it is imported from the reference checkout
(PB_BSS_REFERENCE) as oracle/make_golden_transform.py does, which must be present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_gammatone [OUT_DIR]

Cases: sample rates 8000, 16000, 44100 and 48000; n = 1, 2, 23 and 64; default and explicit low / high
frequencies; 1-D, 2-D and 3-D signals; float32 and integer input.  Stored per case: the signal, the outputs stacked
to (n, *shape), the centre frequencies and the reference's coefficient arrays.  The coefficients alone are stored for
every (sample rate, n) pair, and the exception types of calculate_cfs for invalid n.
"""
import importlib
import os
import sys

import numpy as np

from . import make_golden_transform
from . import ref_shim

OUT = make_golden_transform.OUT
# name: sample_rate, n, low_freq, high_freq, shape, dtype
CASES = {
    'sr16k_n23': (16000, 23, 125, 0, (1200,), 'float64'),
    'sr8k_n2_2d': (8000, 2, 125, 0, (2, 600), 'float64'),
    'sr44k_n1_3d_band': (44100, 1, 50, 8000, (2, 3, 200), 'float64'),
    'sr48k_n64': (48000, 64, 125, 0, (300,), 'float64'),
    'sr16k_n4_f32_band': (16000, 4, 300, 5000, (3, 400), 'float32'),
    'sr16k_n2_int16': (16000, 2, 125, 0, (500,), 'int16'),
    'sr48k_n23_2d_band': (48000, 23, 80, 20000, (2, 600), 'float64'),
}


def _reference():
    ref_shim.load()
    make_golden_transform._add_reference_checkout()
    make_golden_transform._register_nara_wpe_stub()   # pb_bss/transform/__init__ imports the Griffin-Lim module
    return importlib.import_module('pb_bss.transform.gammatone')


def make_gammatone(out_dir=OUT):
    G = _reference()
    rng = np.random.RandomState(35)
    out = {}
    for name, (sr, n, lo, hi, shape, dtype) in CASES.items():
        if dtype == 'int16':
            x = rng.randint(-3000, 3000, size=shape).astype(np.int16)
        else:
            x = rng.randn(*shape).astype(dtype)
        y = G.gammatone_filterbank(x, sr, n, lo, hi)
        assert len(y) == n and all(v.dtype == np.float64 and v.shape == x.shape for v in y)
        cfs = G.calculate_cfs(lo, hi or sr / 2, n)
        out[name + '_x'], out[name + '_y'], out[name + '_cfs'] = x, np.stack(y), cfs
        out[name + '_params'] = np.array([sr, n, lo, hi], dtype=np.float64)
    for sr in (8000, 16000, 44100, 48000):
        for n in (1, 2, 23, 64):
            for lo, hi in ((125, sr / 2), (100, 6000)):
                key = f'coef_{sr}_{n}_{lo}_{int(hi)}'
                cfs = G.calculate_cfs(lo, hi, n)
                c = G._calculate_coefficients(cfs, sr, n)
                out[key + '_cfs'] = cfs
                out[key + '_A0_A2_B0'] = np.array([c[0], c[5], c[6]], dtype=np.float64)
                for cname, v in zip(('A11', 'A12', 'A13', 'A14'), c[1:5]):
                    out[f'{key}_{cname}'] = v
                out[key + '_B1'], out[key + '_B2'], out[key + '_gain'] = c[7], c[8], c[9]
    for label, n in (('zero', 0), ('negative', -1), ('float', 2.5)):
        try:
            G.calculate_cfs(125, 8000, n)
            out['error_' + label] = np.array('')
        except Exception as e:  # noqa: BLE001  (the type is the fixture)
            out['error_' + label] = np.array(type(e).__name__)
    e = np.linspace(0, 40, 9)
    out['erbs'], out['erbs_hz'] = e, np.array([G.ERBS_2_Hz(v) for v in e])
    f = np.array([0, 50, 125, 1000, 4000, 8000, 22050])
    out['hz'], out['hz_erbs'] = f, np.array([G.Hz_2_ERBS(v) for v in f])
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'gammatone.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_gammatone(*sys.argv[1:]))
