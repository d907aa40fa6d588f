"""Generate tests/golden/transform.npz: a few steps of the UNMODIFIED reference GriffinLim and MISI
(pb_bss/transform/griffin_lim_module.py, through oracle/ref_shim.py) on seeded signals.  The reference imports its
transforms from nara_wpe.utils, which is not a dependency of this project; a stub module holding the restated
stft / istft of oracle/transform_oracle.py is registered in its place.

pb_bss/transform is not part of the hot-path copy under oracle/_ref, so it is imported from the reference checkout
(PB_BSS_REFERENCE, the same default as oracle/build_ref.py), which must be present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_transform [OUT_DIR]

Noise-like signals keep every |X_dash_dash| bin away from zero, where the phase is ill-conditioned.
"""
import importlib
import os
import sys
import types

import numpy as np

from . import build_ref
from . import ref_shim
from . import transform_oracle

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
STEPS = 5


def _register_nara_wpe_stub():
    pkg = types.ModuleType('nara_wpe')
    pkg.__path__ = []
    utils = types.ModuleType('nara_wpe.utils')
    utils.stft, utils.istft = transform_oracle.stft, transform_oracle.istft
    pkg.utils = utils
    sys.modules['nara_wpe'], sys.modules['nara_wpe.utils'] = pkg, utils


def _add_reference_checkout():
    """Lets the stub package pb_bss find subpackages that only the checkout has (here: transform)."""
    checkout = os.path.join(build_ref.SRC, 'pb_bss')
    if not os.path.isdir(os.path.join(checkout, 'transform')):
        raise RuntimeError(f'reference checkout with pb_bss/transform not found at {build_ref.SRC}')
    path = sys.modules['pb_bss'].__path__
    if checkout not in path:
        path.append(checkout)


def make_transform(out_dir=OUT):
    ref_shim.load()
    _add_reference_checkout()
    _register_nara_wpe_stub()
    G = importlib.import_module('pb_bss.transform.griffin_lim_module')
    rng = np.random.RandomState(23)
    K, size, shift, T = 3, 128, 32, 20
    n = (T - 1) * shift + size          # the length istft returns without fading: every step keeps T frames
    sources = rng.randn(K, n)
    y = sources.sum(0) + 0.1 * rng.randn(n)
    X = transform_oracle.stft(sources + 0.05 * rng.randn(K, n), size=size, shift=shift, fading=False)
    assert X.shape == (K, T, size // 2 + 1)
    out = {'X': X, 'y': y}
    for name, cls, guess in (('gl', G.GriffinLim, 'istft'), ('gl_y', G.GriffinLim, 'y'),
                             ('misi', G.MISI, 'istft'), ('misi_y', G.MISI, 'y')):
        m = cls(X, y, first_guess=guess, size=size, shift=shift, fading=False)
        for _ in range(STEPS):
            m.step()
        out[name + '_x_hat'], out[name + '_X_dash'], out[name + '_X_dash_dash'] = m.x_hat, m.X_dash, m.X_dash_dash
    # fading: the reconstruction keeps its length, so MISI's y must have it too
    Xf = transform_oracle.stft(sources, size=size, shift=shift, fading=True)
    yf = transform_oracle.istft(Xf, size=size, shift=shift, fading=True).sum(0)
    out.update(X_fading=Xf, y_fading=yf)
    m = G.MISI(Xf, yf, first_guess='istft', size=size, shift=shift, fading=True)
    for _ in range(STEPS):
        m.step()
    out['misi_fading_x_hat'], out['misi_fading_X_dash'] = m.x_hat, m.X_dash
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'transform.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_transform(*sys.argv[1:]))
