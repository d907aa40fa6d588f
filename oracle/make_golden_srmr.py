"""Generate tests/golden/srmr.npz: the UNMODIFIED reference pb_bss/evaluation/module_srmr.py on seeded signals.

The reference checkout must be present (PB_BSS_REFERENCE, as for oracle/make_golden_gammatone.py):

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_srmr [OUT_DIR]

The reference's pb_bss/evaluation/__init__.py imports mir_eval, pystoi and pesq, so a stub package
``pb_bss.evaluation`` whose ``__path__`` points at the checkout is registered instead, and module_srmr's one outside
import, paderbox.array.segment.segment_axis, is the restatement of its ``end='pad'`` contract in
oracle/srmr_oracle.py (not paderbox itself).

Cases: sample rates 8000, 16000, 44100 and 48000; n = 1, 4 and 23; default and explicit low_freq; dry and
reverberant amplitude-modulated harmonic signals; VAD gaps at exactly 0.05 sr (kept) and 0.05 sr + 1 (removed) with
leading and trailing silence; a signal shorter than one frame; float32; int16 (the value of the float64 cast, since
the reference squares max|x| in the integer dtype); 2-D and 3-D input; the exception types for a leading dim of 30
and for 0-d input.  Stored per case: the signal, the parameters, srmr's value(s), and for the VAD cases the output of
_preprocessing_vad, as a packed mask of the kept samples that is checked against that output.  The signals are stored
as 16-bit codes: each float signal is quantised to multiples of 2^-15 (peak 0.9) before the reference sees it, so the
codes reproduce the reference's input exactly in its dtype (``signal``).  Every case's decision margins
(oracle/srmr_oracle.py) must exceed 1e-6.
"""
import importlib
import os
import sys
import types

import numpy as np

from . import make_golden_gammatone
from . import make_golden_transform
from . import srmr_oracle

OUT = make_golden_transform.OUT
MARGIN = 1e-6


def am_harmonic(rng, sr, seconds, f0=140.0, rate=4.0):
    """Harmonics of f0 up to sr / 2.5 (1 / h amplitudes) under a raised-cosine envelope at `rate` Hz, plus a little
    noise."""
    t = np.arange(int(seconds * sr)) / sr
    h = np.arange(1, int(sr / 2.5 / f0) + 1)
    x = np.sum(np.sin(2 * np.pi * f0 * h[:, None] * t + rng.uniform(0, 2 * np.pi, (len(h), 1))) / h[:, None], axis=0)
    x *= 0.5 * (1 - np.cos(2 * np.pi * rate * t)) ** 2
    return x + 1e-3 * rng.randn(len(t))


def reverberant(rng, x, sr, t60=0.6):
    """x convolved with an exponentially decaying noise impulse response, cut to len(x)."""
    n = int(t60 * sr)
    rir = rng.randn(n) * np.exp(-6.9 * np.arange(n) / n)
    rir[0] = 1.0
    return np.convolve(x, rir)[:len(x)] / np.abs(rir).sum() * 10


def vad_gaps(rng, sr):
    """Leading silence, speech, a silent gap whose above-threshold neighbours are exactly 0.05 sr apart (kept), speech,
    a gap of 0.05 sr + 1 (removed), speech, trailing silence."""
    w = int(0.05 * sr)
    seg = lambda s: am_harmonic(rng, sr, s)
    a, b, c = seg(0.3), seg(0.25), seg(0.3)
    for v in (a, b, c):
        v[0] = v[-1] = 0.9                # above threshold at both ends of every segment
    gap1, gap2 = np.zeros(w - 1), np.zeros(w)
    lead, trail = np.zeros(int(0.1 * sr)), np.zeros(int(0.07 * sr))
    return np.concatenate([lead, a, gap1, b, gap2, c, trail])


def cases(rng):
    """name -> (signal, sample_rate, n, low_freq or None)."""
    out = {}
    out['sr16k_dry'] = (am_harmonic(rng, 16000, 1.2), 16000, 23, None)
    out['sr16k_reverb'] = (reverberant(rng, am_harmonic(rng, 16000, 1.2), 16000), 16000, 23, None)
    out['sr8k_n4_reverb_low200'] = (reverberant(rng, am_harmonic(rng, 8000, 1.5, f0=110), 8000, 0.8), 8000, 4, 200)
    out['sr44k_n23_reverb'] = (reverberant(rng, am_harmonic(rng, 44100, 0.6), 44100, 0.4), 44100, 23, None)
    out['sr48k_n1_low300'] = (am_harmonic(rng, 48000, 0.5, f0=200), 48000, 1, 300)
    out['sr48k_n23_dry_low125'] = (am_harmonic(rng, 48000, 0.5, f0=180, rate=6.0), 48000, 23, 125)
    out['sr16k_vad_gaps'] = (vad_gaps(rng, 16000), 16000, 23, None)
    out['sr8k_vad_gaps_n4'] = (vad_gaps(rng, 8000), 8000, 4, None)
    out['sr16k_short'] = (am_harmonic(rng, 16000, 0.6), 16000, 23, None)          # 9600 < W = 16384
    out['sr16k_f32'] = (reverberant(rng, am_harmonic(rng, 16000, 1.0), 16000).astype(np.float32), 16000, 23, None)
    out['sr16k_f32_vad_gaps'] = (vad_gaps(rng, 16000).astype(np.float32), 16000, 4, None)
    x = am_harmonic(rng, 16000, 1.0)
    out['sr16k_int16'] = (np.round(x / np.abs(x).max() * 20000).astype(np.int16), 16000, 4, None)
    out['sr16k_2d'] = (np.stack([am_harmonic(rng, 16000, 1.0),
                                 reverberant(rng, am_harmonic(rng, 16000, 1.0), 16000)]), 16000, 4, None)
    out['sr8k_3d'] = (np.stack([np.stack([am_harmonic(rng, 8000, 1.0, f0=f), reverberant(rng, am_harmonic(
        rng, 8000, 1.0, f0=f), 8000)]) for f in (120, 210)]), 8000, 4, None)
    return out


def _register_stubs():
    make_golden_gammatone._reference()                 # pb_bss stub, checkout path, nara_wpe stub
    checkout = os.path.join(make_golden_transform.build_ref.SRC, 'pb_bss', 'evaluation')
    ev = types.ModuleType('pb_bss.evaluation')
    ev.__path__ = [checkout]
    sys.modules['pb_bss.evaluation'] = ev
    for name in ('paderbox', 'paderbox.array'):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    seg = types.ModuleType('paderbox.array.segment')
    seg.segment_axis = srmr_oracle.segment_axis
    sys.modules['paderbox.array.segment'] = seg
    return importlib.import_module('pb_bss.evaluation.module_srmr')


STEP = 2.0 ** -15   # quantum of the stored float signals


def quantise(x):
    """int16 codes of a float signal scaled to a peak of 0.9: the signal the reference sees is codes * STEP in the
    signal's dtype, exactly, so the fixture stores two bytes per sample."""
    return np.round(x / np.abs(x).max() * 0.9 / STEP).astype(np.int16)


def signal(g, name):
    """The input signal of case `name` from the fixture, in its dtype (float64, float32 or int16)."""
    q, dtype = g[name + '_q'], str(g[name + '_dtype'])
    return q if dtype == 'int16' else q.astype(dtype) * np.dtype(dtype).type(STEP)


def vad_output(g, name):
    """_preprocessing_vad's output of case `name`: the signal's samples at the stored keep mask."""
    x = signal(g, name)
    return x[np.unpackbits(g[name + '_vad_keep'], count=x.shape[-1]).astype(bool)]


def make_srmr(out_dir=OUT):
    R = _register_stubs()
    rng = np.random.RandomState(2024)
    out = {}
    for name, (x, sr, n, lo) in cases(rng).items():
        kw = {} if lo is None else {'low_freq': lo}
        out[name + '_dtype'] = np.array(x.dtype.name)
        out[name + '_q'] = x if x.dtype == np.int16 else quantise(x)
        x = signal(out, name)
        xr = x.astype(np.float64) if x.dtype == np.int16 else x
        v = R.srmr(xr, sr, n, **kw)
        for row in xr.reshape(-1, xr.shape[-1]):
            o = srmr_oracle.srmr_single(row, sr, n, 125 if lo is None else lo)
            assert o['margin_bw'] > MARGIN and o['margin_cutoff'] > MARGIN, (name, o['margin_bw'], o['margin_cutoff'])
        out[name + '_params'] = np.array([sr, n, 125 if lo is None else lo, lo is None], dtype=np.float64)
        out[name + '_value'] = np.asarray(v, dtype=np.float64)
        if 'vad' in name:
            ref = R._preprocessing_vad(x, sr)
            keep = srmr_oracle.vad_keep(x, sr)
            assert np.array_equal(x[keep], ref) and x[keep].dtype == ref.dtype and len(ref) < len(x), name
            out[name + '_vad_keep'] = np.packbits(keep)
            assert np.array_equal(vad_output(out, name), ref)
    for label, x in (('dim30', np.zeros((30, 100))), ('ndim0', np.float64(1.0))):
        try:
            R.srmr(x, 16000)
            out['error_' + label] = np.array('')
        except Exception as e:  # noqa: BLE001  (the type is the fixture)
            out['error_' + label] = np.array(type(e).__name__)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'srmr.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_srmr(*sys.argv[1:]))
