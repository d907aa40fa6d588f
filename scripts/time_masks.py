"""Kernel time of the oracle masks at (K, D, F, T) = (2, 6, 513, 500) complex128, next to the reference's CPU time
and to torch.sort / torch.quantile on the same rows, with the GPU name and power limit read in the same run.

    python scripts/time_masks.py [--out result.json]

Each mask is timed as the public function on a CUDA tensor (device_ms_per_call: CUDA events around N calls, median
over repeats after a warm-up; the Python wrapper's host work is included, the launches are asynchronous).  The
algorithmic bytes count the signal read once plus the mask written once; the share is of the 3.35 TB/s HBM3
data-sheet figure of the H100 SXM.  The torch yardsticks sort / take quantiles of the already-formed rows (power or
|s|), so they do less work than the masks, which also form the rows and write the mask.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim  # noqa: E402
from pb_bss_b200 import extraction as E  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-reference', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    M = None
    if not args.no_reference and ref_shim.available():
        import importlib
        ref_shim.load()
        M = importlib.import_module('pb_bss.extraction.mask_module')
    K, D, F, T = 2, 6, 513, 500
    rng = np.random.RandomState(0)
    sig = rng.randn(K, D, F, T) + 1j * rng.randn(K, D, F, T)
    x = torch.from_numpy(sig).cuda()
    sig_bytes = sig.size * 16
    result = {'gpu': gpu_info(), 'shape': [K, D, F, T], 'dtype': 'complex128', 'configs': {}}

    cases = {
        'ibm_pooled': (lambda: E.ideal_binary_mask(x, sensor_axis=1), lambda: M.ideal_binary_mask(sig, sensor_axis=1),
                       K * F * T * 8),
        'wiener_pooled': (lambda: E.wiener_like_mask(x, sensor_axis=1),
                          lambda: M.wiener_like_mask(sig, sensor_axis=1), K * F * T * 8),
        'ideal_ratio': (lambda: E.ideal_ratio_mask(x), lambda: M.ideal_ratio_mask(sig), sig.size * 8),
        'phase_sensitive': (lambda: E.phase_sensitive_mask(x), lambda: M.phase_sensitive_mask(sig), sig.size * 8),
        'ideal_complex': (lambda: E.ideal_complex_mask(x), lambda: M.ideal_complex_mask(sig), sig.size * 16),
        'lorenz_pooled': (lambda: E.lorenz_mask(x, sensor_axis=1), lambda: M.lorenz_mask(sig, sensor_axis=1),
                          K * F * T * 8),
        'lorenz_time_rows': (lambda: E.lorenz_mask(x, axis=-1, lorenz_fraction=0.9),
                             lambda: M.lorenz_mask(sig, axis=-1, lorenz_fraction=0.9), sig.size * 8),
        'quantile_default': (lambda: E.quantile_mask(x), lambda: M.quantile_mask(sig), 2 * sig.size * 8),
        'biased_binary': (lambda: E.biased_binary_mask(x[:, 0]), lambda: M.biased_binary_mask(sig[:, 0]),
                          K * F * T),
    }
    power_rows = (x.abs() ** 2).sum(1).reshape(K, F * T)           # yardstick inputs only, formed outside the timing
    mag_rows = x.abs().transpose(-2, -1).reshape(-1, F)
    yardsticks = {
        'lorenz_pooled': lambda: torch.sort(power_rows, dim=-1, descending=True),
        'lorenz_time_rows': lambda: torch.sort((x.abs() ** 2).reshape(-1, T), dim=-1, descending=True),
        'quantile_default': lambda: torch.quantile(mag_rows, torch.tensor([0.9, 0.9], device='cuda',
                                                                          dtype=torch.float64), dim=-1),
    }
    for name, (fn, ref, out_bytes) in cases.items():
        calls = 20 if name.startswith(('lorenz', 'quantile')) else 100
        in_bytes = sig_bytes // D if name == 'biased_binary' else sig_bytes
        if name == 'quantile_default':
            in_bytes = 2 * sig_bytes                               # one read per quantile of the default pair
        s, all_s = device_seconds(fn, calls=calls)
        nbytes = in_bytes + out_bytes
        rec = {'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s],
               'algorithmic_bytes': nbytes, 'achieved_GB_per_s': nbytes / s * 1e-9,
               'share_of_3.35TB_per_s': nbytes / s / HBM_BYTES_PER_S}
        if name in yardsticks:
            y, _ = device_seconds(yardsticks[name], calls=calls)
            rec['torch_yardstick_ms_per_call'] = y * 1e3
        if M is not None:
            rec['reference_cpu_ms_per_call'] = host_seconds(ref, repeats=1) * 1e3
        result['configs'][name] = rec
        print(name, json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
