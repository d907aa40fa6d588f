"""Device time of pb_bss_b200.evaluation.srmr at user-sized shapes, (8, 160000) float64 at 16 kHz (8 channels of
10 s) and (1, 2880000) float64 at 48 kHz (60 s), n = 23, with the GPU name and power limit read in the same run.

    python scripts/time_srmr.py [--out result.json]

Times are CUDA events around 5 calls of the public function on a CUDA tensor (median of 5 repeats after a warm-up;
the wrapper's host work is included).  Per-kernel times come from torch.profiler in a separate run.  Algorithmic
bytes per stage, each array read or written once: VAD 8 rows N (in) + 8 rows N (out) and the normalisation's
read-modify-write; gammatone 8 rows N (n + 1); Hilbert, per sequence, the signal read twice and written once
(3 x 8 N) and the FFT workspace of 2P = M points written and read three times (3 x 2 x 16 P); energies 8 rows N n
read twice.  The bound is that traffic at 3.35 TB/s (HBM3, H100 SXM data sheet).  Host: the NumPy restatement of the
reference (oracle/srmr_oracle.py) on one row, one call.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import srmr_oracle as SO  # noqa: E402
from pb_bss_b200.evaluation import srmr  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def kernel_times(fn, calls=3):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
        if t and ('srmr' in e.key or 'vad' in e.key or 'fl_' in e.key or 'gammatone' in e.key):
            out[e.key.split('(')[0].replace('void ', '').replace('pbb::', '')[:90]] = t / calls
    return out


def stage_bytes(rows, N, n):
    M = 1 << max(1, int(np.ceil(np.log2(2 * N - 1))))
    seq = rows * n
    return {'vad': 8 * rows * N * 4, 'gammatone': 8 * rows * N * (n + 1),
            'hilbert': seq * (3 * 8 * N + 3 * 2 * 8 * M) + rows * 2 * 8 * M,
            'energies': 2 * 8 * rows * N * n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    n = 23
    for rows, N, sr in ((8, 160000, 16000), (1, 2880000, 48000)):
        rng = np.random.RandomState(0)
        t = np.arange(N) / sr
        x_host = rng.randn(rows, N) * (1 + np.sin(2 * np.pi * 4 * t)) ** 2
        x = torch.from_numpy(x_host).cuda()
        s, all_s = device_seconds(lambda: srmr(x, sr, n), calls=5)
        b = stage_bytes(rows, N, n)
        total = sum(b.values())
        rec = {'shape': [rows, N], 'sample_rate': sr, 'n': n, 'device_ms_per_call': s * 1e3,
               'device_ms_all': [v * 1e3 for v in all_s], 'algorithmic_bytes': b,
               'bound_ms_hbm': total / HBM_BYTES_PER_S * 1e3, 'share_of_bound': total / HBM_BYTES_PER_S / s}
        rec['kernel_us_per_call'] = kernel_times(lambda: srmr(x, sr, n))
        rec['oracle_host_ms_per_row'] = host_seconds(lambda: SO.srmr_single(x_host[0], sr, n), repeats=1) * 1e3
        result['configs'][f'{rows}x{N}'] = rec
        print(f'{rows}x{N}', json.dumps(rec), flush=True)
        del x
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
