"""Device time of pb_bss_b200.transform.gammatone.gammatone_filterbank at user-sized shapes, (8, 160000) float64
(8 channels, 10 s at 16 kHz) and (1, 2880000) float64 (60 s at 48 kHz), n = 23, with the GPU name and power limit
read in the same run.

    python scripts/time_gammatone.py [--out result.json]

Times are CUDA events around 20 calls of the public function on a CUDA tensor (median of 5 repeats after a warm-up;
the wrapper's host work is included, the launches are asynchronous).  The algorithmic bytes are the signal read once
and the n outputs written once, 8 rows N (n + 1).  The fp64 operations are those of the chunked scan, which runs the
cascade twice (end states, then output): 2 x 4 sections x 7 flops (3 FMA counted as 2 each, 1 multiply) per sample
and filter; the carry is below 1 % of that.  The share is of the larger of the two data-sheet bounds of the H100 SXM,
3.35 TB/s of HBM3 and 34 TFLOP/s fp64 (non-tensor), and the bound that applies is named.  Host: the oracle's
scipy.signal.lfilter cascade (oracle/gammatone_oracle.py, the reference's arithmetic) on the same machine, one call.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gammatone_oracle as GO  # noqa: E402
from pb_bss_b200.transform import gammatone  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP64_FLOP_PER_S = 34e12
FLOPS_PER_SAMPLE_FILTER = 2 * 4 * 7


def kernel_times(fn, calls=10):
    """Device time per call of each kernel, from torch.profiler in a run of its own (after the timed one)."""
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
        if 'gammatone' in e.key and t:
            out[e.key.split('(')[0].replace('void ', '').replace('pbb::', '')] = t / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    n = 23
    for rows, N, sr in ((8, 160000, 16000), (1, 2880000, 48000)):
        x_host = np.random.RandomState(0).randn(rows, N)
        x = torch.from_numpy(x_host).cuda()
        s, all_s = device_seconds(lambda: gammatone.gammatone_filterbank(x, sr, n), calls=20)
        nbytes = 8 * rows * N * (n + 1)
        flops = FLOPS_PER_SAMPLE_FILTER * rows * N * n
        t_bytes, t_flops = nbytes / HBM_BYTES_PER_S, flops / FP64_FLOP_PER_S
        rec = {'shape': [rows, N], 'sample_rate': sr, 'n': n, 'chunk_length': gammatone.chunk_length(rows, n, N),
               'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s],
               'algorithmic_bytes': nbytes, 'fp64_flops': flops,
               'bound_us_bytes': t_bytes * 1e6, 'bound_us_fp64': t_flops * 1e6,
               'bound': 'HBM bytes' if t_bytes >= t_flops else 'fp64',
               'share_of_bound': max(t_bytes, t_flops) / s,
               'achieved_GB_per_s': nbytes / s * 1e-9, 'achieved_fp64_TFLOP_per_s': flops / s * 1e-12}
        rec['kernel_us_per_call'] = kernel_times(lambda: gammatone.gammatone_filterbank(x, sr, n))
        rec['oracle_lfilter_host_ms_per_call'] = host_seconds(lambda: GO.gammatone_filterbank(x_host, sr, n),
                                                              repeats=1) * 1e3
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
