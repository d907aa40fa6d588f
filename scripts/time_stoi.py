"""Device time of pb_bss_b200.evaluation.stoi, STOI (extended=False) and ESTOI (extended=True), at user-sized shapes,
with the GPU name and power limit read in the same run:
  - (2, 6, 80000) float64 at 8 kHz: InputMetrics' shape (sources x channels x 10 s);
  - (256, 160000) float64 at 16 kHz: a batch of 10-s utterances;
  - (8, 441000) float64 at 44.1 kHz: 10 s at the rate with the longest resampling filter (320 taps per phase).

    python scripts/time_stoi.py [--out result.json]

Times are CUDA events around 5 calls of the public function on CUDA tensors, the two modes alternating over 5
rounds after a warm-up (median per mode; the wrapper's host work is included).  Per-kernel times come from
torch.profiler in a separate run per mode.  Algorithmic bytes and FLOPs per stage count each array once per kernel
(an FMA = 2 FLOPs); a stage's bound is the larger of its bytes at 3.35 TB/s (HBM3) and its FLOPs at 34 TFLOP/s (fp64
without tensor cores), both from the H100 SXM data sheet.  Host: the NumPy restatements (oracle/stoi_oracle.py,
oracle/estoi_oracle.py) on one pair, one call.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import estoi_oracle as O  # noqa: E402
from pb_bss_b200.evaluation import module_stoi as M  # noqa: E402
from pb_bss_b200.evaluation import stoi  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP64_FLOP_PER_S = 34e12
CONFIGS = (((2, 6, 80000), 8000), ((256, 160000), 16000), ((8, 441000), 44100))


MODES = (('stoi', False), ('estoi', True))


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
        if t and 'stoi' in e.key:
            out[e.key.split('(')[0].replace('void ', '').replace('pbb::', '')[:90]] = t / calls
    return out


def stage_cost(rows, n, fs, extended):
    """{stage: (bytes, flops)} with every frame kept (the upper bound of the later stages)."""
    up, down = M.rates(fs)
    L = M.resampled_length(n, fs)
    F = len(range(0, L - 256, 128))
    Mx = F - 1
    J = max(Mx - 29, 0)
    out = {}
    if (up, down) != (1, 1):
        tpp = M.polyphase_taps(fs)[0].shape[1]
        out['resample'] = (rows * 2 * (8 * n + 8 * L), rows * 2 * L * 2 * tpp)
    out['energy'] = (rows * (8 * L + 8 * F), rows * F * 256 * 3)
    out['compact'] = (rows * F * (8 + 4), rows * F * 2)
    # each STFT frame reads 4 half-frames of samples; a 512-point real FFT is about 2.5 * 512 * 9 FLOPs
    out['bands'] = (rows * 2 * Mx * (512 * 8 + 15 * 8), rows * 2 * Mx * (2.5 * 512 * 9 + 257 * 3 + 256 * 6))
    if extended:
        # per segment: 15 rows x 2 signals x 30 frames (sum, raw and centred squares: 6 FLOPs), then 30 columns x 15
        # bands x 2 signals, each value formed twice (about 10 FLOPs), with the column sums and the inner product
        out['segment'] = (rows * (2 * 15 * Mx * 8), rows * J * (15 * 2 * 30 * 6 + 30 * 15 * 2 * 10))
    else:
        out['segment'] = (rows * (2 * 15 * Mx * 8), rows * J * 15 * 30 * 14)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    for shape, fs in CONFIGS:
        rng = np.random.default_rng(0)
        n = shape[-1]
        t = np.arange(n) / fs
        env = (1.2 + np.sin(2 * np.pi * 3 * t)) ** 2
        ref_host = rng.standard_normal(shape) * env
        est_host = ref_host + 0.5 * rng.standard_normal(shape)
        ref, est = torch.from_numpy(ref_host).cuda(), torch.from_numpy(est_host).cuda()
        calls = {name: (lambda ext=ext: stoi(ref, est, fs, extended=ext)) for name, ext in MODES}
        times = {name: [] for name, _ in MODES}
        for fn in calls.values():
            fn()
        for _ in range(5):
            for name, _ in MODES:
                times[name].append(device_seconds(calls[name], calls=5, repeats=1)[0])
        rows = int(np.prod(shape[:-1]))
        flat_r, flat_e = ref_host.reshape(-1, n), est_host.reshape(-1, n)
        rec = {'shape': list(shape), 'sample_rate': fs}
        for name, ext in MODES:
            s = float(np.median(times[name]))
            cost = stage_cost(rows, n, fs, ext)
            bound = sum(max(b / HBM_BYTES_PER_S, f / FP64_FLOP_PER_S) for b, f in cost.values())
            m = {'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in times[name]],
                 'stages': {k: {'bytes': b, 'flops': f,
                                'bound_us': max(b / HBM_BYTES_PER_S, f / FP64_FLOP_PER_S) * 1e6,
                                'bound_by': 'hbm' if b / HBM_BYTES_PER_S > f / FP64_FLOP_PER_S else 'fp64'}
                            for k, (b, f) in cost.items()},
                 'bound_ms': bound * 1e3, 'share_of_bound': bound / s}
            m['kernel_us_per_call'] = kernel_times(calls[name])
            m['oracle_host_ms_per_row'] = host_seconds(lambda: O.stoi(flat_r[0], flat_e[0], fs, extended=ext),
                                                       repeats=1) * 1e3
            d = calls[name]().cpu().numpy().reshape(-1)
            m['max_abs_diff_vs_oracle_first_row'] = abs(float(d[0]) - float(O.stoi(flat_r[0], flat_e[0], fs,
                                                                                    extended=ext)))
            rec[name] = m
        rec['estoi_over_stoi'] = rec['estoi']['device_ms_per_call'] / rec['stoi']['device_ms_per_call']
        result['configs']['x'.join(map(str, shape)) + f'@{fs}'] = rec
        print(json.dumps(rec), flush=True)
        del ref, est
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
