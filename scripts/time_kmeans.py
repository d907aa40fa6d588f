"""Time BinaryGMMTrainer().fit (sklearn's KMeans on the device) at deep-clustering sizes.

    python scripts/time_kmeans.py [--reps 10] [--host]

Per shape (N, E, K): ms per fit (CUDA events around the fit of a CUDA tensor, steady state), the iteration count,
the Lloyd kernel's time per pass from torch.profiler (n_iter passes plus the final labels / inertia pass), the bytes
a pass must read (N E 8 of the centred data plus the labels) and their share of the H100 SXM's 3.35 TB/s.  --host
adds one fit of the NumPy restatement and of sklearn (if importable) on the host.  The card's name and power limit
are read in the same run."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pb_bss_b200  # noqa: E402
from oracle import kmeans_oracle as KO  # noqa: E402
from pb_bss_b200.distribution import BinaryGMMTrainer  # noqa: E402

SHAPES = [(256500, 20, 3), (256500, 40, 4), (513000, 40, 4)]
HBM = 3.35e12


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'{torch.cuda.get_device_name()} (power limit unknown: {e})'
    return q


def fit(x, K, seed):
    np.random.seed(seed)
    with pb_bss_b200.deferred_status():
        return BinaryGMMTrainer().fit(x, K).kmeans


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--host', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'time_kmeans.py needs a CUDA device'
    print('card:', card())
    for N, E, K in SHAPES:
        xh = KO.blobs(N + E + K, N, E, K, 1.0)
        x = torch.from_numpy(xh).cuda()
        km = fit(x, K, 0)
        n_iter = int(km.n_iter_)
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(args.reps):
            fit(x, K, 0)
        stop.record()
        torch.cuda.synchronize()
        ms_fit = start.elapsed_time(stop) / args.reps
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fit(x, K, 0)
            torch.cuda.synchronize()
        kt = {}
        for ev in prof.key_averages():
            if ev.key.startswith('_ZN3pbb') or 'kmeans' in ev.key:
                kt[ev.key] = getattr(ev, 'device_time_total', getattr(ev, 'cuda_time_total', 0.0)) / 3 / 1e3
        lloyd = sum(v for k, v in kt.items() if 'lloyd' in k)
        init = sum(v for k, v in kt.items() if 'init' in k)
        passes = n_iter + 1
        ms_pass = lloyd / passes
        nbytes = N * E * 8 + 2 * N * 4
        print(f'N={N} E={E} K={K}: {ms_fit:.3f} ms/fit, n_iter={n_iter}, init kernel {init:.3f} ms, lloyd kernel '
              f'{lloyd:.3f} ms = {ms_pass * 1e3:.1f} us/pass over {passes} passes, {nbytes / 1e6:.1f} MB/pass -> '
              f'{nbytes / (ms_pass * 1e-3) / 1e12:.2f} TB/s = {100 * nbytes / (ms_pass * 1e-3) / HBM:.0f} % of 3.35 TB/s')
        if args.host:
            np.random.seed(0)
            t0 = time.perf_counter()
            KO.fit(xh, K)
            t1 = time.perf_counter()
            line = f'    host: NumPy oracle {1e3 * (t1 - t0):.0f} ms'
            try:
                from sklearn.cluster import KMeans
                t0 = time.perf_counter()
                KMeans(n_clusters=K).fit(xh)
                line += f', sklearn {1e3 * (time.perf_counter() - t0):.0f} ms'
            except ImportError:
                line += ', sklearn not importable'
            print(line)


if __name__ == '__main__':
    main()
