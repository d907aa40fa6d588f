"""Device time per EM iteration of the embedding mixture models (GMMTrainer, VMFMMTrainer), with the GPU name and
power limit of the same run and the bytes / flops one iteration moves and computes.

    python scripts/time_embedding_mm.py [--out result.json]

E1: B = 1, N = 102,800, E = 20, K = 3 (full covariance, spherical covariance, vMF);
E2: B = 16, N = 25,700, E = 40, K = 4 (full covariance).
An iteration's time is (t(21 iterations) - t(1 iteration)) / 20 between CUDA events, inputs already on the device.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pb_bss_b200.distribution import GMMTrainer, VMFMMTrainer  # noqa: E402

CONFIGS = [
    ('E1_full', 1, 102800, 20, 3, 'full'),
    ('E1_spherical', 1, 102800, 20, 3, 'spherical'),
    ('E1_vmf', 1, 102800, 20, 3, 'vmf'),
    ('E2_full', 16, 25700, 40, 4, 'full'),
]


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        limit = None
    return {'name': name, 'power_limit_w': limit}


def cost_per_iteration(B, N, E, K, kind):
    """Bytes to / from HBM and fp64 flops (an FMA = 2) of one iteration, counting each array once per kernel that
    streams it.  x: (B, N, E); affiliations, weights and log pdfs: (B, K, N)."""
    x, bkn = 8.0 * B * N * E, 8.0 * B * K * N
    P = E * (E + 1) / 2
    if kind == 'full':
        # fit: 2 passes over x and the weights; log pdf: x, write (B, K, N); posterior: read, write; class weight
        nbytes = 2 * (x + bkn) + (x + bkn) + 2 * bkn + bkn
        flops = B * K * N * (2 * 2 * (E + 1) + 3 * P + 2 * P + E)
    elif kind == 'spherical':
        nbytes = 2 * (x + bkn) + (x + bkn) + 2 * bkn + bkn
        flops = B * K * N * (2 * 2 * (E + 1) + 3 * E + 2 * E + E)
    else:
        nbytes = (x + bkn) + (x + bkn) + 2 * bkn + bkn
        flops = B * K * N * (2 * (E + 1) + 2 * E) + B * N * 3 * E
    return nbytes, flops


def time_fit(kind, y, init, iterations):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    if kind == 'vmf':
        VMFMMTrainer().fit(y, initialization=init, iterations=iterations)
    else:
        GMMTrainer().fit(y, initialization=init, iterations=iterations, covariance_type=kind)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    for name, B, N, E, K, kind in CONFIGS:
        rng = np.random.RandomState(0)
        # separated clouds and a start half way between the true labels and uniform noise: the reference's full
        # log pdf (U d instead of U^T d) is no density, and from a purely random start at E = 40 its EM can starve a
        # class into a singular covariance within a few iterations (the reference raises there too)
        centers = rng.randn(B, K, E) * 4.0
        labels = rng.randint(0, K, size=(B, N))
        y = centers[np.arange(B)[:, None], labels] + rng.randn(B, N, E)
        init = 0.5 * np.eye(K)[labels].transpose(0, 2, 1) + 0.5 * rng.uniform(size=(B, K, N))
        init /= init.sum(-2, keepdims=True)
        if B == 1:
            y, init = y[0], init[0]
        yd, idd = torch.from_numpy(y).cuda(), torch.from_numpy(init).cuda()
        time_fit(kind, yd, idd, 2)   # warm-up (library load, allocator)
        per = []
        for _ in range(args.repeats):
            per.append((time_fit(kind, yd, idd, 21) - time_fit(kind, yd, idd, 1)) / 20)
        t = float(np.median(per))
        nbytes, flops = cost_per_iteration(B, N, E, K, kind)
        result['configs'][name] = {
            'B': B, 'N': N, 'E': E, 'K': K, 'model': kind, 'ms_per_iteration': t * 1e3,
            'ms_per_iteration_all': [p * 1e3 for p in per], 'bytes_per_iteration': nbytes,
            'flops_per_iteration': flops, 'GB_per_s': nbytes / t / 1e9, 'GFLOP_per_s': flops / t / 1e9}
        print(name, json.dumps(result['configs'][name]), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
