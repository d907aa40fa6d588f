"""Time the differentiable STOI / ESTOI on the device against torch autograd of their restatement
(oracle/stoi_autograd_oracle.py) on the same GPU, with the GPU name and power limit read in the same run.

    python scripts/time_stoi_autograd.py [--out result.json]

Shapes a user trains on: 16 signals of 4 s at 16 kHz, and 8 signals of 10 s at 16 kHz; float64, the reference and
the estimate both require grad, loss = sum of the values.  Forward and forward + backward times are medians of
CUDA-event windows after a warm-up, inside deferred_status (the forward's status word is read once per window, not
per call).  A profiled run (torch.profiler, CUDA activity) of forward + backward per shape gives each kernel's time;
with its algorithmic bytes (each array read or written once per call) it gives the share of the H100 SXM's
3.35 TB/s HBM3.  The backward's own launch sequence runs the forward's resample, energy, compact and bands kernels
again, so those appear with two calls per step.
"""
import argparse
import json
import os
import sys

import numpy as np
import scipy.signal
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import stoi_autograd_oracle as A  # noqa: E402
from pb_bss_b200 import _device  # noqa: E402
from pb_bss_b200.evaluation import module_stoi as MS  # noqa: E402
from pb_bss_b200.evaluation import stoi  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds  # noqa: E402

HBM = 3.35e12
FS = 16000
SHAPES = [(16, 4 * FS), (8, 10 * FS)]


def signals(rng, rows, n):
    t = np.arange(n) / FS
    x = np.stack([scipy.signal.lfilter([1.0], [1.0, -1.3, 0.6], rng.standard_normal(n))
                  * (1 + 0.9 * np.sign(np.sin(2 * np.pi * 4 * t + rng.uniform(0, 6)))) for _ in range(rows)])
    return x, x + 0.7 * rng.standard_normal(x.shape)


def kernel_bytes(B, n, extended):
    """Algorithmic bytes of one call of each kernel for B rows of n samples at 16 kHz (fp64, every kept frame)."""
    L = MS.resampled_length(n, FS)
    F = A.num_frames(L)
    M = F - 1
    J = max(M - 29, 0)
    d = 8
    tob = B * 2 * 15 * M * d
    seg = B * J * d * ((8 * 15 + 7 * 30) if extended else 10 * 15)
    return {
        'stoi_resample_kernel': B * 2 * (n + L) * d,
        'stoi_energy_kernel': B * (L + F) * d,
        'stoi_compact_kernel': B * F * (d + 4),
        'stoi_bands_kernel': B * 2 * L * d + tob,
        'stoi_rank_kernel': B * F * 8,
        'stoi_segment_prep_kernel': tob + seg,
        'estoi_segment_prep_kernel': tob + seg,
        'stoi_segment_grad_kernel': 2 * tob + seg,
        'estoi_segment_grad_kernel': 2 * tob + seg,
        'stoi_spectral_grad_kernel': B * 2 * L * d + 2 * tob + B * 2 * M * 256 * d,
        'stoi_removal_grad_kernel': B * 2 * M * 256 * d + B * 2 * L * d,
        'stoi_resample_grad_kernel': B * 2 * (L + n) * d,
        'stoi_segment_kernel': tob,
        'estoi_segment_kernel': tob,
        'stoi_value_kernel': B * 8,
    }


def ms(fn, calls):
    def window():
        with _device.deferred_status():
            fn()
    return device_seconds(window, calls=calls, repeats=5)[0] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    result = {'gpu': gpu_info(), 'sample_rate': FS, 'shapes': {}}
    for B, n in SHAPES:
        xn, yn = signals(rng, B, n)
        x = torch.tensor(xn, device='cuda')
        y = torch.tensor(yn, device='cuda')
        xr, yr = x.clone().requires_grad_(), y.clone().requires_grad_()
        entry = {}
        for extended in (False, True):
            name = 'estoi' if extended else 'stoi'

            def dev_fwd(e=extended):
                with torch.no_grad():
                    stoi(x, y, FS, extended=e)

            def dev_fb(e=extended):
                torch.autograd.grad(stoi(xr, yr, FS, extended=e).sum(), (xr, yr))

            def ref_fwd(e=extended):
                with torch.no_grad():
                    A.stoi(x, y, FS, e)

            def ref_fb(e=extended):
                torch.autograd.grad(A.stoi(xr, yr, FS, e)[0].sum(), (xr, yr))

            entry[name] = {
                'device': {'forward_ms': ms(dev_fwd, 5), 'forward_backward_ms': ms(dev_fb, 5)},
                'torch': {'forward_ms': ms(ref_fwd, 2), 'forward_backward_ms': ms(ref_fb, 2)},
            }
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    dev_fb()
                torch.cuda.synchronize()
            cost = kernel_bytes(B, n, extended)
            kernels = {}
            for evt in prof.key_averages():
                base = next((k for k in sorted(cost, key=len, reverse=True) if k in evt.key), None)
                if base is None:
                    continue
                dev_us = getattr(evt, 'device_time_total', None)
                if dev_us is None:
                    dev_us = evt.cuda_time_total
                k = kernels.setdefault(base, {'calls': 0, 'us_total': 0.0})
                k['calls'] += evt.count
                k['us_total'] += dev_us
            for base, k in kernels.items():
                us = k['us_total'] / k['calls']
                k.update({'us_per_call': us, 'calls_per_step': k['calls'] / 3, 'bytes': cost[base],
                          'share_of_3.35TBs': cost[base] / (us * 1e-6) / HBM})
                del k['us_total'], k['calls']
            entry[name]['kernels'] = kernels
        result['shapes'][f'{B}x{n}'] = entry
        print(json.dumps({f'{B}x{n}': entry}), flush=True)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
