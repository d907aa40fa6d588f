"""Device time of pb_bss_b200.wpe.wpe with nara_wpe's defaults (taps = 10, delay = 3, iterations = 3,
psd_context = 0, 'full') at (F, D, T) = (513, 8, 500), (513, 6, 500), (257, 2, 2000) and (513, 8, 4000), with the
GPU name and power limit read in the same run.

    python scripts/time_wpe.py [--out result.json]

Times are CUDA events around calls of the public function on complex128 CUDA tensors (median of 5 repeats of 5 calls
after a warm-up; the wrapper's host work and its one status read are included).  Per-kernel times come from
torch.profiler in a separate run.  Algorithmic FLOPs per bin and iteration (complex multiply-add = 8), n = taps D:
correlations 8 T (n (n + 1) / 2 + n D) (the Hermitian half of R and all of P), solve 8 n^3 / 3 + 8 n^2 D, filter
8 n D T.  The correlation kernel's rate is set against the 67 TFLOP/s fp64 tensor-core rate of the H100 SXM data
sheet, and so is the whole call's.  Yardsticks: the NumPy restatement (oracle/wpe_oracle.py) on the host, one call,
and a torch complex128 version on the device (batched matmul + torch.linalg.solve, per-bin weights).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import wpe_oracle as O  # noqa: E402
from pb_bss_b200.wpe import wpe  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

FP64_TC_FLOPS = 67e12
TAPS, DELAY, ITERATIONS = 10, 3, 3
SHAPES = ((513, 8, 500), (513, 6, 500), (257, 2, 2000), (513, 8, 4000))


def flops(F, D, T):
    n = TAPS * D
    per = {'correlation': 8.0 * T * (n * (n + 1) / 2 + n * D), 'solve': 8.0 * n ** 3 / 3 + 8.0 * n * n * D,
           'filter': 8.0 * n * D * T}
    return {k: F * ITERATIONS * v for k, v in per.items()}


def torch_wpe(Y):
    """The same iteration in torch complex128 on the device: Yt by padding, R and P by batched matmul."""
    F, D, T = Y.shape
    Yp = torch.nn.functional.pad(Y, (DELAY + TAPS - 1, 0))
    Yt = torch.cat([Yp[..., TAPS - 1 - k:TAPS - 1 - k + T] for k in range(TAPS)], dim=1)   # (F, taps D, T)
    X = Y
    for _ in range(ITERATIONS):
        lam = (X.real ** 2 + X.imag ** 2).mean(dim=1)
        w = 1 / torch.maximum(lam, 1e-10 * lam.amax(dim=1, keepdim=True))
        Ytw = Yt * w[:, None, :]
        R = Ytw @ Yt.conj().transpose(1, 2)
        P = Ytw @ Y.conj().transpose(1, 2)
        G = torch.linalg.solve(R, P)
        X = Y - G.conj().transpose(1, 2) @ Yt
    return X


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
        if t and 'wpe_' in e.key:
            name = e.key.split('(')[0].replace('void ', '').replace('pbb::', '')
            name = name.split('<')[0]
            out[name] = out.get(name, 0.0) + t / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'taps': TAPS, 'delay': DELAY, 'iterations': ITERATIONS, 'configs': {}}
    for F, D, T in SHAPES:
        rng = np.random.default_rng(F + D + T)
        Y = rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T))
        y = torch.from_numpy(Y).cuda()
        s, all_s = device_seconds(lambda: wpe(y), calls=5)
        kt = kernel_times(lambda: wpe(y))
        fl = flops(F, D, T)
        total = sum(fl.values())
        corr_us = kt.get('wpe_corr_kernel', 0.0)
        ts, _ = device_seconds(lambda: torch_wpe(y), calls=3)
        err = (torch_wpe(y) - wpe(y)).abs().max().item() / y.abs().max().item()
        rec = {'F': F, 'D': D, 'T': T, 'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s],
               'kernel_us_per_call': kt, 'flops': fl, 'flops_total': total,
               'call_share_of_fp64_tc_peak': total / s / FP64_TC_FLOPS,
               'corr_kernel_share_of_fp64_tc_peak': fl['correlation'] / (corr_us * 1e-6) / FP64_TC_FLOPS
               if corr_us else None,
               'torch_complex128_ms_per_call': ts * 1e3, 'torch_max_rel_diff': err,
               'oracle_host_ms': host_seconds(lambda: O.wpe(Y), repeats=1) * 1e3}
        result['configs'][f'F{F}_D{D}_T{T}'] = rec
        print(f'F{F}_D{D}_T{T}', json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
