"""Time the single distributions of pb_bss.distribution on the device.

    python scripts/time_distributions.py [--reps 20] [--host]

Two workloads at D = 8: M = 513 models (one per STFT bin) x N = 500 frames, and one model x 10^6 frames.  Per call:
ms from CUDA events around `reps` calls on CUDA tensors (steady state, status words read once at the end), the bytes
the algorithm must move -- the observation (16 D bytes per frame) once per pass plus the output -- and their share of
the H100 SXM's 3.35 TB/s.  Calls: the three log_pdf, ComplexAngularCentralGaussianTrainer.fit (10 iterations, ten
passes over y), ComplexWatsonTrainer.fit and ComplexCircularSymmetricGaussianTrainer.fit.  --host adds one call of
the reference from oracle/_ref when it exists (its cACG trainer slice by slice: it rejects leading dims).  The card's
name and power limit are read in the same run."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pb_bss_b200  # noqa: E402
from oracle import distributions_oracle as DO  # noqa: E402
from oracle import ref_shim  # noqa: E402
from pb_bss_b200 import distribution as dist  # noqa: E402

WORKLOADS = [(513, 500, 8), (1, 1_000_000, 8)]
HBM = 3.35e12


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f'{torch.cuda.get_device_name()} (power limit unknown: {e})'


def models(M, D, rng):
    cov = DO.hermitian_pd(rng, M, D=D)
    mode = rng.normal(size=(M, D)) + 1j * rng.normal(size=(M, D))
    mode /= np.linalg.norm(mode, axis=-1, keepdims=True)
    return cov, mode, rng.uniform(1.0, 50.0, size=M)


def calls(y, cov, mode, kappa, M):
    """name -> (callable, passes over y, output bytes per frame)."""
    cacg = dist.ComplexAngularCentralGaussian.from_covariance(cov)
    watson = dist.ComplexWatson(mode=mode, concentration=kappa)
    ccsg = dist.ComplexCircularSymmetricGaussian(covariance=cov)
    return {
        'cacg.log_pdf': (lambda: cacg.log_pdf(y), 1, 8),
        'watson.log_pdf': (lambda: watson.log_pdf(y), 1, 8),
        'ccsg.log_pdf': (lambda: ccsg.log_pdf(y), 1, 8),
        'cacg_trainer.fit(10 it)': (lambda: dist.ComplexAngularCentralGaussianTrainer().fit(y), 10, 0),
        'watson_trainer.fit': (lambda: dist.ComplexWatsonTrainer().fit(y), 1, 0),
        'ccsg_trainer.fit': (lambda: dist.ComplexCircularSymmetricGaussianTrainer().fit(y), 1, 0),
    }


def host_calls(ref, y, cov, mode, kappa):
    d = ref.distribution
    cacg = d.ComplexAngularCentralGaussian.from_covariance(cov.copy())
    return {
        'cacg.log_pdf': lambda: cacg.log_pdf(y),
        'watson.log_pdf': lambda: d.ComplexWatson(mode=mode, concentration=kappa).log_pdf(y),
        'ccsg.log_pdf': lambda: d.ComplexCircularSymmetricGaussian(covariance=cov).log_pdf(y),
        'cacg_trainer.fit(10 it)': lambda: [d.ComplexAngularCentralGaussianTrainer().fit(s) for s in y],
        'watson_trainer.fit': lambda: d.ComplexWatsonTrainer().fit(y),
        'ccsg_trainer.fit': lambda: d.ComplexCircularSymmetricGaussianTrainer().fit(y),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--host', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'time_distributions.py needs a CUDA device'
    print('card:', card())
    ref = ref_shim.load() if args.host and ref_shim.available() else None
    for M, N, D in WORKLOADS:
        rng = np.random.default_rng(M + N)
        yh = DO.directional(rng, N, D, lead=(M,))
        cov, mode, kappa = models(M, D, rng)
        y = torch.from_numpy(yh).cuda()
        print(f'-- M={M} models x N={N} frames x D={D}')
        for name, (fn, passes, out_bytes) in calls(y, torch.from_numpy(cov).cuda(), torch.from_numpy(mode).cuda(),
                                                   torch.from_numpy(kappa).cuda(), M).items():
            fn()
            torch.cuda.synchronize()
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with pb_bss_b200.deferred_status():
                start.record()
                for _ in range(args.reps):
                    fn()
                stop.record()
            torch.cuda.synchronize()
            ms = start.elapsed_time(stop) / args.reps
            nbytes = M * N * (passes * 16 * D + out_bytes)
            line = (f'{name:26s} {ms:9.3f} ms  {nbytes / 1e6:8.1f} MB  '
                    f'{nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s  {100 * nbytes / HBM / (ms * 1e-3):5.1f} % of 3.35 TB/s')
            if ref is not None:
                hfn = host_calls(ref, yh, cov, mode, kappa)[name]
                t0 = time.perf_counter()
                hfn()
                line += f'  reference {1e3 * (time.perf_counter() - t0):9.1f} ms'
            print(line)


if __name__ == '__main__':
    main()
