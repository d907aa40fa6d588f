"""Time the differentiable cACGMM on the device against torch autograd of its restatement
(oracle/cacgmm_autograd_oracle.py) on the same GPU, with the GPU name and power limit read in the same run.

    python scripts/time_cacgmm_autograd.py [--out result.json]

Two workloads at F = 513, T = 500, D = 8, K = 3 (a 1024-point STFT of 8 s at 16 kHz, 8 microphones), complex128:
  unsupervised: logits -> softmax -> cacgmm_m_step -> -log_likelihood (the network's affiliations define the model);
  unrolled:     logits -> softmax -> fit(iterations=5) -> predict -> sum(R * posterior) with a fixed random R (a
                network-initialised EM; the plain sum would be the constant F T).
Forward and forward + backward times are medians of CUDA-event windows after a warm-up, inside deferred_status (the
forward's status words are read once per window).  A profiled forward + backward of each workload (torch.profiler,
CUDA activity) gives each kernel's time per step.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cacgmm_autograd_oracle as A  # noqa: E402
from oracle import synth  # noqa: E402
from pb_bss_b200 import _device  # noqa: E402
from pb_bss_b200.distribution import CACGMMTrainer  # noqa: E402
from pb_bss_b200.distribution.cacgmm import cacgmm_m_step  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds  # noqa: E402

F, T, D, K, ITERATIONS = 513, 500, 8, 3, 5


def workloads(y, logits, R):
    def unsup_dev():
        return -cacgmm_m_step(y, None, torch.softmax(logits, 1)).log_likelihood(y)

    def unsup_ref():
        return -A.log_likelihood(y, A.m_step(y, None, torch.softmax(logits, 1)))

    def unrolled_dev():
        model = CACGMMTrainer().fit(y, initialization=torch.softmax(logits, 1), iterations=ITERATIONS)
        return model.predict(y).mul(R).sum()

    def unrolled_ref():
        return A.predict(y, A.fit(y, torch.softmax(logits, 1), ITERATIONS)).mul(R).sum()
    return {'unsupervised': (unsup_dev, unsup_ref), 'unrolled_fit5': (unrolled_dev, unrolled_ref)}


def step(loss_fn, logits, backward):
    def run():
        with _device.deferred_status():
            loss = loss_fn()
            if backward:
                torch.autograd.grad(loss, logits)
    return run


def kernel_table(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
        if 'pbb' in e.key and t > 0:
            rows.append({'kernel': e.key.split('(')[0][:80], 'calls': e.count, 'us': round(t, 1)})
    return sorted(rows, key=lambda r: -r['us'])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    y_np, _ = synth.structured_stft(F, T, D, K, seed=1)
    y = torch.tensor(y_np, device='cuda')
    logits = torch.tensor(np.random.default_rng(2).standard_normal((F, K, T)), device='cuda', requires_grad=True)
    R = torch.tensor(np.random.default_rng(3).standard_normal((F, K, T)), device='cuda')
    result = {'gpu': gpu_info(), 'shape': {'F': F, 'T': T, 'D': D, 'K': K, 'iterations': ITERATIONS}}
    for name, (dev, ref) in workloads(y, logits, R).items():
        r = {}
        for label, fn, calls in (('device', dev, 10), ('restatement', ref, 3)):
            r[label + '_forward_ms'] = device_seconds(step(fn, logits, False), calls=calls)[0] * 1e3
            r[label + '_forward_backward_ms'] = device_seconds(step(fn, logits, True), calls=calls)[0] * 1e3
        ld, lr = dev(), ref()
        gd, = torch.autograd.grad(ld, logits)
        gr, = torch.autograd.grad(lr, logits)
        r['max_grad_rel_diff'] = ((gd - gr).abs().max() / gr.abs().max()).item()
        r['kernels'] = kernel_table(step(dev, logits, True))
        result[name] = r
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
