"""Time the differentiable WPE on the device against torch autograd of its restatement (oracle/wpe_autograd_oracle.py:
batched matmul and torch.linalg.solve) on the same GPU, with the GPU name and power limit read in the same run.

    python scripts/time_wpe_autograd.py [--out result.json]

Shapes (F, D, T) = (513, 8, 500), (513, 6, 500) and (257, 2, 2000), complex128, taps 10, delay 3; wpe_step with
given weights and wpe with 3 iterations.  Also the DNN-WPE front end at F = 257, D = 6, T = 1002 (size 512, shift 128):
float32 logits -> power = sigmoid(logits) mean_d |Y|^2 -> wpe_step(Y, 1 / max(power, 1e-10)) -> PSD -> Souden MVDR
(reference channel 0) -> apply -> istft -> -si_sdr.  Forward and forward + backward times are medians of CUDA-event
windows after a warm-up.  A profiled run (torch.profiler, CUDA activity) of one wpe forward + backward per shape gives
each backward kernel's time; with its algorithmic flops (fp64, an FMA = 2) and bytes (each array read or written once)
it gives the share of the H100 SXM's 67 TFLOP/s FP64 tensor-core peak (wpe_corr_kernel) or of its 3.35 TB/s HBM3
(the per-frame kernels).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import autograd_oracle as AO  # noqa: E402
from oracle import wpe_autograd_oracle as WA  # noqa: E402
from pb_bss_b200 import wpe as W  # noqa: E402
from pb_bss_b200.evaluation import si_sdr  # noqa: E402
from pb_bss_b200.extraction import beamformer as B  # noqa: E402
from pb_bss_b200.transform import istft, stft  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds  # noqa: E402

HBM = 3.35e12
TC_FP64 = 67e12
TAPS, DELAY, ITERATIONS = 10, 3, 3
SHAPES = [(513, 8, 500), (513, 6, 500), (257, 2, 2000)]
SIZE, SHIFT, D_CHAIN = 512, 128, 6
N = 999 * SHIFT - 3


def kernel_cost(F, D, T):
    """(flops, bytes) of one call of each backward kernel over all F bins, complex128 input"""
    n = TAPS * D
    t8 = (2 * (n + D) + 7) // 8
    c, r = 16, 8
    return {
        'wpe_corr_kernel': (F * t8 * (t8 + 1) // 2 * 64 * 2 * T, F * (D * T * c + T * r)),
        'wpe_gbar_kernel': (F * n * D * T * 8, F * (2 * D * T * c + n * D * c)),
        'wpe_solve_rhs_kernel': (F * (8 * n ** 3 / 3 + 8 * n * n * D), F * 2 * n * D * c),
        'wpe_step_backward_kernel': (F * 4 * n * D * T * 8,
                                     F * (D * T * c * 8 + T * r * 2 + 2 * n * D * c)),
        'wpe_power_backward_kernel': (F * n * D * T * 8, F * (3 * D * T * c + 4 * T * r)),
    }


def front_end(device, y, logits, target):
    power = torch.sigmoid(logits[:, 0]).to(torch.float64) * (y.abs() ** 2).mean(-2)
    inv = 1 / torch.clamp(power, min=1e-10)
    mask = torch.sigmoid(logits[:, 1:]).to(torch.float64)
    if device:
        x = W.wpe_step(y, inv, TAPS, DELAY)
        pt = B.get_power_spectral_density_matrix(x, mask[:, 0])
        pn = B.get_power_spectral_density_matrix(x, mask[:, 1])
        s = B.apply_beamforming_vector(B.get_mvdr_vector_souden(pt, pn, 0), x)
        return -si_sdr(target, istft(s.transpose(0, 1), size=SIZE, shift=SHIFT)[:N])
    x = WA.wpe_step(y, inv, TAPS, DELAY)[0]
    pt = AO.power_spectral_density(x, mask[:, 0])
    pn = AO.power_spectral_density(x, mask[:, 1])
    s = AO.apply_beamforming_vector(AO.mvdr_vector_souden(pt, pn, 0)[0], x)
    return -AO.si_sdr(target, AO.istft(s.transpose(0, 1), SIZE, SHIFT)[:N])


def ms(fn, calls):
    return device_seconds(fn, calls=calls, repeats=5)[0] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    result = {'gpu': gpu_info(), 'taps': TAPS, 'delay': DELAY, 'iterations': ITERATIONS, 'shapes': {}}
    for F, D, T in SHAPES:
        y = torch.tensor(rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T)), device='cuda')
        w = torch.tensor(rng.uniform(0.5, 2.0, (F, T)), device='cuda')
        g = torch.randn_like(y)
        yr, wr = y.clone().requires_grad_(), w.clone().requires_grad_()
        fns = {
            'device_wpe_step': (lambda: W.wpe_step(y, w, TAPS, DELAY),
                                lambda: torch.autograd.grad(W.wpe_step(yr, wr, TAPS, DELAY), (yr, wr), g)),
            'torch_wpe_step': (lambda: WA.wpe_step(y, w, TAPS, DELAY),
                               lambda: torch.autograd.grad(WA.wpe_step(yr, wr, TAPS, DELAY)[0], (yr, wr), g)),
            'device_wpe': (lambda: W.wpe(y, TAPS, DELAY, ITERATIONS),
                           lambda: torch.autograd.grad(W.wpe(yr, TAPS, DELAY, ITERATIONS), yr, g)),
            'torch_wpe': (lambda: WA.wpe(y, TAPS, DELAY, ITERATIONS),
                          lambda: torch.autograd.grad(WA.wpe(yr, TAPS, DELAY, ITERATIONS), yr, g)),
        }
        entry = {}
        for name, (fwd, fwd_bwd) in fns.items():
            def no_grad_fwd(fwd=fwd):
                with torch.no_grad():
                    fwd()
            entry[name] = {'forward_ms': ms(no_grad_fwd, 5), 'forward_backward_ms': ms(fwd_bwd, 5)}
        # the backward kernels of one wpe forward + backward
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                torch.autograd.grad(W.wpe(yr, TAPS, DELAY, ITERATIONS), yr, g)
            torch.cuda.synchronize()
        cost = kernel_cost(F, D, T)
        kernels = {}
        for evt in prof.key_averages():
            base = next((k for k in cost if k in evt.key), None)
            if base is None:
                continue
            dev_us = getattr(evt, 'device_time_total', None)
            if dev_us is None:
                dev_us = evt.cuda_time_total
            us = dev_us / evt.count
            k = kernels.setdefault(base, {'calls': 0, 'us_total': 0.0})
            k['calls'] += evt.count
            k['us_total'] += dev_us
        for base, k in kernels.items():
            us = k['us_total'] / k['calls']
            flops, nbytes = cost[base]
            k.update({'us_per_call': us, 'calls_per_step': k['calls'] / 3, 'flops': flops, 'bytes': nbytes,
                      'share_of_67TFLOPs': flops / (us * 1e-6) / TC_FP64,
                      'share_of_3.35TBs': nbytes / (us * 1e-6) / HBM})
            del k['us_total'], k['calls']
        # wpe_corr_kernel runs in the forward too (3 calls) and once per stage in the backward (3 calls)
        entry['wpe_kernels'] = kernels
        result['shapes'][f'{F}x{D}x{T}'] = entry
        print(json.dumps({f'{F}x{D}x{T}': entry}), flush=True)
        del y, w, g, yr, wr

    # the DNN-WPE front end
    sig = torch.tensor(rng.standard_normal((D_CHAIN, N)), device='cuda')
    y = stft(sig, size=SIZE, shift=SHIFT).permute(2, 0, 1).contiguous()
    F, _, T = y.shape
    logits = torch.tensor(rng.standard_normal((F, 3, T)), dtype=torch.float32, device='cuda', requires_grad=True)
    target = torch.tensor(rng.standard_normal(N), device='cuda')
    chain = {'F': F, 'D': D_CHAIN, 'T': T}
    for name, dev in (('device', True), ('torch', False)):
        def fwd(dev=dev):
            with torch.no_grad():
                front_end(dev, y, logits, target)

        def fwd_bwd(dev=dev):
            torch.autograd.grad(front_end(dev, y, logits, target), logits)
        chain[name] = {'forward_ms': ms(fwd, 10), 'forward_backward_ms': ms(fwd_bwd, 10)}
    result['dnn_wpe_front_end'] = chain
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
