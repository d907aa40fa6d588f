"""Device time of frame-online WPE (pb_bss_b200.wpe.online_wpe and online_wpe_step) with the GPU name and power
limit read in the same run.

    python scripts/time_online_wpe.py [--out result.json]

Whole streams (F, D, taps, delay, T) = (257, 8, 10, 2, 500), (513, 8, 10, 2, 500), (513, 2, 10, 2, 2000) and
(513, 8, 12, 2, 4000), alpha = 0.9999, complex128 CUDA tensors (T, F, D); the per-step latency of online_wpe_step
at (F, D, taps) = (257, 8, 10), delay 2, on CUDA tensors; and the whole-stream time at F = 132 .. 528 bins, to show
the cost of each wave of one CTA per bin over the 132 SMs.  Times are CUDA events around calls of the public
functions (median of 5 repeats; the wrapper's host work is included).  Yardsticks: the same step loop in torch
complex128 on the device (batched matmuls, one step per frame) and the NumPy oracle (oracle/wpe_online_oracle.py) on
the host, timed over the first ORACLE_FRAMES frames and scaled to T.  FLOPs: 3 n^2 complex multiply-adds (8 FLOP
each) per bin and frame, n = taps D (u = Q w, v = w^H Q and the rank-1 update); the kernel runs them on the FP64
units (DFMA), so its rate is set against the 34 TFLOP/s FP64 (non-tensor) figure of the H100 SXM data sheet.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import wpe_online_oracle as O  # noqa: E402
from pb_bss_b200.wpe import online_wpe, online_wpe_step  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

FP64_FLOPS = 34e12
ALPHA = 0.9999
STREAMS = ((257, 8, 10, 2, 500), (513, 8, 10, 2, 500), (513, 2, 10, 2, 2000), (513, 8, 12, 2, 4000))
WAVES = (132, 264, 396, 513, 528)
ORACLE_FRAMES = 100
SMS = 132


def flops(F, D, taps, T):
    n = taps * D
    return 8.0 * 3 * n * n * F * T


def torch_stream(Y, taps, delay, alpha):
    """The step loop in torch complex128 on the device."""
    T, F, D = Y.shape
    n, L = taps * D, taps + delay + 1
    stream = torch.cat([torch.zeros((L - 1, F, D), dtype=Y.dtype, device=Y.device), Y])
    Q = torch.eye(n, dtype=Y.dtype, device=Y.device).expand(F, n, n).contiguous()
    G = torch.zeros((F, n, D), dtype=Y.dtype, device=Y.device)
    Z = torch.empty_like(Y)
    for t in range(T):
        buf = stream[t:t + L]
        lam = (buf.real ** 2 + buf.imag ** 2).mean(dim=(0, 2))
        Z[t], Q, G = torch_step(buf, lam, Q, G, alpha, taps, delay)
    return Z


def torch_step(buf, lam, Q, G, alpha, taps, delay):
    F, D = buf.shape[1:]
    w = buf[:-delay - 1].flip(0).permute(1, 2, 0).reshape(F, taps * D)
    pred = buf[-1] - (G.conj().transpose(1, 2) @ w[:, :, None])[..., 0]
    u = (Q @ w[:, :, None])[..., 0]
    den = alpha * lam + (w.conj() * u).sum(-1)
    k = u / den[:, None]
    v = (w.conj()[:, None, :] @ Q)[:, 0]
    Q = (Q - k[:, :, None] * v[:, None, :]) / alpha
    G = G + k[:, :, None] * pred.conj()[:, None, :]
    return pred, Q, G


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'alpha': ALPHA, 'streams': {}, 'waves': {}}
    for F, D, taps, delay, T in STREAMS:
        rng = np.random.default_rng(F + D + T)
        Y = rng.standard_normal((T, F, D)) + 1j * rng.standard_normal((T, F, D))
        y = torch.from_numpy(Y).cuda()
        s, all_s = device_seconds(lambda: online_wpe(y, taps, delay, ALPHA), calls=3)
        ts, _ = device_seconds(lambda: torch_stream(y, taps, delay, ALPHA), calls=1, repeats=3)
        Zd = online_wpe(y, taps, delay, ALPHA)[0]
        err = ((torch_stream(y, taps, delay, ALPHA) - Zd).abs().max() / y.abs().max()).item()
        Yo = Y[:ORACLE_FRAMES]
        oracle_s = host_seconds(lambda: O.online_wpe(Yo, taps, delay, ALPHA), repeats=1) * T / len(Yo)
        fl = flops(F, D, taps, T)
        waves = -(-F // SMS)
        rec = {'F': F, 'D': D, 'taps': taps, 'delay': delay, 'T': T, 'device_ms': s * 1e3,
               'device_ms_all': [v * 1e3 for v in all_s], 'gflop': fl / 1e9,
               'share_of_fp64_peak': fl / s / FP64_FLOPS, 'waves': waves,
               'us_per_frame_per_wave': s * 1e6 / (waves * T),
               'torch_complex128_ms': ts * 1e3, 'torch_max_rel_diff': err,
               'oracle_host_ms_scaled': oracle_s * 1e3}
        result['streams'][f'F{F}_D{D}_taps{taps}_T{T}'] = rec
        print(json.dumps(rec), flush=True)
    # one step at (257, 8, 10)
    F, D, taps, delay = 257, 8, 10, 2
    rng = np.random.default_rng(0)
    n = taps * D
    buf = torch.from_numpy(rng.standard_normal((taps + delay + 1, F, D)) + 0j).cuda()
    lam = torch.ones(F, dtype=torch.float64, device='cuda')
    Q = torch.eye(n, dtype=torch.complex128, device='cuda').expand(F, n, n).contiguous()
    G = torch.zeros((F, n, D), dtype=torch.complex128, device='cuda')
    s, _ = device_seconds(lambda: online_wpe_step(buf, lam, Q, G, ALPHA, taps, delay), calls=50)
    ts, _ = device_seconds(lambda: torch_step(buf, lam, Q, G, ALPHA, taps, delay), calls=50)
    b, q, g = buf.cpu().numpy(), Q.cpu().numpy(), G.cpu().numpy()
    oracle_s = host_seconds(lambda: O.online_wpe_step(b, np.ones(F), q, g, ALPHA, taps, delay), repeats=5)
    result['step'] = {'F': F, 'D': D, 'taps': taps, 'delay': delay, 'device_us': s * 1e6,
                      'torch_complex128_us': ts * 1e6, 'oracle_host_us': oracle_s * 1e6}
    print(json.dumps(result['step']), flush=True)
    # waves of one CTA per bin
    for F in WAVES:
        D, taps, delay, T = 8, 10, 2, 500
        y = torch.from_numpy(np.random.default_rng(F).standard_normal((T, F, D)) + 0j).cuda()
        s, _ = device_seconds(lambda: online_wpe(y, taps, delay, ALPHA), calls=3)
        result['waves'][F] = {'device_ms': s * 1e3, 'waves': -(-F // SMS)}
        print(F, json.dumps(result['waves'][F]), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
