"""Device time of pb_bss_b200.transform.stft / istft at a user-sized shape, (8, 128000) float64 (8 channels, 8 s at
16 kHz), size 1024, shift 256, fading (T = 503), and of 100 Griffin-Lim steps, with the GPU name and power limit read
in the same run.

    python scripts/time_stft.py [--out result.json]

Times are CUDA events around N calls of the public function on CUDA tensors (median over repeats after a warm-up; the
wrapper's host work is included, the launches are asynchronous).  The algorithmic bytes count the signal read once and
the spectrum written once (the forward: 8.2 MB in, 33.0 MB out); the share is of the 3.35 TB/s HBM3 data-sheet figure
of the H100 SXM.  The FFT work (about 0.1 GFLOP fp64) is far below the time that traffic takes, so the bytes bound it.
Yardstick: torch.stft / torch.istft (cuFFT) on the same tensor with centre padding, which frames the signal slightly
differently.  Host: the NumPy restatement of the contract (oracle/transform_oracle.py), not nara_wpe.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import transform_oracle as TO  # noqa: E402
from pb_bss_b200 import transform  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _rec(s, all_s, nbytes):
    return {'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s], 'algorithmic_bytes': nbytes,
            'achieved_GB_per_s': nbytes / s * 1e-9, 'share_of_3.35TB_per_s': nbytes / s / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    C, n, size, shift = 8, 128000, 1024, 256
    x_host = np.random.RandomState(0).randn(C, n)
    x = torch.from_numpy(x_host).cuda()
    X = transform.stft(x, size=size, shift=shift)
    T, F = X.shape[-2], X.shape[-1]
    sig_bytes, spec_bytes = C * n * 8, C * T * F * 16
    result = {'gpu': gpu_info(), 'shape': [C, n], 'size': size, 'shift': shift, 'frames': T, 'configs': {}}

    s, all_s = device_seconds(lambda: transform.stft(x, size=size, shift=shift), calls=100)
    fwd = _rec(s, all_s, sig_bytes + spec_bytes)
    s, all_s = device_seconds(lambda: transform.istft(X, size=size, shift=shift), calls=100)
    inv = _rec(s, all_s, spec_bytes + sig_bytes)
    win = torch.from_numpy(TO.analysis_window(size)).cuda()
    ts = torch.stft(x, size, shift, window=win, center=True, pad_mode='constant', return_complex=True)
    fwd['torch_yardstick_ms_per_call'] = device_seconds(
        lambda: torch.stft(x, size, shift, window=win, center=True, pad_mode='constant', return_complex=True),
        calls=100)[0] * 1e3
    inv['torch_yardstick_ms_per_call'] = device_seconds(
        lambda: torch.istft(ts, size, shift, window=win, center=True), calls=100)[0] * 1e3
    fwd['numpy_restatement_host_ms_per_call'] = host_seconds(lambda: TO.stft(x_host, size=size, shift=shift)) * 1e3
    X_host = X.cpu().numpy()
    inv['numpy_restatement_host_ms_per_call'] = host_seconds(lambda: TO.istft(X_host, size=size, shift=shift)) * 1e3
    result['configs']['stft'], result['configs']['istft'] = fwd, inv
    print('stft', json.dumps(fwd), flush=True)
    print('istft', json.dumps(inv), flush=True)

    # Griffin-Lim: 3 sources of 8 s, the reference's size 512 / shift 128, 100 steps per timed call
    K, gsize, gshift = 3, 512, 128
    Xg = transform.stft(x[:K], size=gsize, shift=gshift, fading=False)
    gl = transform.GriffinLim(Xg, size=gsize, shift=gshift)

    def hundred_steps():
        for _ in range(100):
            gl.step()

    s, all_s = device_seconds(hundred_steps, calls=1, repeats=3)
    rec = {'device_ms_per_100_steps': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s],
           'shape': list(Xg.shape), 'size': gsize, 'shift': gshift}
    Xg_host = Xg.cpu().numpy()
    rec['numpy_restatement_host_ms_first_guess_and_one_step'] = host_seconds(
        lambda: TO.griffin_lim(Xg_host, size=gsize, shift=gshift, steps=1), repeats=1) * 1e3
    result['configs']['griffin_lim_100_steps'] = rec
    print('griffin_lim', json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
