"""Host time per enqueue of a library call through _device.call, against the same call written out by hand as
lib.pbb_x(_device.ptr(a), ..., _device.stream_ptr()) + _lib.check, in one process, with the GPU name and power limit.

    python scripts/time_abi_calls.py [--batches 400] [--batch 20] [--out result.json]

Calls: pbb_abs_square (4 arguments, 1k complex128 elements) and pbb_wpe (21 arguments, 4 bins, D = 2, T = 64,
taps = 3, delay = 1, one iteration).  Each batch enqueues `batch` calls of one form between perf_counter reads and
then synchronises outside the timed window; batches small enough that the launch queue never fills measure the host
alone.  The two forms alternate batch by batch; the medians over all batches are reported.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pb_bss_b200 import _device, _lib  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        limit = None
    return {'name': name, 'power_limit_w': limit}


def abs_square_forms():
    t = torch.randn(1024, dtype=torch.complex128, device='cuda')
    out = torch.empty(1024, dtype=torch.float64, device='cuda')
    code, n = _lib.PBB_C128, t.numel()
    lib = _lib.load()

    def helper():
        _device.call('pbb_abs_square', t, code, n, out)

    def by_hand():
        _lib.check(lib.pbb_abs_square(_device.ptr(t), code, n, _device.ptr(out), _device.stream_ptr()),
                   'pbb_abs_square')
    return helper, by_hand


def wpe_forms():
    bins, D, T, taps, delay, iterations, valid = 4, 2, 64, 3, 1, 1, 0
    y = torch.randn(bins, D, T, dtype=torch.complex128, device='cuda')
    out = torch.empty_like(y)
    ysb, ysd, yst = y.stride()
    osb, osd, ost = out.stride()
    lib = _lib.load()
    group = bins
    nbytes = lib.pbb_wpe_workspace_bytes(group, D, T, taps, delay, valid)
    ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    code, context = _lib.PBB_C128, 0

    def helper():
        _device.call('pbb_wpe', y, code, bins, D, T, ysb, ysd, yst, out, osb, osd, ost, taps, delay, iterations,
                     context, valid, group, ws, nbytes, status)

    def by_hand():
        _lib.check(lib.pbb_wpe(_device.ptr(y), code, bins, D, T, ysb, ysd, yst, _device.ptr(out), osb, osd, ost, taps,
                               delay, iterations, context, valid, group, _device.ptr(ws), nbytes, _device.ptr(status),
                               _device.stream_ptr()), 'pbb_wpe')
    return helper, by_hand


def measure(forms, batches, batch):
    per = {name: [] for name in forms}
    for _ in range(20):  # warm-up: module load, first launches
        for f in forms.values():
            f()
    torch.cuda.synchronize()
    for _ in range(batches):
        for name, f in forms.items():
            t0 = time.perf_counter()
            for _ in range(batch):
                f()
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            per[name].append((t1 - t0) / batch * 1e6)
    return {name: {'median_us': float(np.median(v)), 'p10_us': float(np.percentile(v, 10)),
                   'p90_us': float(np.percentile(v, 90))} for name, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, default=400)
    ap.add_argument('--batch', type=int, default=20)
    ap.add_argument('--out')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'batch': args.batch, 'batches': args.batches}
    for call, make in (('pbb_abs_square', abs_square_forms), ('pbb_wpe', wpe_forms)):
        helper, by_hand = make()
        r = measure({'call': helper, 'by_hand': by_hand}, args.batches, args.batch)
        r['extra_us'] = r['call']['median_us'] - r['by_hand']['median_us']
        result[call] = r
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
