"""Device time of pb_bss_b200.evaluation.mir_eval_sources at the shapes pb_bss evaluates, with the GPU name and power
limit read in the same run:
  - (K = 2, E = 2, T = 64000) with the permutation (OutputMetrics);
  - (K = 3, E = 4, T = 160000) with the permutation (K + 1 estimates: _bss_eval_sources_and_noise);
  - references (4, 6, 80000) without the permutation, as InputMetrics calls it (6 channels, 6 items).

    python scripts/time_bss_eval.py [--out result.json]

Times are CUDA events around calls of the public function on CUDA tensors (median of 5 repeats after a warm-up; the
wrapper's host work is included).  Per-kernel times come from torch.profiler in a separate run and are summed per
stage.  FLOPs per item (2 per multiply-add): correlation 2 K (K + E) L T; LU 2/3 N^3 + K 2/3 L^3 (N = 512 K,
L = 512); projections 2 (2 E K L T).  Each stage's rate is set against the 67 TFLOP/s fp64 tensor-core rate of the
H100 SXM data sheet.  Host: the NumPy restatement (oracle/bss_eval_oracle.py, np.linalg.solve), one call.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import bss_eval_oracle as O  # noqa: E402
from pb_bss_b200.evaluation import mir_eval_sources  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

FP64_TC_FLOPS = 67e12
L = 512
STAGES = {'correlation': ('bss_corr',), 'lu': ('bss_lu', 'bss_backsub', 'bss_assemble'),
          'projections': ('bss_project',), 'other': ('bss_check', 'bss_ratio', 'bss_status')}


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
        if t and 'bss_' in e.key:
            out[e.key.split('(')[0].replace('void ', '').replace('pbb::', '')[:80]] = t / calls
    return out


def stage_flops(items, K, E, T):
    N = K * L
    return {'correlation': items * 2.0 * K * (K + E) * L * T,
            'lu': items * (2.0 / 3 * N ** 3 + (K * 2.0 / 3 * L ** 3 if K > 1 else 0.0)),
            'projections': items * 2.0 * 2 * E * K * L * T}


def signals(K, E, middle, T, seed=0):
    rng = np.random.default_rng(seed)
    src = rng.standard_normal((K, *middle, T))
    mix = rng.standard_normal((E, K))
    est = np.einsum('ek,k...->e...', mix, src) + 0.1 * rng.standard_normal((E, *middle, T))
    return src, est


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    for name, K, E, middle, T, perm in (('K2_E2_T64000', 2, 2, (), 64000, True),
                                        ('K3_E4_T160000', 3, 4, (), 160000, True),
                                        ('input_4x6x80000', 4, 4, (6,), 80000, False)):
        src, est = signals(K, E, middle, T)
        r, e = torch.from_numpy(src).cuda(), torch.from_numpy(est).cuda()
        fn = lambda: mir_eval_sources(r, e, compute_permutation=perm)  # noqa: E731
        s, all_s = device_seconds(fn, calls=1)
        items = int(np.prod(middle))
        flops = stage_flops(items, K, E, T)
        kt = kernel_times(fn)
        stage_us = {st: sum(v for k, v in kt.items() if any(p in k for p in pre)) for st, pre in STAGES.items()}
        rec = {'K': K, 'E': E, 'items': items, 'T': T, 'compute_permutation': perm,
               'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s],
               'kernel_us_per_call': kt, 'stage_us_per_call': stage_us, 'stage_flops': flops,
               'stage_share_of_fp64_tc_peak': {st: flops[st] / (stage_us[st] * 1e-6) / FP64_TC_FLOPS
                                               for st in flops if stage_us[st] > 0}}
        rec['oracle_host_ms'] = host_seconds(lambda: O.mir_eval_sources(src, est, compute_permutation=perm),
                                             repeats=1) * 1e3
        result['configs'][name] = rec
        print(name, json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
