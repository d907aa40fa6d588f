"""Device time of SI-SDR, the mean square and the OutputMetrics wrapper at user-sized shapes, with the GPU name and
power limit read in the same run:
  - si_sdr on (256, 160000) float64: a batch of 10-s utterances at 16 kHz;
  - get_variance_for_zero_mean_signal on one 2^26-sample row (axis=None);
  - OutputMetrics.as_dict() at the mixture-model notebook's shape (2 sources, 3 outputs, 6 channels' contributions
    summed, 8 kHz, 10 s), per metric and whole.

    python scripts/time_metrics.py [--out result.json]

Times are CUDA events around calls of the public functions on CUDA tensors (median of 5 repeats after a warm-up).
Algorithmic bytes: SI-SDR reads both signals in each of its two passes, 32 B per sample pair; the mean square reads
the signal once.  The bound is those bytes at 3.35 TB/s (HBM3, H100 SXM data sheet); whether pass 2 hits L2 is not
measured.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pb_bss_b200.evaluation import OutputMetrics, si_sdr  # noqa: E402
from pb_bss_b200.evaluation.sxr_module import get_variance_for_zero_mean_signal  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _rec(seconds, all_s, nbytes):
    bound = nbytes / HBM_BYTES_PER_S
    return {'device_ms_per_call': seconds * 1e3, 'device_ms_all': [v * 1e3 for v in all_s], 'bytes': nbytes,
            'hbm_bound_ms': bound * 1e3, 'share_of_hbm_bound': bound / seconds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info()}
    rng = np.random.default_rng(0)

    r = torch.from_numpy(rng.standard_normal((256, 160000))).cuda()
    e = r * 0.8 + 0.1 * torch.from_numpy(rng.standard_normal((256, 160000))).cuda()
    s, all_s = device_seconds(lambda: si_sdr(r, e), calls=20)
    result['si_sdr_256x160000'] = _rec(s, all_s, 2 * 2 * 8 * r.numel())
    print(json.dumps(result['si_sdr_256x160000']), flush=True)
    del r, e

    x = torch.from_numpy(rng.standard_normal(1 << 26)).cuda()
    s, all_s = device_seconds(lambda: get_variance_for_zero_mean_signal(x), calls=20)
    result['mean_square_2^26'] = _rec(s, all_s, 8 * x.numel())
    print(json.dumps(result['mean_square_2^26']), flush=True)
    del x

    K, Kt, D, fs, T = 2, 3, 6, 8000, 80000
    source = rng.standard_normal((K, T))
    mixing = rng.uniform(0, 1, (K, Kt, D))
    contribution = np.einsum('kt,kld->kldt', source, mixing).sum(-2)          # the channels summed per output
    noise = 0.1 * rng.standard_normal((Kt, T))
    prediction = contribution.sum(0) + noise
    dev = [torch.from_numpy(v).cuda() for v in (prediction, source, contribution, noise)]

    def make():
        return OutputMetrics(*dev, sample_rate=fs, enable_si_sdr=True)

    names = make()._available_metric_names()
    per = {}
    for name in names:
        def one(name=name):
            m = make()
            m._d_mir_eval                       # the selection every metric uses is computed first
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m[name]
            torch.cuda.synchronize()
            return time.perf_counter() - t0
        one()
        per[name] = float(np.median([one() for _ in range(5)])) * 1e3
    per['mir_eval (the selection)'], _ = device_seconds(lambda: make()._d_mir_eval, calls=3)
    per['mir_eval (the selection)'] *= 1e3
    whole, all_s = device_seconds(lambda: make().as_dict(), calls=3)
    result['output_metrics_notebook'] = {'shape': {'K_source': K, 'K_target': Kt, 'samples': T, 'sample_rate': fs},
                                         'as_dict_ms': whole * 1e3, 'as_dict_ms_all': [v * 1e3 for v in all_s],
                                         'per_metric_ms_after_selection': per}
    print(json.dumps(result['output_metrics_notebook']), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
