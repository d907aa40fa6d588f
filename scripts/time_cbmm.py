"""Device time per EM iteration of CBMMTrainer, the parameter solve on its own, and the reference's CPU time per
iteration, all from the same run, with the GPU name and power limit.

    python scripts/time_cbmm.py [--out result.json]

B1: F = 129, T = 200, D = 4, K = 2;  B2: F = 257, T = 500, D = 6, K = 3;  B3: 16 x B2 (F = 4112).
A device iteration is (t(21 iterations) - t(1 iteration)) / 20 between CUDA events, inputs already on the device.
The parameter solve (pbb_bingham_parameters, one warp per problem) is timed on the F K scatter spectra of the
shape.  The reference (oracle/_ref, built by __graft_entry__.build() from a reference checkout) runs 2 iterations
of its own CBMMTrainer on one thread; its time per iteration is the 2-iteration time / 2.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import bingham_oracle as B, ref_shim, synth  # noqa: E402
from pb_bss_b200.distribution import CBMMTrainer, ComplexBinghamTrainer  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402

CONFIGS = [('B1', 129, 200, 4, 2, True), ('B2', 257, 500, 6, 3, True), ('B3', 16 * 257, 500, 6, 3, False)]


def time_fit(y, init, iterations):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    CBMMTrainer().fit(y, initialization=init, iterations=iterations)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e-3


def time_solve(s, repeats=20):
    ComplexBinghamTrainer.find_eigenvalues_v3(s)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(repeats):
        ComplexBinghamTrainer.find_eigenvalues_v3(s)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e-3 / repeats


def reference_seconds_per_iteration(y, init):
    if not ref_shim.available():
        return None
    ref_shim.load()
    import pb_bss.distribution.cbmm as RC
    t0 = time.perf_counter()
    RC.CBMMTrainer().fit(y, initialization=init, iterations=2)
    return (time.perf_counter() - t0) / 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--no-reference', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {'gpu': gpu_info(), 'configs': {}}
    base = {}
    for name, F, T, D, K, with_ref in CONFIGS:
        if name == 'B3':
            y = np.concatenate([base['y']] * 16)
            init = np.concatenate([base['init']] * 16)
        else:
            y = synth.structured_stft(F, T, D, K, seed=F)[0]
            init = synth.init_affiliation(F, K, T, seed=K)
            base = dict(y=y, init=init)
        yd, idd = torch.from_numpy(y).cuda(), torch.from_numpy(init).cuda()
        time_fit(yd, idd, 2)  # warm-up (library load, allocator)
        per = [(time_fit(yd, idd, 21) - time_fit(yd, idd, 1)) / 20 for _ in range(args.repeats)]
        # the solve's inputs of the first M-step: scatter eigenvalues of every (bin, class)
        z = B.normalize_observation_cw(y[:F])
        s = np.linalg.eigvalsh(B.scatter(z[:, None], init[:F])).reshape(-1, D)
        solve = time_solve(torch.from_numpy(np.concatenate([s] * (len(y) // F))).cuda())
        rec = {'F': F, 'T': T, 'D': D, 'K': K, 'ms_per_iteration': float(np.median(per)) * 1e3,
               'ms_per_iteration_all': [p * 1e3 for p in per], 'parameter_solve_ms': solve * 1e3,
               'parameter_solve_problems': int(s.shape[0]) * (len(y) // F)}
        if with_ref and not args.no_reference:
            t = reference_seconds_per_iteration(y, init)
            rec['reference_cpu_s_per_iteration'] = t
            if t is not None:
                rec['speedup'] = t / (rec['ms_per_iteration'] * 1e-3)
        result['configs'][name] = rec
        print(name, json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
