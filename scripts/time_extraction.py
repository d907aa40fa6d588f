"""Device time per call of get_lcmv_vector and apply_online_beamforming_vector, next to the reference's CPU time in
the same run, with the GPU name and power limit.

    python scripts/time_extraction.py [--out result.json]

L1: get_lcmv_vector, K = 3 ATFs, F = 513, D = 8 (inputs on the device).
O1 / O2: apply_online_beamforming_vector, T = 500, F = 513, D = 8, complex128 / complex64 mix.  Achieved bandwidth
counts the algorithmic bytes once: vector (T F D complex128) + mix (F D T of the mix dtype) + out (F T complex128),
against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM; it is taken from the kernel time (the C entry called
directly into a preallocated output), while device_ms_per_call is the public function with its host-side work.
A device time is the median over repeats of (CUDA-event time of N calls) / N after a warm-up.  The reference
(oracle/_ref, built by __graft_entry__.build() from a reference checkout) runs the same call on the host.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim, synth  # noqa: E402
from pb_bss_b200 import _lib, extraction as E  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def device_seconds(fn, calls=50, repeats=5):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(calls):
            fn()
        end.record()
        torch.cuda.synchronize()
        out.append(start.elapsed_time(end) * 1e-3 / calls)
    return float(np.median(out)), out


def host_seconds(fn, repeats=3):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-reference', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    RB = None
    if not args.no_reference and ref_shim.available():
        RB = ref_shim.load().beamformer
    result = {'gpu': gpu_info(), 'configs': {}}
    rng = np.random.RandomState(0)

    K, F, D = 3, 513, 8
    atf = rng.randn(K, F, D) + 1j * rng.randn(K, F, D)
    noise = synth.pos_def_hermitian(F, D, D, seed=1)
    resp = np.array([1, 1e-3, 1e-3])
    a_d, n_d, r_d = (torch.from_numpy(x).cuda() for x in (atf, noise, resp))
    s, all_s = device_seconds(lambda: E.get_lcmv_vector(a_d, r_d, n_d))
    rec = {'K': K, 'F': F, 'D': D, 'device_ms_per_call': s * 1e3, 'device_ms_all': [x * 1e3 for x in all_s]}
    if RB is not None:
        rec['reference_cpu_ms_per_call'] = host_seconds(lambda: RB.get_lcmv_vector(atf, resp, noise)) * 1e3
    result['configs']['L1_lcmv'] = rec
    print('L1_lcmv', json.dumps(rec), flush=True)

    T = 500
    v = rng.randn(T, F, D) + 1j * rng.randn(T, F, D)
    mix = rng.randn(F, D, T) + 1j * rng.randn(F, D, T)
    for name, dt, es in (('O1_online_c128', np.complex128, 16), ('O2_online_c64', np.complex64, 8)):
        m = mix.astype(dt)
        v_d, m_d = torch.from_numpy(v).cuda(), torch.from_numpy(m).cuda()
        s, all_s = device_seconds(lambda: E.apply_online_beamforming_vector(v_d, m_d), calls=200)
        # the C entry alone, output preallocated: the kernel without the Python wrapper's per-call host work
        lib, out = _lib.load(), torch.empty(F, T, dtype=torch.complex128, device='cuda')
        code = _lib.PBB_C128 if dt == np.complex128 else _lib.PBB_C64
        stream = torch.cuda.current_stream().cuda_stream
        k, _ = device_seconds(lambda: lib.pbb_apply_online_beamforming_vector(
            v_d.data_ptr(), m_d.data_ptr(), code, 1, F, D, T, F * D, D, 0, D * T, out.data_ptr(), stream), calls=200)
        nbytes = T * F * D * 16 + F * D * T * es + F * T * 16
        rec = {'T': T, 'F': F, 'D': D, 'mix_dtype': np.dtype(dt).name, 'device_ms_per_call': s * 1e3,
               'device_ms_all': [x * 1e3 for x in all_s], 'kernel_ms_per_call': k * 1e3,
               'algorithmic_bytes': nbytes, 'achieved_GB_per_s': nbytes / k * 1e-9,
               'share_of_3.35TB_per_s': nbytes / k / HBM_BYTES_PER_S}
        if RB is not None:
            rec['reference_cpu_ms_per_call'] = host_seconds(lambda: RB.apply_online_beamforming_vector(v, m)) * 1e3
        result['configs'][name] = rec
        print(name, json.dumps(rec), flush=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
