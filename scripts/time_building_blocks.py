"""Time the building blocks on the device: log_pdf_to_affiliation and estimate_mixture_weight at (F, K, T) =
(513, 3, 500) and (8 * 513, 6, 1000) with the (F, K, 1) weight, estimate_mixture_weight with the
frequency-tied weight_constant_axis=(-3, -1) at both shapes (K outputs, each a sum over F * T), and _unit_norm and
get_energy (axis=None: one output) of a (513, 500, 8) complex128 observation; next to a torch yardstick and the
reference on the CPU (when oracle/_ref is present), with the GPU name and power limit read in the same run.

    python scripts/time_building_blocks.py [--out result.json]

device_ms_per_call: the public function on CUDA tensors, CUDA events around N calls, median over repeats after a
warm-up (the wrapper's host work is included; launches are asynchronous).  kernel_ms_per_call: the same kernel
launched through the C entry point with its arguments prepared once, so it is the kernel plus one ctypes call.
Algorithmic bytes: every operand read once and the result written once; the share is of the 3.35 TB/s HBM3
data-sheet figure of the H100 SXM.  Yardsticks: torch.softmax(log_pdf + log weight) for the affiliation,
torch.mean / torch.linalg.vector_norm / torch.sum for the others.  The reference arm of get_energy evaluates the
reference's one-line expression (sxr_module.py:13-14) in NumPy, since oracle/_ref holds no evaluation modules.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim  # noqa: E402
from pb_bss_b200 import _device, _lib, _nd  # noqa: E402
from pb_bss_b200.distribution import mixture_model_utils as MMU  # noqa: E402
from pb_bss_b200.distribution.utils import _unit_norm  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds, host_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _affiliation_kernel(w, lp):
    """The launch of log_pdf_to_affiliation with its layout prepared once."""
    lib = _lib.load()
    out = torch.empty_like(lp)
    shape = tuple(lp.shape)
    ws = _nd.broadcast_strides(w, shape)
    lay = _nd.layout([shape[0], shape[2]], [lp.stride(0), lp.stride(2)], [ws[0], ws[2]], [0, 0],
                     [out.stride(0), out.stride(2)])
    cs = (ctypes.c_longlong * 4)(lp.stride(1), ws[1], 0, out.stride(1))
    args = (lp.data_ptr(), _lib.PBB_F64, w.data_ptr(), None, lay, shape[1], cs, 0.0, out.data_ptr(),
            _device.stream_ptr())
    return lambda: lib.pbb_affiliation_nd(*args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-reference', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    R = None
    if not args.no_reference and ref_shim.available():
        R = ref_shim.load().mixture_model_utils
    result = {'gpu': gpu_info(), 'configs': {}}
    rng = np.random.default_rng(0)

    def record(name, fn, nbytes, yard=None, ref=None, kernel=None, calls=100):
        s, all_s = device_seconds(fn, calls=calls)
        rec = {'device_ms_per_call': s * 1e3, 'device_ms_all': [v * 1e3 for v in all_s], 'algorithmic_bytes': nbytes,
               'achieved_GB_per_s': nbytes / s * 1e-9, 'share_of_3.35TB_per_s': nbytes / s / HBM_BYTES_PER_S}
        if kernel is not None:
            k, _ = device_seconds(kernel, calls=calls)
            rec['kernel_ms_per_call'] = k * 1e3
            rec['kernel_share_of_3.35TB_per_s'] = nbytes / k / HBM_BYTES_PER_S
        if yard is not None:
            rec['torch_yardstick_ms_per_call'] = device_seconds(yard, calls=calls)[0] * 1e3
        if ref is not None:
            rec['reference_cpu_ms_per_call'] = host_seconds(ref, repeats=1) * 1e3
        result['configs'][name] = rec
        print(name, json.dumps(rec), flush=True)

    for F, K, T in [(513, 3, 500), (8 * 513, 6, 1000)]:
        lp_h = rng.normal(scale=5, size=(F, K, T))
        w_h = rng.random((F, K, 1)) + 0.1
        aff_h = rng.random((F, K, T))
        lp, w, aff = (torch.from_numpy(a).cuda() for a in (lp_h, w_h, aff_h))
        logw = torch.log(w)
        n = F * K * T * 8
        record(f'log_pdf_to_affiliation_{F}x{K}x{T}', lambda: MMU.log_pdf_to_affiliation(w, lp), 2 * n + F * K * 8,
               yard=lambda: torch.softmax(lp + logw, dim=-2),
               ref=None if R is None else (lambda: R.log_pdf_to_affiliation(w_h, lp_h)),
               kernel=_affiliation_kernel(w, lp))
        record(f'estimate_mixture_weight_{F}x{K}x{T}', lambda: MMU.estimate_mixture_weight(aff), n + F * K * 8,
               yard=lambda: torch.mean(aff, dim=-1, keepdim=True),
               ref=None if R is None else (lambda: R.estimate_mixture_weight(aff_h)))
        # frequency-tied: K outputs, each a sum over F * T
        record(f'estimate_mixture_weight_tied_{F}x{K}x{T}',
               lambda: MMU.estimate_mixture_weight(aff, weight_constant_axis=(-3, -1)), n + K * 8,
               yard=lambda: torch.mean(aff, dim=(-3, -1), keepdim=True),
               ref=None if R is None else (lambda: R.estimate_mixture_weight(aff_h, weight_constant_axis=(-3, -1))))
    y_h = rng.normal(size=(513, 500, 8)) + 1j * rng.normal(size=(513, 500, 8))
    y = torch.from_numpy(y_h).cuda()
    ref_un = None
    if R is not None:
        import pb_bss.distribution.utils as dutils
        ref_un = (lambda: dutils._unit_norm(y_h))
    record('unit_norm_513x500x8_c128', lambda: _unit_norm(y), 2 * y_h.size * 16,
           yard=lambda: y / (torch.linalg.vector_norm(y, dim=-1, keepdim=True) + 1e-4), ref=ref_un)
    # get_energy with its default axis=None: one output, a sum over every element
    from pb_bss_b200.evaluation.sxr_module import get_energy
    ref_energy = None
    if R is not None:
        def ref_energy():
            return np.sum(np.abs(y_h * y_h.conj()))  # sxr_module.py:13-14
    record('get_energy_all_513x500x8_c128', lambda: get_energy(y), y_h.size * 16 + 8,
           yard=lambda: torch.sum(y.real ** 2 + y.imag ** 2), ref=ref_energy)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('total %.1f s' % (time.time() - t0))
