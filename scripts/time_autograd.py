"""Time the differentiable mask-based beamforming chain on the device against the same chain restated in torch
(oracle/autograd_oracle.py and oracle/bf_autograd_oracle.py, cuFFT / cuBLAS / cuSOLVER through torch) on the same
GPU, with the GPU name and power limit read in the same run.

    python scripts/time_autograd.py [--beamformer souden|gev+ban|pca+mvdr|rank1_gev+mvdr_souden]
                                    [--out result.json] [--trace-dir DIR]

Shape: F = 257, D = 6, T = 1002 frames, size 512, shift 128 (an 8 s, 16 kHz six-channel STFT).  The chain is
float32 mask logits -> sigmoid -> PSD (target, noise) -> beamformer -> apply -> istft -> -si_sdr.  The beamformer is
the Souden MVDR (automatic reference channel; the default) or one of get_bf_vector's gev+ban, pca+mvdr and
rank1_gev+mvdr_souden (reference channel 0); the torch side restates it with the eigenvectors' phase aligned to the
device's.  Forward and forward + backward times are medians of CUDA-event windows over several calls after a warm-up
(the forward synchronises once to pick the reference channel, on both sides).  A separate profiled run (torch.profiler,
CUDA activity) gives each backward kernel's time; with the kernel's algorithmic bytes (each array it must read or
write, once) it gives the achieved bandwidth and the share of the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM.
The STFT backward is not on the chain (the observation is a constant there) and is profiled on its own, on the
six-channel signal.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import autograd_oracle as AO  # noqa: E402
from oracle import bf_autograd_oracle as BO  # noqa: E402
from pb_bss_b200.evaluation import si_sdr  # noqa: E402
from pb_bss_b200.extraction import beamformer as B  # noqa: E402
from pb_bss_b200.extraction import beamformer_wrapper as W  # noqa: E402
from pb_bss_b200.transform import istft, stft  # noqa: E402
from scripts.time_embedding_mm import gpu_info  # noqa: E402
from scripts.time_extraction import device_seconds  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZE, SHIFT, D = 512, 128, 6
N = 999 * SHIFT - 3


BEAMFORMERS = ('souden', 'gev+ban', 'pca+mvdr', 'rank1_gev+mvdr_souden')


def torch_beamformer(name, pt, pn, phase):
    """get_bf_vector(name) restated in torch; phase: the device's eigenvector (the GEV or PCA vector), whose per-bin
    phase the restatement takes (oracle/bf_autograd_oracle.py: fix_phase)"""
    if name == 'gev+ban':
        return BO.blind_analytic_normalization(BO.gev_vector(pt, pn, phase)[0], pn)
    if name == 'pca+mvdr':
        return BO.mvdr_vector(BO.pca(pt, phase)[1], pn)
    a = BO.matvec(pn, BO.gev_vector(pt, pn, phase)[0])  # rank1_gev+mvdr_souden
    return AO.mvdr_vector_souden(BO.rank_one_estimate(a, pt), pn, 0)[0]


def device_phase(name, pt, pn):
    """the device's eigenvector of the chain, for the torch side's phase"""
    with torch.no_grad():
        return B.get_pca_vector(pt) if name == 'pca+mvdr' else B.get_gev_vector(pt, pn)


def chain(torch_side, y, logits, target, ref_channel=None, beamformer='souden', phase=None):
    mask = torch.sigmoid(logits)
    if torch_side:
        pt = AO.power_spectral_density(y, mask[:, 0])
        pn = AO.power_spectral_density(y, mask[:, 1])
        if beamformer == 'souden':
            w, ref = AO.mvdr_vector_souden(pt, pn, ref_channel)
        else:
            w, ref = torch_beamformer(beamformer, pt, pn, phase), None
        x = AO.istft(AO.apply_beamforming_vector(w, y).transpose(0, 1), SIZE, SHIFT)
        return -AO.si_sdr(target, x[:target.shape[-1]]), ref
    pt = B.get_power_spectral_density_matrix(y, mask[:, 0])
    pn = B.get_power_spectral_density_matrix(y, mask[:, 1])
    if beamformer == 'souden':
        w, ref = B.get_mvdr_vector_souden(pt, pn, ref_channel, return_ref_channel=True)
    else:
        kw = {'ref_channel': 0} if 'souden' in beamformer else {}
        w, ref = W.get_bf_vector(beamformer, pt, pn, **kw), None
    x = istft(B.apply_beamforming_vector(w, y).transpose(0, 1), size=SIZE, shift=SHIFT)
    return -si_sdr(target, x[:target.shape[-1]]), ref


def kernel_bytes(F, T, n_out, rows_stft, frames_stft, pencil=True):
    """Algorithmic bytes of one call of each backward kernel at this shape (complex128 16 B, float64 8 B)."""
    c, r, wl, bins = 16, 8, SIZE, SIZE // 2 + 1
    return {
        # Y read, grad Y written, the mask read and its gradient written (K = 1 per call); G and Phi are small
        'psd_backward_kernel': F * D * T * c * 2 + F * T * r * 2 + F * D * D * c * 2,
        'souden_backward_kernel': F * D * D * c * 2 + F * D * c,
        'solve_kernel': F * D * D * c * 3,
        'souden_noise_backward_kernel': F * D * D * c * 3,
        'apply_bf_vector_backward_kernel': F * D * T * c + F * T * c + F * D * c,
        'apply_bf_mix_backward_kernel': F * D * T * c + F * T * c + F * D * c,
        'istft_backward_kernel': n_out * r + T * bins * c,
        'si_sdr_backward_kernel': 3 * N * r,
        'stft_backward_kernel': rows_stft * frames_stft * (bins * c + wl * r),
        # the get_bf_vector backward kernels: A and B (or N) read, their gradients written, the vectors
        'eig_backward_kernel': F * D * D * c * (4 if pencil else 2) + 2 * F * D * c,
        'mvdr_backward_rhs_kernel': 4 * F * D * c + F * D * c,
        'mvdr_backward_kernel': F * D * c * 4 + F * D * D * c + F * D * c,
        'ban_backward_kernel': F * D * D * c * 2 + 3 * F * D * c,
        'rank_one_backward_kernel': F * D * D * c * 3 + 2 * F * D * c,
        'matvec_backward_kernel': F * D * D * c * 2 + 3 * F * D * c,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--trace-dir', default=None)
    ap.add_argument('--beamformer', default='souden', choices=BEAMFORMERS)
    args = ap.parse_args()
    bf = args.beamformer
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    sig = torch.tensor(rng.standard_normal((D, N)), device='cuda')
    y = stft(sig, size=SIZE, shift=SHIFT).permute(2, 0, 1).contiguous()  # (F, D, T)
    F, _, T = y.shape
    logits = torch.tensor(rng.standard_normal((F, 2, T)), dtype=torch.float32, device='cuda', requires_grad=True)
    target = torch.tensor(rng.standard_normal(N), device='cuda')
    _, ref = chain(False, y, logits, target, beamformer=bf)
    phase = None
    if bf in ('gev+ban', 'pca+mvdr', 'rank1_gev+mvdr_souden'):
        with torch.no_grad():
            mask = torch.sigmoid(logits)
            phase = device_phase(bf, B.get_power_spectral_density_matrix(y, mask[:, 0]),
                                 B.get_power_spectral_density_matrix(y, mask[:, 1]))
    result = {'gpu': gpu_info(), 'beamformer': bf, 'F': F, 'D': D, 'T': T, 'size': SIZE, 'shift': SHIFT,
              'samples': N, 'reference_channel': ref if bf == 'souden' else (0 if 'souden' in bf else None),
              'chain': {}}

    def fwd(torch_side):
        with torch.no_grad():
            chain(torch_side, y, logits, target, ref if torch_side else None, bf, phase)

    def fwd_bwd(torch_side):
        loss, _ = chain(torch_side, y, logits, target, ref if torch_side else None, bf, phase)
        torch.autograd.grad(loss, logits)

    # alternate the two sides so that drift on the shared machine hits both
    times = {k: [] for k in ('device_forward', 'device_forward_backward', 'torch_forward', 'torch_forward_backward')}
    for _ in range(3):
        for side, name in ((False, 'device'), (True, 'torch')):
            times[name + '_forward'].append(device_seconds(lambda: fwd(side), calls=20)[0])
            times[name + '_forward_backward'].append(device_seconds(lambda: fwd_bwd(side), calls=20)[0])
    result['chain'] = {k: {'ms_median': float(np.median(v)) * 1e3, 'ms_all': [t * 1e3 for t in v]}
                       for k, v in times.items()}

    # profiled run: one chain backward and one STFT backward of the six-channel signal
    x = sig.clone().requires_grad_()
    X = stft(x, size=SIZE, shift=SHIFT)
    gX = torch.randn_like(X)
    for _ in range(3):
        fwd_bwd(False)
        torch.autograd.grad(X, x, gX, retain_graph=True)
    torch.cuda.synchronize()
    steps = 10
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            loss, _ = chain(False, y, logits, target, beamformer=bf)
            torch.autograd.grad(loss, logits)
            torch.autograd.grad(X, x, gX, retain_graph=True)
        torch.cuda.synchronize()
    if args.trace_dir:
        os.makedirs(args.trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace_dir, 'time_autograd.pt.trace.json'))
    nbytes = kernel_bytes(F, T, T * SHIFT - SHIFT - (SIZE - SHIFT), D, T, pencil=bf != 'pca+mvdr')
    kernels = {}
    for evt in prof.key_averages():
        name = evt.key
        base = next((k for k in nbytes if k in name), None)
        if base is None:
            continue
        # solve_kernel runs once in the forward and once in the backward at the same shape; overlap_add_kernel, which
        # the STFT backward shares with the forward iSTFT at another shape, is left out
        if base == 'solve_kernel' or 'backward' in name:
            dev_us = getattr(evt, 'device_time_total', None)
            if dev_us is None:
                dev_us = evt.cuda_time_total
            per_call_s = dev_us * 1e-6 / evt.count
            k = kernels.setdefault(base, {'calls_per_step': 0, 'us_per_call': [], 'names': []})
            k['calls_per_step'] += evt.count / steps
            k['us_per_call'].append(per_call_s * 1e6)
            k['names'].append(name)
    for base, k in kernels.items():
        us = float(np.mean(k['us_per_call']))
        k['us_per_call'] = us
        k['algorithmic_bytes'] = nbytes[base]
        k['achieved_GB_per_s'] = nbytes[base] / (us * 1e-6) * 1e-9
        k['share_of_3.35TB_per_s'] = nbytes[base] / (us * 1e-6) / HBM_BYTES_PER_S
    result['backward_kernels'] = kernels
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
