"""Pure-torch restatement of the six differentiable forwards of pb_bss_b200 (framing + torch.fft, torch.linalg.solve,
einsums), so that torch's own autograd gives the reference gradients of the device backward passes.  Runs on CPU or
CUDA tensors in float64 / complex128.  Test infrastructure only, like the rest of oracle/.

Closed forms of the gradients (PyTorch's convention grad z = dL/dRe z + i dL/dIm z) are restated next to the forwards
for the CPU tests that check them against autograd."""
import math

import numpy as np
import scipy.signal
import torch

from . import transform_oracle as TO


def _windows(size, shift, window_length, window, symmetric_window, device):
    wa = TO.analysis_window(size, window, window_length, symmetric_window)
    ws = TO.synthesis_window(wa, shift)
    return torch.from_numpy(wa).to(device), torch.from_numpy(ws).to(device)


def stft(x, size=1024, shift=256, window=scipy.signal.windows.blackman, window_length=None, fading=True, pad=True,
         symmetric_window=False):
    """nara_wpe stft over the last axis of a real tensor: (..., n) -> (..., T, size // 2 + 1)."""
    wl = window_length or size
    wa, _ = _windows(size, shift, window_length, window, symmetric_window, x.device)
    n = x.shape[-1]
    T = TO.num_frames(n, size, shift, window_length, fading, pad)
    off = wl - shift if fading else 0
    total = max(T - 1, 0) * shift + wl
    keep = min(n, total - off)
    padded = torch.nn.functional.pad(x[..., :keep].to(torch.float64), (off, total - off - keep))
    idx = (torch.arange(T, device=x.device)[:, None] * shift + torch.arange(wl, device=x.device)[None, :])
    frames = padded[..., idx] * wa
    return torch.fft.rfft(frames, n=size, dim=-1)


def istft(X, size=1024, shift=256, window=scipy.signal.windows.blackman, fading=True, window_length=None,
          symmetric_window=False):
    """nara_wpe istft: (..., T, size // 2 + 1) -> (..., T shift + wl - shift [- 2 (wl - shift)])."""
    wl = window_length or size
    _, ws = _windows(size, shift, window_length, window, symmetric_window, X.device)
    T = X.shape[-2]
    frames = torch.fft.irfft(X, n=size, dim=-1)[..., :wl] * ws
    full = T * shift + wl - shift
    idx = (torch.arange(T, device=X.device)[:, None] * shift + torch.arange(wl, device=X.device)[None, :]).reshape(-1)
    out = torch.zeros(X.shape[:-2] + (full,), dtype=torch.float64, device=X.device)
    out = out.index_add(-1, idx, frames.reshape(X.shape[:-2] + (T * wl,)))
    if fading:
        out = out[..., wl - shift:full - (wl - shift)]
    return out


def power_spectral_density(observation, mask=None, normalize=True):
    """observation (..., D, T); mask None, (..., T) or (..., K, T) -> (..., D, D) or (..., K, D, D)."""
    y = observation.to(torch.complex128)
    if mask is None:
        return torch.einsum('...dt,...et->...de', y, y.conj()) / y.shape[-1]
    m = mask.to(torch.float64)
    if normalize:
        m = m / torch.clamp(m.sum(-1, keepdim=True), min=1e-10)
    if m.dim() + 1 == y.dim():
        return torch.einsum('...t,...dt,...et->...de', m.to(y.dtype), y, y.conj())
    return torch.einsum('...kt,...dt,...et->...kde', m.to(y.dtype), y, y.conj())


def mvdr_vector_souden(target_psd, noise_psd, ref_channel=None, eps=None):
    """(w, ref_channel): w = mat[..., ref], mat = solve(noise, target) / max(Re tr, eps); the SNR rule picks ref."""
    phi = torch.linalg.solve(noise_psd, target_psd)
    lam = torch.diagonal(phi, dim1=-2, dim2=-1).sum(-1).real[..., None, None]
    eps = np.finfo(np.float64).tiny if eps is None else eps
    mat = phi / torch.clamp(lam, min=eps)
    if ref_channel is None:
        with torch.no_grad():
            num = torch.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), target_psd, mat)
            den = torch.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), noise_psd, mat)
            snr = num / torch.clamp(den.real, min=eps)
            ref_channel = int(torch.argmax(snr.real))
    return mat[..., ref_channel], ref_channel


def apply_beamforming_vector(vector, mix):
    """sum_a conj(vector[..., a]) mix[..., a, t]."""
    return torch.einsum('...a,...at->...t', vector.conj(), mix.to(torch.complex128))


def si_sdr(reference, estimation):
    """10 log10(|alpha r|^2 / |e - alpha r|^2), alpha = <r, e> / <r, r>, over the last axis after broadcasting."""
    e, r = torch.broadcast_tensors(estimation, reference)
    alpha = (r * e).sum(-1, keepdim=True) / (r * r).sum(-1, keepdim=True)
    p = alpha * r
    q = e - p
    return 10 * torch.log10((p * p).sum(-1) / (q * q).sum(-1))


# ---- closed forms of the gradients (restated from include/pbb.h) ----------------------------------------------------

def si_sdr_grad(reference, estimation, grad):
    """(grad r, grad e) of si_sdr for 1-D reference / estimation and a scalar incoming gradient."""
    alpha = (reference @ estimation) / (reference @ reference)
    p = alpha * reference
    q = estimation - p
    P, Q = p @ p, q @ q
    c = 20 / math.log(10) * grad
    return c * alpha * (1 / P + 1 / Q) * q, c * (p / P - q / Q)


def psd_grad(observation, mask, grad_psd, normalize=True):
    """(grad y, grad mask) of power_spectral_density for observation (F, D, T), mask (F, K, T), grad_psd (F, K, D, D)."""
    y = observation.to(torch.complex128)
    S = mask.sum(-1)
    if normalize:
        w = mask / torch.clamp(S, min=1e-10)[..., None]
    else:
        w = mask
    H = grad_psd + grad_psd.conj().transpose(-1, -2)
    gy = torch.einsum('fkt,fkde,fet->fdt', w.to(y.dtype), H, y)
    quad = torch.einsum('fdt,fkde,fet->fkt', y.conj(), grad_psd, y).real
    if not normalize:
        return gy, quad
    phi = power_spectral_density(y, mask, normalize=True)
    c = (grad_psd.conj() * phi).sum((-1, -2)).real
    active = S > 1e-10
    gm = torch.where(active[..., None], (quad - c[..., None]) / S[..., None], quad / 1e-10)
    return gy, gm


def souden_grad(target_psd, noise_psd, ref_channel, grad_w, eps=None):
    """(grad target, grad noise) of mvdr_vector_souden with a fixed reference channel."""
    eps = np.finfo(np.float64).tiny if eps is None else eps
    phi = torch.linalg.solve(noise_psd, target_psd)
    lam = torch.diagonal(phi, dim1=-2, dim2=-1).sum(-1).real
    D = phi.shape[-1]
    e_r = torch.zeros(D, dtype=phi.dtype)
    e_r[ref_channel] = 1
    outer = grad_w[..., :, None] * e_r
    c = (grad_w.conj() * phi[..., :, ref_channel]).sum(-1).real
    eye = torch.eye(D, dtype=phi.dtype)
    gphi = torch.where((lam > eps)[..., None, None], outer / lam[..., None, None] - (c / lam ** 2)[..., None, None] * eye,
                       outer / eps)
    gx = torch.linalg.solve(noise_psd.conj().transpose(-1, -2), gphi)
    gn = -gx @ phi.conj().transpose(-1, -2)
    return gx, gn
