"""Deflation seed (pb_bss/initializer/deflation.py:6-89): class after class, take the most salient frames of every
bin, estimate a steering vector from them (saliency-weighted PSD -> principal component) and turn the similarity of
every frame to it into the class posterior; the saliency of the explained frames is deflated before the next class.

Every arithmetic step runs in the library's kernels: ``pbb_normalize_observation`` (unit-norm observation),
``pbb_power_spectral_density`` and ``pbb_heig_batched`` (steering vector), ``pbb_apply_beamforming_vector`` (the
similarity |z^H m|^2).  torch only selects the frames around the saliency maximum and rescales the saliency."""
import numpy as np
import torch

from .. import _device
from ..extraction import (apply_beamforming_vector, get_pca_vector,
                          get_power_spectral_density_matrix)


def _unit_norm(Y):
    """_parameterized_vector_norm over the last axis (permutation_alignment.py:358-377) of (F, T, D)."""
    F, T, D = Y.shape
    z = torch.empty_like(Y)
    _device.call('pbb_normalize_observation', Y, z, F, T, D, _device.complex_dtype_code(Y), 0)
    return z


def deflationSeed(Y, sources: int, saliencies=None, permutation_free: bool = True, neighbors: int = 5,
                  similarity_transform=None, eps=0):
    """Y (F, T, D) -> posterior (K, F, T), signature of deflation.py:6-14."""
    like_numpy = not _device.is_tensor(Y)
    Yd = _device.to_device(Y)
    if not Yd.is_complex():
        Yd = Yd.to(torch.complex128)
    Yd = Yd.contiguous()
    F, T, D = Yd.shape
    assert F in [257, 513], F
    if saliencies is None:
        sal = torch.linalg.vector_norm(Yd, dim=-1)
    else:
        sal = _device.to_device(saliencies, torch.float64)
    sal = sal.to(torch.float64)
    assert tuple(sal.shape) == (F, T), (sal.shape, (F, T))
    Z = _unit_norm(Yd)
    Zt = Z.transpose(-1, -2).contiguous()                      # (F, D, T) for the beamforming kernel
    offsets = torch.arange(-neighbors, neighbors + 1, device=Yd.device)
    rows = torch.arange(F, device=Yd.device)
    posterior = []
    for _ in range(sources - 1):
        if permutation_free:
            maxidx = torch.argmax(sal.mean(dim=0), dim=-1).repeat(F)
        else:
            maxidx = torch.argmax(sal, dim=-1)
        maxidx = torch.clamp(maxidx, neighbors, T - 1 - neighbors)
        idx = maxidx[:, None] + offsets[None, :]                # (F, 2 neighbors + 1)
        Y_local = Yd[rows[:, None], idx, :].transpose(-1, -2).contiguous()   # (F, D, T_local)
        sal_local = sal[rows[:, None], idx].contiguous()
        psd = get_power_spectral_density_matrix(Y_local, mask=sal_local)
        mode = get_pca_vector(psd)                              # unit norm (F, D)
        # |sum_d conj(z_d) m_d|^2 = |apply_beamforming_vector(m, z)|^2
        similarity = apply_beamforming_vector(mode, Zt).abs() ** 2
        if similarity_transform is not None:
            similarity = similarity_transform(similarity, sal)
        posterior.append(similarity)
        sal = sal * (1 - similarity)
    post = torch.stack(posterior, dim=0)
    post = torch.cat([post, (1 - post.sum(dim=0))[None]], dim=0)   # the last class takes the rest
    post = torch.clamp(post, min=eps)
    post = post / post.sum(dim=0, keepdim=True)
    return _device.to_host(post, like_numpy)
