"""String-dispatched beamformer construction, API of pb_bss/extraction/beamformer_wrapper.py.

``get_bf_vector('rank1_gev+mvdr_souden+ban', target_psd, noise_psd)`` chains the
device kernels of ``beamformer.py``: an optional rank-1 approximation of the
target PSD, the core beamformer, an optional blind analytic normalisation.

Every string get_bf_vector accepts is differentiable for CUDA tensors that
require grad, except ``chN`` (a constant vector) and ``wmwf`` (not built): the
rank-1 estimates and the scaled GEV ATF have device backward passes here
(pbb_rank_one_estimate_backward, pbb_matvec_batched_backward), the beamformers
theirs in ``beamformer.py``.  Through a GEV or PCA vector the gradient holds each
bin's eigenvector phase fixed (see ``beamformer.py``); the rank-1 estimates do
not depend on that phase, so their gradients are exact.
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _device
from .beamformer import (
    blind_analytic_normalization,
    get_gev_vector,
    get_mvdr_vector,
    get_mvdr_vector_souden,
    get_pca_vector,
)

__all__ = ['get_bf_vector', 'get_pca_rank_one_estimate', 'get_gev_rank_one_estimate']


def _rank_one(vector, covariance):
    like_numpy = not _device.is_tensor(covariance)
    a = _device.to_device(vector, torch.complex128)
    c = _device.to_device(covariance, torch.complex128)
    D = c.shape[-1]
    lead = tuple(c.shape[:-2])
    af = a.expand(*lead, D).reshape(-1, D).contiguous()
    cf = c.reshape(-1, D, D).contiguous()
    out = _RankOne.apply(af, cf)
    return _device.to_host(out.reshape(*lead, D, D), like_numpy)


class _RankOne(torch.autograd.Function):
    """vector (n, D), covariance (n, D, D) complex128 -> a a^H tr(C) / |a|^2 (n, D, D) by pbb_rank_one_estimate;
    backward pbb_rank_one_estimate_backward."""

    @staticmethod
    def forward(ctx, af, cf):
        n, D = af.shape
        out = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_rank_one_estimate', af, cf, n, D, out)
        ctx.save_for_backward(af, cf)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        af, cf = ctx.saved_tensors
        n, D = af.shape
        g = grad.to(torch.complex128).contiguous()
        ga = _device.empty((n, D), torch.complex128)
        gc = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_rank_one_estimate_backward', af, cf, g, n, D, ga, gc)
        return ga, gc


def _matvec(matrix, vector):
    like_numpy = not _device.is_tensor(matrix)
    m = _device.to_device(matrix, torch.complex128)
    v = _device.to_device(vector, torch.complex128)
    D = m.shape[-1]
    lead = torch.broadcast_shapes(m.shape[:-2], v.shape[:-1])
    mf = m.expand(*lead, D, D).reshape(-1, D, D).contiguous()
    vf = v.expand(*lead, D).reshape(-1, D).contiguous()
    out = _Matvec.apply(mf, vf)
    return _device.to_host(out.reshape(*lead, D), like_numpy)


class _Matvec(torch.autograd.Function):
    """matrix (n, D, D), vector (n, D) complex128 -> matrix @ vector (n, D) by pbb_matvec_batched; backward
    pbb_matvec_batched_backward."""

    @staticmethod
    def forward(ctx, mf, vf):
        n, D = vf.shape
        out = _device.empty((n, D), torch.complex128)
        _device.call('pbb_matvec_batched', mf, vf, n, D, out)
        ctx.save_for_backward(mf, vf)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        mf, vf = ctx.saved_tensors
        n, D = vf.shape
        g = grad.to(torch.complex128).contiguous()
        gm = _device.empty((n, D, D), torch.complex128)
        gv = _device.empty((n, D), torch.complex128)
        _device.call('pbb_matvec_batched_backward', mf, vf, g, n, D, gm, gv)
        return gm, gv


def get_pca_rank_one_estimate(covariance_matrix, **atf_kwargs):
    """Outer product of the principal eigenvector, trace-matched (beamformer_wrapper.py:11-24)."""
    return _rank_one(get_pca_vector(covariance_matrix, **atf_kwargs), covariance_matrix)


def _get_gev_atf_vector(covariance_matrix, noise_covariance_matrix, **gev_kwargs):
    """Phi_nn w_gev as an ATF estimate (beamformer_wrapper.py:27-46)."""
    assert noise_covariance_matrix is not None
    w = get_gev_vector(covariance_matrix, noise_covariance_matrix, **gev_kwargs)
    return _matvec(noise_covariance_matrix, w)


def get_gev_rank_one_estimate(covariance_matrix, noise_covariance_matrix, **gev_kwargs):
    """beamformer_wrapper.py:49-69."""
    a = _get_gev_atf_vector(covariance_matrix, noise_covariance_matrix, **gev_kwargs)
    return _rank_one(a, covariance_matrix)


def _atf_vector(atf_type, target, noise, **kw):
    if atf_type == 'pca':
        return get_pca_vector(target, **kw)
    if atf_type == 'scaled_gev_atf':
        return _get_gev_atf_vector(target, noise, **kw)
    raise ValueError(atf_type, 'use either pca or scaled_gev_atf')


def _rank_1_approximation(kind, target, noise, **kw):
    if kind == 'rank1_pca':
        return get_pca_rank_one_estimate(target, **kw)
    if kind == 'rank1_gev':
        return get_gev_rank_one_estimate(target, noise, **kw)
    raise ValueError(kind, 'use either rank1_pca or rank1_gev')


def get_bf_vector(beamformer, target_psd_matrix, noise_psd_matrix=None, **bf_kwargs):
    """Beamforming vector from a description such as 'mvdr_souden',
    'mvdr_souden+ban', 'rank1_gev+mvdr_souden+ban', 'gev+ban', 'pca+mvdr', 'ch0'
    (beamformer_wrapper.py:117-236).  WMWF / LCMV variants are outside the hot path."""
    assert isinstance(beamformer, str), beamformer
    assert 'lcmv' not in beamformer, 'LCMV beamformers have their own wrapper in the reference and are out of scope'
    ban = beamformer.endswith('+ban')
    core = beamformer[:-len('+ban')] if ban else beamformer
    target, noise = target_psd_matrix, noise_psd_matrix
    if core == 'pca':
        w = get_pca_vector(target, **bf_kwargs)
    elif core in ('pca+mvdr', 'scaled_gev_atf+mvdr'):
        atf = _atf_vector(core.split('+')[0], target, noise, **bf_kwargs.pop('atf_kwargs', {}))
        w = get_mvdr_vector(atf, noise)
    elif core in ('mvdr_souden', 'rank1_pca+mvdr_souden', 'rank1_gev+mvdr_souden'):
        if core != 'mvdr_souden':
            target = _rank_1_approximation(core.split('+')[0], target, noise, **bf_kwargs.pop('atf_kwargs', {}))
        w = get_mvdr_vector_souden(target, noise, **bf_kwargs)
    elif core in ('gev', 'rank1_pca+gev', 'rank1_gev+gev'):
        if core != 'gev':
            target = _rank_1_approximation(core.split('+')[0], target, noise, **bf_kwargs.pop('atf_kwargs', {}))
        w = get_gev_vector(target, noise, **bf_kwargs)
    elif core in ('wmwf', 'rank1_pca+wmwf', 'rank1_gev+wmwf'):
        raise NotImplementedError('WMWF is outside the hot path (SURVEY.md section 2)')
    elif core.startswith('ch') and core[2:].isdigit():
        D = target.shape[-1]
        w = np.zeros(D)
        w[int(core[2:])] = 1
        w = np.broadcast_to(w, tuple(target.shape[:-1]))
        if _device.is_tensor(target):
            w = _device.to_device(np.ascontiguousarray(w))
    else:
        raise ValueError(f'Could not find implementation for {core}.\nOriginal call contained {beamformer}.')
    if ban:
        w = blind_analytic_normalization(w, noise)
    return w
