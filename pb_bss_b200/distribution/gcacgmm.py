"""Gaussian + complex-angular-central-Gaussian mixture model: the integration of per-(bin, frame) embeddings with the
spatial model [Drude2019Integration] (pb_bss/distribution/gcacgmm.py:38-333).

Same class / argument names and defaults as the reference.  Every array of size F*T lives on the device: the spatial
quadratic form and the cACG M-step are the cACGMM kernels (``pbb_cacgmm_predict`` / ``pbb_cacgmm_mstep``), the
spectral log pdf, the Gaussian fit and the posterior (with the optional per-bin pairing of spatial and spectral
classes) are the kernels of ``csrc/api_integration.cu``, the class weights the axis sums and unit norms of
``estimate_mixture_weight`` (``pbb_axis_sum`` / ``pbb_unit_norm``).  The Gaussians are tied over all bins, so the
EM loop is a per-iteration sequence of launches like the frequency-tied cACGMM (``mixture_model_utils.coupled_fit``)."""
import ctypes
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from .. import _device, _lib
from .cacgmm import CACGMM, _NORMS
from .complex_angular_central_gaussian import ComplexAngularCentralGaussian
from .gaussian import gaussian_fit_fkt
from .mixture_model_utils import (check_initialization, class_weight, initial_affiliation, masked_affiliation,
                                  model_to_host, saliency_bn, status_check, tied_weight)
from .utils import _ProbabilisticModel


def _axes(weight_constant_axis):
    if isinstance(weight_constant_axis, int):
        weight_constant_axis = (weight_constant_axis,)
    return tuple(sorted(a % 3 - 3 for a in weight_constant_axis))


def _weight_layout(weight_constant_axis):
    """(mode of the posterior kernel, shape of the squeezed weight) for the (F, K, T) affiliations."""
    ax = _axes(weight_constant_axis)
    if -2 in ax:
        return _lib.WEIGHT_CONST
    if ax == (-1,):
        return _lib.WEIGHT_TIME          # 'fk'
    if ax == (-3,):
        return _lib.WEIGHT_TIED_TIME     # 'kt'
    if ax == (-3, -1):
        return _lib.WEIGHT_TIED          # 'k'
    raise NotImplementedError(f'weight_constant_axis={weight_constant_axis!r}')


def _unit_norm_obs(observation):
    """observation / max(||observation||, tiny) over the channels (gcacgmm.py:62-65): the cACG kernels normalise the
    observation themselves, so this only validates and uploads."""
    od = _device.to_device(observation)
    assert od.is_complex(), od.dtype
    assert od.dim() == 3, ('(F, T, D) expected: the integrated models do not take independent dims', od.shape)
    return od.contiguous()


def spatial_log_pdf(cacg, od):
    """Quadratic form and cACG log pdf (F, K, T) of the device observation (cacg.py:167-203)."""
    F, T, D = od.shape
    probe = CACGMM(weight=np.full([cacg.covariance_eigenvalues.shape[-2], 1], 1.0), cacg=cacg)
    _, q, _, _ = probe._run_predict(od, None, 0., want_aff=False, want_q=True)
    lam = _device.to_device(cacg.covariance_eigenvalues, torch.float64).contiguous()
    K = lam.shape[-2]
    lp = _device.empty((F, K, T), torch.float64)
    _device.call('pbb_cacg_log_pdf', q.contiguous(), lam, F, K, T, D, lp)
    return q, lp


def integrated_posterior(model, spectral, od, affiliation_eps, inline_permutation_alignment):
    """Posterior of an integrated model (gcacgmm.py:86-128, vmfcacgmm.py:66-97): spatial_weight * cACG log pdf +
    spectral_weight * spectral log pdf, mixture weights, optional per-bin pairing of the two models' classes."""
    F, T, D = od.shape
    quadratic_form, spatial = spatial_log_pdf(model.cacg, od)
    K = spatial.shape[1]
    assert spectral.shape == spatial.shape, (spectral.shape, spatial.shape)
    mode = _weight_layout(model.weight_constant_axis)
    if mode == _lib.WEIGHT_CONST:
        # the reference unsqueezes its scalar weight 1 / K to len(axes) dims (gcacgmm.py:109, utils.py:324-329): an
        # axis below -len(axes), as in (-2,) or (-3, -2), raises IndexError there
        axes = _axes(model.weight_constant_axis)
        if axes[0] < -len(axes):
            raise IndexError((), [], model.weight_constant_axis)
    w = None if mode == _lib.WEIGHT_CONST else _device.to_device(model.weight, torch.float64).contiguous()
    aff = _device.empty((F, K, T), torch.float64)
    _device.call('pbb_log_pdf_to_affiliation', spatial, spectral, float(model.spatial_weight),
                 float(model.spectral_weight), w, mode, None, float(affiliation_eps),
                 int(bool(inline_permutation_alignment)), F, K, T, aff, None)
    return aff, quadratic_form


def class_weights(masked, weight_constant_axis):
    """Mixture weights of an integrated model from the masked affiliations (F, K, T) (gcacgmm.py:283-291), sums
    L1-normalised over the classes: per bin (F, K), NaN for a bin without weight as in the reference, or the
    frequency-tied (K, T) / (K,), 0 for a frame without weight."""
    mode = _weight_layout(weight_constant_axis)
    if mode == _lib.WEIGHT_CONST:
        return 1 / masked.shape[1]
    if mode == _lib.WEIGHT_TIME:
        return class_weight(masked)
    weight = tied_weight(masked, None, mode, saliency_form=True)
    return weight[0] if mode == _lib.WEIGHT_TIED_TIME else weight[0, :, 0]


def cacg_m_step(od, affiliation, quadratic_form, sal, hermitize, covariance_norm, eigenvalue_floor, what):
    """cACG of every (bin, class) from the affiliations: the cACGMM M-step kernel (cacg.py:253-342)."""
    F, T, D = od.shape
    K = affiliation.shape[1]
    lib = _lib.load()
    V = _device.empty((F, K, D, D), torch.complex128)
    lam = _device.empty((F, K, D), torch.float64)
    w_unused = _device.empty((F, K), torch.float64)
    status = _device.empty((1,), torch.int32)
    opts = _lib.CacgmmOptions(
        iterations=1, covariance_norm=_NORMS[covariance_norm], weight_mode=_lib.WEIGHT_TIME,
        hermitize=int(bool(hermitize)), affiliation_eps=0., eigenvalue_floor=float(eigenvalue_floor),
        frames_per_block=0, reserved=0)
    nbytes = lib.pbb_cacgmm_workspace_bytes(F, T, D, K)
    ws = _device.workspace(nbytes)
    _device.call('pbb_cacgmm_mstep', od, _device.complex_dtype_code(od), F, T, D, K, affiliation.contiguous(),
                 quadratic_form, sal, ctypes.byref(opts), V, lam, w_unused, ws, nbytes, status)
    status_check(status, what)
    return ComplexAngularCentralGaussian(covariance_eigenvectors=V, covariance_eigenvalues=lam)


@dataclass
class GCACGMM(_ProbabilisticModel):
    weight: np.array = None  # Shape (), (K,), (F, K), (K, T)
    weight_constant_axis: tuple = None
    gaussian: Any = None     # DiagonalGaussian or SphericalGaussian
    cacg: ComplexAngularCentralGaussian = None
    spatial_weight: float = 1.
    spectral_weight: float = 1.

    def predict(self, observation, embedding):
        """observation (F, T, D) complex, embedding (F, T, E) real -> affiliation (F, K, T)  (gcacgmm.py:48-68)."""
        like_numpy = not _device.is_tensor(observation)
        od = _unit_norm_obs(observation)
        ed = _device.to_device(embedding, torch.float64).contiguous()
        assert not (embedding.is_complex() if _device.is_tensor(embedding) else np.iscomplexobj(embedding))
        affiliation, _ = self._predict(od, ed)
        return _device.to_host(affiliation, like_numpy)

    def _predict(self, od, ed, affiliation_eps=0., inline_permutation_alignment=False):
        """gcacgmm.py:70-128 on device tensors -> (affiliation, quadratic_form), both (F, K, T)."""
        return integrated_posterior(self, self.gaussian.log_pdf_fkt(ed), od, affiliation_eps,
                                    inline_permutation_alignment)


class GCACGMMTrainer:
    def fit(self, observation, embedding, initialization=None, num_classes=None, iterations=100, saliency=None,
            hermitize=True, covariance_norm='eigenvalue', eigenvalue_floor=1e-10, covariance_type='spherical',
            fixed_covariance=None, affiliation_eps=1e-10, weight_constant_axis=(-1,), spatial_weight=1.,
            spectral_weight=1., inline_permutation_alignment=False) -> GCACGMM:
        """EM of the integrated model, signature and semantics of gcacgmm.py:131-227."""
        check_initialization(initialization, num_classes)
        like_numpy = not _device.is_tensor(observation)
        od = _unit_norm_obs(observation)
        assert not (embedding.is_complex() if _device.is_tensor(embedding) else np.iscomplexobj(embedding)), (
            'real embedding expected')
        ed = _device.to_device(embedding, torch.float64).contiguous()
        assert od.shape[-1] > 1
        F, T, D = od.shape
        assert ed.shape[:2] == (F, T), (ed.shape, od.shape)
        affiliation = initial_affiliation(initialization, num_classes, (F,), T)   # gcacgmm.py:187-192, host stream
        sal = saliency_bn(saliency, (F,), T)
        quadratic_form = None
        model = None
        for _ in range(iterations):
            if model is not None:
                affiliation, quadratic_form = model._predict(
                    od, ed, inline_permutation_alignment=inline_permutation_alignment,
                    affiliation_eps=affiliation_eps)
            model = self._m_step(od, ed, quadratic_form, affiliation, sal, hermitize, covariance_norm,
                                 eigenvalue_floor, covariance_type, fixed_covariance, weight_constant_axis,
                                 spatial_weight, spectral_weight)
        return model_to_host(model) if like_numpy else model

    def fit_predict(self, observation, embedding, **kwargs):
        """Fit a model, then return the posterior affiliations (gcacgmm.py:229-267)."""
        model = self.fit(observation=observation, embedding=embedding, **kwargs)
        return model.predict(observation=observation, embedding=embedding)

    def _m_step(self, od, ed, quadratic_form, affiliation, sal, hermitize, covariance_norm, eigenvalue_floor,
                covariance_type, fixed_covariance, weight_constant_axis, spatial_weight, spectral_weight):
        """gcacgmm.py:269-333 on device tensors."""
        masked = masked_affiliation(affiliation, sal)
        weight = class_weights(masked, weight_constant_axis)
        gaussian = gaussian_fit_fkt(ed, masked, covariance_type)
        if fixed_covariance is not None:
            assert np.shape(fixed_covariance) == np.shape(gaussian.covariance), (
                f'{np.shape(fixed_covariance)} != {np.shape(gaussian.covariance)}')
            gaussian = gaussian.__class__(mean=gaussian.mean, covariance=np.asarray(fixed_covariance))
        cacg = cacg_m_step(od, affiliation, quadratic_form, sal, hermitize, covariance_norm, eigenvalue_floor,
                           'GCACGMMTrainer._m_step')
        return GCACGMM(weight=weight, weight_constant_axis=weight_constant_axis, gaussian=gaussian, cacg=cacg,
                       spatial_weight=spatial_weight, spectral_weight=spectral_weight)
