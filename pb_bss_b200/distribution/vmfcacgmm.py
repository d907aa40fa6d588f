"""von-Mises-Fisher + complex-angular-central-Gaussian mixture model [Drude2019Integration]
(pb_bss/distribution/vmfcacgmm.py:34-301): like GCACGMM with a vMF over the (unit-norm) embeddings as the spectral
model.  Same names, arguments and defaults as the reference; the F*T-sized work runs in the device kernels shared
with gcacgmm.py."""
from dataclasses import dataclass

import numpy as np
import torch

from .. import _device
from .complex_angular_central_gaussian import ComplexAngularCentralGaussian
from .gcacgmm import _unit_norm_obs, cacg_m_step, class_weights, integrated_posterior
from .mixture_model_utils import (check_initialization, initial_affiliation, masked_affiliation, model_to_host,
                                  saliency_bn)
from .utils import _ProbabilisticModel
from .von_mises_fisher import VonMisesFisher, vmf_fit_fkt


def _real(embedding):
    assert not (embedding.is_complex() if _device.is_tensor(embedding) else np.iscomplexobj(embedding)), (
        'real embedding expected')
    return _device.to_device(embedding, torch.float64).contiguous()


@dataclass
class VMFCACGMM(_ProbabilisticModel):
    weight: np.array = None  # Shape (), (K,), (F, K), (K, T)
    weight_constant_axis: tuple = None
    vmf: VonMisesFisher = None
    cacg: ComplexAngularCentralGaussian = None
    spatial_weight: float = 1.
    spectral_weight: float = 1.

    def predict(self, observation, embedding):
        """observation (F, T, D), embedding (F, T, E) -> affiliation (F, K, T)  (vmfcacgmm.py:44-57)."""
        like_numpy = not _device.is_tensor(observation)
        affiliation, _ = self._predict(_unit_norm_obs(observation), _real(embedding))
        return _device.to_host(affiliation, like_numpy)

    def _predict(self, od, ed, affiliation_eps=0., inline_permutation_alignment=False):
        """vmfcacgmm.py:59-97 on device tensors (the vMF log pdf normalises the embedding itself)."""
        return integrated_posterior(self, self.vmf.log_pdf_fkt(ed), od, affiliation_eps,
                                    inline_permutation_alignment)


class VMFCACGMMTrainer:
    def fit(self, observation, embedding, initialization=None, num_classes=None, iterations=100, saliency=None,
            min_concentration=1e-10, max_concentration=500, hermitize=True, covariance_norm='eigenvalue',
            eigenvalue_floor=1e-10, affiliation_eps=1e-10, weight_constant_axis=(-1,), spatial_weight=1.,
            spectral_weight=1., inline_permutation_alignment=False) -> VMFCACGMM:
        """EM of the integrated model, signature and semantics of vmfcacgmm.py:101-199."""
        check_initialization(initialization, num_classes)
        like_numpy = not _device.is_tensor(observation)
        od = _unit_norm_obs(observation)
        ed = _real(embedding)
        assert od.shape[-1] > 1
        F, T, D = od.shape
        assert ed.shape[:2] == (F, T), (ed.shape, od.shape)
        affiliation = initial_affiliation(initialization, num_classes, (F,), T)   # vmfcacgmm.py:165-169, host stream
        sal = saliency_bn(saliency, (F,), T)
        quadratic_form = None
        model = None
        for _ in range(iterations):
            if model is not None:
                affiliation, quadratic_form = model._predict(
                    od, ed, inline_permutation_alignment=inline_permutation_alignment,
                    affiliation_eps=affiliation_eps)
            masked = masked_affiliation(affiliation, sal)
            model = VMFCACGMM(
                weight=class_weights(masked, weight_constant_axis), weight_constant_axis=weight_constant_axis,
                # the M-step fits the vMF on the embedding as given (vmfcacgmm.py:280-285 calls _fit, which does not
                # normalise; only the public fit() does, von_mises_fisher.py:108-111)
                vmf=vmf_fit_fkt(ed, masked, min_concentration, max_concentration),
                cacg=cacg_m_step(od, affiliation, quadratic_form, sal, hermitize, covariance_norm, eigenvalue_floor,
                                 'VMFCACGMMTrainer._m_step'),
                spatial_weight=spatial_weight, spectral_weight=spectral_weight)
        return model_to_host(model) if like_numpy else model

    def fit_predict(self, observation, embedding, **kwargs):
        """Fit a model, then return the posterior affiliations (vmfcacgmm.py:201-242)."""
        model = self.fit(observation=observation, embedding=embedding, **kwargs)
        return model.predict(observation=observation, embedding=embedding)
