"""von Mises-Fisher mixture model over embedding vectors (pb_bss/distribution/vmfmm.py:14-172), with any number of
independent leading dims: y (..., N, E), affiliations (..., K, N), one model (K, E) per leading index.

Same class / argument names, defaults and error types as the reference (``saliency`` is positional here, unlike in
``GMMTrainer``).  Per EM iteration the weighted resultants (``pbb_vmf_resultant``), class weights, log pdf
(``pbb_vmf_log_pdf``) and posterior run on the device; the B*K*E parameter math and the log normaliser (scipy's
``ive``) run on the host, as in ``VonMisesFisher``, which costs one small copy per iteration."""
import math
from dataclasses import dataclass
from typing import Any

import numpy as np

from .. import _device
from .gaussian import _dev, _is_real, check_embedding_dim
from .gmm import check_classes, mixture_weight, posterior, weight_from_public, weight_kind, weight_to_public
from .mixture_model_utils import check_initialization, initial_affiliation, masked_affiliation, saliency_bn
from .utils import _ProbabilisticModel
from .von_mises_fisher import VonMisesFisher, _np, vmf_fit_bkn, vmf_log_pdf_bkn


def _params_bk(vmf, lead, K, E):
    mean, kappa = _np(vmf.mean), _np(vmf.concentration)
    np.broadcast_shapes(mean.shape[:-2], lead)   # the reference's broadcast check (ValueError)
    log_norm = VonMisesFisher(mean=mean, concentration=kappa).log_norm()
    B = math.prod(lead)
    return (_dev(np.broadcast_to(mean, lead + (K, E)).reshape(B, K, E)),
            _dev(np.broadcast_to(kappa, lead + (K,)).reshape(B, K)),
            _dev(np.broadcast_to(log_norm, lead + (K,)).reshape(B, K)))


@dataclass
class VMFMM(_ProbabilisticModel):
    vmf: VonMisesFisher = None
    weight: Any = None  # (..., K, 1), (K, 1) or (..., 1, N)

    def predict(self, y):
        """y (..., N, E) (any norm) -> affiliation (..., K, N) (vmfmm.py:19-37)."""
        assert _is_real(y), y.dtype
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        N, E = yd.shape[-2:]
        check_embedding_dim(E)
        lead = tuple(yd.shape[:-2])
        K = np.shape(self.vmf.mean)[-2]
        check_classes(K)
        lp = vmf_log_pdf_bkn(yd.reshape(-1, N, E), *_params_bk(self.vmf, lead, K, E))
        mode, w = weight_from_public(self.weight, lead, K, N)
        return _device.to_host(posterior(lp, mode, w).reshape(lead + (K, N)), like_numpy)


class VMFMMTrainer:
    """The vMFMM can be used to cluster the embeddings."""

    def fit(self, y, initialization=None, num_classes=None, iterations=100, saliency=None,
            weight_constant_axis=(-1,), min_concentration=1e-10, max_concentration=500) -> VMFMM:
        """EM of vmfmm.py:43-98: y (..., N, E), initialization (..., K, N), saliency (..., N)."""
        check_initialization(initialization, num_classes)
        assert _is_real(y), y.dtype
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        N, E = yd.shape[-2:]
        lead = tuple(yd.shape[:-2])
        B = math.prod(lead)
        check_embedding_dim(E)
        kind = weight_kind(weight_constant_axis)
        K = num_classes if initialization is None else np.shape(initialization)[-2]
        check_classes(K)
        x = yd.reshape(B, N, E)
        aff = initial_affiliation(initialization, num_classes, lead, N)
        sal = saliency_bn(saliency, lead, N)
        mean = concentration = mode = w = None
        for it in range(iterations):
            if it > 0:
                log_norm = VonMisesFisher(mean=mean, concentration=concentration).log_norm()
                lp = vmf_log_pdf_bkn(x, _dev(mean), _dev(concentration), _dev(log_norm))
                aff = posterior(lp, mode, w)
            masked = masked_affiliation(aff, sal)                      # vmfmm.py:151-172
            mode, w = mixture_weight(masked, kind)
            mean, concentration = vmf_fit_bkn(x, masked, min_concentration, max_concentration)
        mean, concentration = mean.reshape(lead + (K, E)), concentration.reshape(lead + (K,))
        if not like_numpy:
            mean, concentration = _dev(mean), _dev(concentration)
        return VMFMM(vmf=VonMisesFisher(mean=mean, concentration=concentration),
                     weight=weight_to_public(mode, w, lead, K, N, like_numpy))

    def fit_predict(self, y, initialization=None, num_classes=None, iterations=100, saliency=None,
                    weight_constant_axis=(-1,), min_concentration=1e-10, max_concentration=500):
        """Fit a model. Then just return the posterior affiliations (vmfmm.py:100-122)."""
        model = self.fit(y=y, initialization=initialization, num_classes=num_classes, iterations=iterations,
                         saliency=saliency, min_concentration=min_concentration,
                         max_concentration=max_concentration, weight_constant_axis=weight_constant_axis)
        return model.predict(y)
