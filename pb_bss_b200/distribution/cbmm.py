"""Complex Bingham mixture model: ``CBMMTrainer.fit / fit_predict`` and ``CBMM.predict`` with the signatures of
pb_bss/distribution/cbmm.py, executed by the kernels behind ``pbb_cbmm_fit`` / ``pbb_cbmm_predict``."""
from dataclasses import dataclass
from functools import cached_property

import numpy as np
import torch

from .. import _device, _lib
from .complex_bingham import (ComplexBingham, ComplexBinghamTrainer, _cbmm_fit_device, _check_dimension,
                              _status_error)
from .mixture_model_utils import (check_initialization, coupled_fit, fit_tied_leading, flatten_obs, initial_affiliation,
                                  model_to_host, saliency_bn, weight_mode, weight_to_device, weight_to_host)
from .utils import _ProbabilisticModel

__all__ = ['CBMM', 'CBMMTrainer']


@dataclass
class CBMM(_ProbabilisticModel):
    weight: np.array = None  # (..., K, 1), (K, 1) for weight_constant_axis=-2, (1, K, T) / (1, K, 1) tied
    complex_bingham: ComplexBingham = None

    def predict(self, y, affiliation_eps=0):
        """Posterior affiliations (..., K, T) for y (..., T, D); y is normalised first (cbmm.py:26-55)."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        code = _device.complex_dtype_code(yd)
        independent, F, N, D = flatten_obs(yd)
        _check_dimension(D)
        V = _device.to_device(self.complex_bingham.covariance_eigenvectors, torch.complex128)
        K = V.shape[-3]
        assert V.shape[-1] == D, (V.shape, D)
        V = V.expand(*independent, K, D, D).reshape(F, K, D, D).contiguous()
        lam = _device.to_device(self.complex_bingham.covariance_eigenvalues, torch.float64)
        lam = lam.expand(*independent, K, D).reshape(F, K, D).contiguous()
        w, wmode = weight_to_device(self.weight, independent, F, K, N)
        aff = _device.empty((F, K, N), torch.float64)
        status = _device.empty((1,), torch.int32)
        lib = _lib.load()
        nbytes = lib.pbb_cbmm_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cbmm_predict', yd, code, F, N, D, K, V, lam, w, wmode, float(affiliation_eps), aff, ws,
                     nbytes, status)
        _device.check_status(status, _status_error('CBMM.predict', K))
        return _device.to_host(aff.reshape(*independent, K, N), like_numpy)


class CBMMTrainer:
    def __init__(self, dimension=None, max_concentration=np.inf, eigenvalue_eps=1e-8):
        self.dimension = dimension
        self.max_concentration = max_concentration
        self.eigenvalue_eps = eigenvalue_eps

    @cached_property
    def complex_bingham_trainer(self):
        return ComplexBinghamTrainer(self.dimension, max_concentration=self.max_concentration,
                                     eignevalue_eps=self.eigenvalue_eps)

    def fit(self, y, initialization=None, num_classes=None, iterations=100, *,
            saliency=None, weight_constant_axis=(-1,), affiliation_eps=0,
            inline_permutation_aligner=None):
        """EM for the complex Bingham mixture model (cbmm.py:79-205).

        y: (..., T, D); initialization: affiliations (..., K, T) or None with ``num_classes`` (then drawn from
        NumPy's global RNG, cbmm.py:120-126).  D must be 2..6 (KeyError otherwise, like the reference).
        """
        check_initialization(initialization, num_classes)
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1
        assert iterations > 0, iterations
        independent, F, N, D = flatten_obs(yd)
        _check_dimension(D)
        init = initial_affiliation(initialization, num_classes, independent, N)
        K = init.shape[-2]
        sal = saliency_bn(saliency, independent, N)
        if self.dimension is None:
            self.dimension = D
        else:
            assert self.dimension == D, (
                'You initialized the trainer with a different dimension than '
                'you are using to fit a model. Use a new trainer, when you '
                'change the dimension.')
        mode = weight_mode(weight_constant_axis, len(independent) + 2)
        tied = mode in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED)
        if tied and len(independent) > 1:
            model = fit_tied_leading(
                self.fit, independent[:-1], y=yd, initialization=init.reshape(*independent, K, N),
                iterations=iterations, saliency=saliency, weight_constant_axis=weight_constant_axis,
                affiliation_eps=affiliation_eps, inline_permutation_aligner=inline_permutation_aligner)
        elif inline_permutation_aligner is not None or tied:
            # parameters of every (bin, class) from the affiliations: pbb_cbmm_fit with one iteration
            model = coupled_fit(
                yd, init, None, iterations, weight_constant_axis, sal, inline_permutation_aligner,
                predict=lambda m: (m.predict(yd, affiliation_eps=affiliation_eps), None),
                m_step=lambda aff, q: self._fit_device(yd, False, aff, sal, K, 1, _lib.WEIGHT_TIME, affiliation_eps),
                saliency_form=True)
        else:
            return self._fit_device(yd, like_numpy, init, sal, K, iterations, mode, affiliation_eps)
        return model_to_host(model) if like_numpy else model

    def _fit_device(self, yd, like_numpy, init, sal, K, iterations, weight_mode, affiliation_eps):
        """All iterations in one C-ABI call (bins independent).  With ``iterations=1`` this is exactly the
        reference's ``_m_step`` from the given affiliations (cbmm.py:215-237)."""
        independent, F, N, D = flatten_obs(yd)
        V, lam, w = _cbmm_fit_device(yd, init, sal, K, iterations, weight_mode, affiliation_eps,
                                     self.eigenvalue_eps, self.max_concentration, 'CBMMTrainer.fit')
        return CBMM(
            weight=weight_to_host(weight_mode, w, independent, K, like_numpy),
            complex_bingham=ComplexBingham(
                covariance_eigenvectors=_device.to_host(V.reshape(*independent, K, D, D), like_numpy),
                covariance_eigenvalues=_device.to_host(lam.reshape(*independent, K, D), like_numpy)))

    def fit_predict(self, y, initialization=None, num_classes=None, iterations=100, *,
                    saliency=None, weight_constant_axis=(-1,), affiliation_eps=0,
                    inline_permutation_aligner=None):
        model = self.fit(y=y, initialization=initialization, num_classes=num_classes, iterations=iterations,
                         saliency=saliency, weight_constant_axis=weight_constant_axis,
                         affiliation_eps=affiliation_eps, inline_permutation_aligner=inline_permutation_aligner)
        return model.predict(y)
