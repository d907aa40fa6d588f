"""Complex Watson mixture model: ``CWMMTrainer.fit / fit_predict`` and
``CWMM.predict`` with the signatures of pb_bss/distribution/cwmm.py, executed by
the kernels behind ``pbb_cwmm_fit`` / ``pbb_cwmm_predict``."""
from dataclasses import dataclass
from functools import cached_property

import numpy as np
import torch

from .. import _device, _lib
from .complex_watson import ComplexWatson, ComplexWatsonTrainer
from .mixture_model_utils import (check_initialization, coupled_fit, fit_tied_leading, flatten_obs, initial_affiliation,
                                  model_to_host, saliency_bn, status_check, weight_mode, weight_to_device,
                                  weight_to_host)
from .utils import _ProbabilisticModel

__all__ = ['CWMM', 'CWMMTrainer']


@dataclass
class CWMM(_ProbabilisticModel):
    weight: np.array = None  # (..., K, 1)
    complex_watson: ComplexWatson = None

    def predict(self, y):
        """Posterior affiliations (..., K, T) for y (..., T, D) (cwmm.py:26-52)."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        code = _device.complex_dtype_code(yd)
        independent, F, N, D = flatten_obs(yd)
        mode = _device.to_device(self.complex_watson.mode, torch.complex128)
        K = mode.shape[-2]
        assert mode.shape[-1] == D, (mode.shape, D)
        mode = mode.expand(*independent, K, D).reshape(F, K, D).contiguous()
        kappa = _device.to_device(self.complex_watson.concentration, torch.float64)
        kappa = kappa.expand(*independent, K).reshape(F, K).contiguous()
        w, wmode = weight_to_device(self.weight, independent, F, K, N)
        aff = _device.empty((F, K, N), torch.float64)
        status = _device.empty((1,), torch.int32)
        lib = _lib.load()
        nbytes = lib.pbb_cwmm_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cwmm_predict', yd, code, F, N, D, K, mode, kappa, w, wmode, aff, ws, nbytes, status)
        status_check(status, 'CWMM.predict')
        return _device.to_host(aff.reshape(*independent, K, N), like_numpy)


class CWMMTrainer:
    def __init__(self, dimension=None, max_concentration=500,
                 spline_markers=1000):
        self.dimension = dimension
        self.max_concentration = max_concentration
        self.spline_markers = spline_markers

    @cached_property
    def complex_watson_trainer(self):
        return ComplexWatsonTrainer(
            self.dimension, max_concentration=self.max_concentration,
            spline_markers=self.spline_markers)

    def fit(self, y, initialization=None, num_classes=None, iterations=100, *,
            saliency=None, weight_constant_axis=(-1,), affiliation_eps=0,
            inline_permutation_aligner=None):
        """EM for the complex Watson mixture model (cwmm.py:76-149).

        y: (..., T, D); initialization: affiliations (..., K, T) or None with
        ``num_classes`` (then drawn from NumPy's global RNG, cwmm.py:121-127).
        """
        check_initialization(initialization, num_classes)
        assert affiliation_eps == 0, affiliation_eps  # cwmm.py:161
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1
        assert iterations > 0, iterations
        independent, F, N, D = flatten_obs(yd)
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
                inline_permutation_aligner=inline_permutation_aligner)
        elif inline_permutation_aligner is not None or tied:
            # mode / concentration of every (bin, class) from the affiliations: pbb_cwmm_fit with one iteration
            model = coupled_fit(
                yd, init, None, iterations, weight_constant_axis, sal, inline_permutation_aligner,
                predict=lambda m: (m.predict(yd), None),
                m_step=lambda aff, q: self._fit_device(yd, False, aff, sal, K, 1, _lib.WEIGHT_TIME),
                saliency_form=True)
        else:
            return self._fit_device(yd, like_numpy, init, sal, K, iterations, mode)
        return model_to_host(model) if like_numpy else model

    def _fit_device(self, yd, like_numpy, init, sal, K, iterations, weight_mode):
        """All iterations in one C-ABI call (bins independent).  With ``iterations=1`` this is exactly the
        reference's ``_m_step`` from the given affiliations (cwmm.py:220-240)."""
        code = _device.complex_dtype_code(yd)
        independent, F, N, D = flatten_obs(yd)
        t_dev, c_dev = self.complex_watson_trainer.device_spline_table()
        mode = _device.empty((F, K, D), torch.complex128)
        kappa = _device.empty((F, K), torch.float64)
        w = _device.empty((F, K), torch.float64)
        status = _device.empty((1,), torch.int32)
        lib = _lib.load()
        nbytes = lib.pbb_cwmm_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cwmm_fit', yd, code, F, N, D, K, init, sal, int(iterations), weight_mode, t_dev, c_dev,
                     int(c_dev.numel()), float(self.max_concentration), mode, kappa, w, ws, nbytes, status)
        status_check(status, 'CWMMTrainer.fit')
        return CWMM(
            weight=weight_to_host(weight_mode, w, independent, K, like_numpy),
            complex_watson=ComplexWatson(
                mode=_device.to_host(mode.reshape(*independent, K, D), like_numpy),
                concentration=_device.to_host(kappa.reshape(*independent, K), like_numpy)))

    def fit_predict(self, y, initialization=None, num_classes=None,
                    iterations=100, **kwargs):
        model = self.fit(y=y, initialization=initialization,
                         num_classes=num_classes, iterations=iterations,
                         **kwargs)
        return model.predict(y)
