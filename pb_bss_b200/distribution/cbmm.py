"""Complex Bingham mixture model: ``CBMMTrainer.fit / fit_predict`` and ``CBMM.predict`` with the signatures of
pb_bss/distribution/cbmm.py, executed by the kernels behind ``pbb_cbmm_fit`` / ``pbb_cbmm_predict``."""
from dataclasses import dataclass
from functools import cached_property
from operator import xor

import numpy as np
import torch

from .. import _device, _lib
from .cacgmm import _flatten_obs, _weight_mode
from .complex_bingham import (ComplexBingham, ComplexBinghamTrainer, _cbmm_fit_device, _check_dimension,
                              _status_error)
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
        independent, F, N, D = _flatten_obs(yd)
        _check_dimension(D)
        V = _device.to_device(self.complex_bingham.covariance_eigenvectors, torch.complex128)
        K = V.shape[-3]
        assert V.shape[-1] == D, (V.shape, D)
        V = V.expand(*independent, K, D, D).reshape(F, K, D, D).contiguous()
        lam = _device.to_device(self.complex_bingham.covariance_eigenvalues, torch.float64)
        lam = lam.expand(*independent, K, D).reshape(F, K, D).contiguous()
        w = _device.to_device(self.weight, torch.float64)
        wmode = _lib.WEIGHT_TIME
        if w.shape[-1] != 1:
            # frequency-tied weights (weight_constant_axis=(-3,), mixture_model_utils.py:187-190): (1, K, N)
            assert w.shape[-1] == N and all(int(n) == 1 for n in w.shape[:-2]), (w.shape, N)
            w = w.reshape(K, N).contiguous()
            wmode = _lib.WEIGHT_TIED_TIME
        else:
            w = w[..., 0].expand(*independent, K).reshape(F, K).contiguous()
        aff = _device.empty((F, K, N), torch.float64)
        status = _device.empty((1,), torch.int32)
        lib = _lib.load()
        nbytes = lib.pbb_cbmm_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _lib.check(lib.pbb_cbmm_predict(
            _device.ptr(yd), code, F, N, D, K, _device.ptr(V), _device.ptr(lam), _device.ptr(w), wmode,
            float(affiliation_eps), _device.ptr(aff), _device.ptr(ws), nbytes, _device.ptr(status),
            _device.stream_ptr()), 'pbb_cbmm_predict')
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
        assert xor(initialization is None, num_classes is None), (
            'Incompatible input combination. '
            'Exactly one of the two inputs has to be None: '
            f'{initialization is None} xor {num_classes is None}')
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1
        assert iterations > 0, iterations
        independent, F, N, D = _flatten_obs(yd)
        _check_dimension(D)
        if initialization is None:
            shape = (*independent, num_classes, N)
            initialization = np.random.uniform(size=shape)
            initialization /= np.einsum('...kn->...n', initialization)[..., None, :]
        K = initialization.shape[-2]
        init = _device.to_device(initialization, torch.float64)
        init = init.expand(*independent, K, N).reshape(F, K, N).contiguous()
        sal = None
        if saliency is not None:
            sal = _device.to_device(saliency, torch.float64)
            sal = sal.expand(*independent, N).reshape(F, N).contiguous()
        if self.dimension is None:
            self.dimension = D
        else:
            assert self.dimension == D, (
                'You initialized the trainer with a different dimension than '
                'you are using to fit a model. Use a new trainer, when you '
                'change the dimension.')
        weight_mode = _weight_mode(weight_constant_axis, len(independent) + 2)
        tied = weight_mode in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED)
        if inline_permutation_aligner is not None or tied:
            return self._fit_coupled(yd, like_numpy, init, sal, K, iterations, weight_mode, affiliation_eps,
                                     inline_permutation_aligner, weight_constant_axis)
        return self._fit_device(yd, like_numpy, init, sal, K, iterations, weight_mode, affiliation_eps)

    def _fit_device(self, yd, like_numpy, init, sal, K, iterations, weight_mode, affiliation_eps):
        """All iterations in one C-ABI call (bins independent).  With ``iterations=1`` this is exactly the
        reference's ``_m_step`` from the given affiliations (cbmm.py:215-237)."""
        independent, F, N, D = _flatten_obs(yd)
        V, lam, w = _cbmm_fit_device(yd, init, sal, K, iterations, weight_mode, affiliation_eps,
                                     self.eigenvalue_eps, self.max_concentration, 'CBMMTrainer.fit')
        if weight_mode == _lib.WEIGHT_CONST:
            weight = np.full([K, 1], 1 / K)
            if not like_numpy:
                weight = _device.to_device(weight)
        else:
            weight = _device.to_host(w.reshape(*independent, K, 1), like_numpy)
        return CBMM(
            weight=weight,
            complex_bingham=ComplexBingham(
                covariance_eigenvectors=_device.to_host(V.reshape(*independent, K, D, D), like_numpy),
                covariance_eigenvalues=_device.to_host(lam.reshape(*independent, K, D), like_numpy)))

    def _fit_coupled(self, yd, like_numpy, init, sal, K, iterations, weight_mode, affiliation_eps, aligner,
                     weight_constant_axis):
        """EM with per-iteration coupling across bins (cbmm.py:186-203): frequency-tied weights
        (``weight_constant_axis`` (-3,) / (-3, -1)) and / or the inline permutation alignment
        (mixture_model_utils.py:264-306).  Every step runs on the device."""
        from ..permutation_alignment import apply_mapping
        independent, F, N, D = _flatten_obs(yd)
        tied = weight_mode in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED)
        if aligner is not None:
            message = ('Inline permutation alignment reduces mismatch between frequency independent '
                       'mixtures weights and a frequency independent observation model. Therefore, we '
                       f'require `affiliation.ndim == 3` and a corresponding `weight_constant_axis` '
                       f'({weight_constant_axis}).')
            assert len(independent) == 1 and tied, message
        lib = _lib.load()
        affiliation = init
        model = None
        for _ in range(iterations):
            if model is not None:
                affiliation = model.predict(yd, affiliation_eps=affiliation_eps).reshape(F, K, N)
                if aligner is not None:
                    mask_kft = affiliation.permute(1, 0, 2).contiguous()
                    mapping = aligner.calculate_mapping(mask_kft)
                    affiliation = apply_mapping(mask_kft, mapping).permute(1, 0, 2).contiguous()
            # parameters of every (bin, class) from the affiliations; per-bin weights unless tied
            model = self._fit_device(yd, False, affiliation.contiguous(), sal, K, 1,
                                     _lib.WEIGHT_TIME if tied else weight_mode, affiliation_eps)
            if tied:
                w_kt = _device.empty((K, N), torch.float64)
                w_k = _device.empty((K,), torch.float64)
                flags = (1 if weight_mode == _lib.WEIGHT_TIED else 0) | 2
                # saliency form of estimate_mixture_weight (mixture_model_utils.py:192-203, cbmm.py:222-226)
                aff_w = (affiliation * sal[:, None, :] if sal is not None else affiliation).contiguous()
                _lib.check(lib.pbb_mixture_weight_over_bins(
                    _device.ptr(aff_w), F, K, N, flags, _device.ptr(w_kt), _device.ptr(w_k),
                    _device.stream_ptr()), 'pbb_mixture_weight_over_bins')
                model.weight = w_kt[None] if weight_mode == _lib.WEIGHT_TIED_TIME else w_k[None, :, None]
        if like_numpy:
            cb = model.complex_bingham
            model = CBMM(
                weight=_device.to_host(model.weight, True) if _device.is_tensor(model.weight) else model.weight,
                complex_bingham=ComplexBingham(_device.to_host(cb.covariance_eigenvectors, True),
                                               _device.to_host(cb.covariance_eigenvalues, True)))
        return model

    def fit_predict(self, y, initialization=None, num_classes=None, iterations=100, *,
                    saliency=None, weight_constant_axis=(-1,), affiliation_eps=0,
                    inline_permutation_aligner=None):
        model = self.fit(y=y, initialization=initialization, num_classes=num_classes, iterations=iterations,
                         saliency=saliency, weight_constant_axis=weight_constant_axis,
                         affiliation_eps=affiliation_eps, inline_permutation_aligner=inline_permutation_aligner)
        return model.predict(y)
