"""Complex Watson distribution -- ``ComplexWatson`` and ``ComplexWatsonTrainer`` with the names, arguments,
defaults and error types of pb_bss/distribution/complex_watson.py.

The trainer's state is the quadratic spline that inverts the hypergeometric ratio (:237-271).  The spline is built
once on the host with the reference's recipe (SciPy ``hyp1f1`` and ``interp1d(kind='quadratic')``) and evaluated on
the device by ``cw_update_kernel``; it is model state, not hot-path arithmetic.  ``log_pdf`` runs on
``pbb_cw_log_pdf``, the log normalisers on ``pbb_cw_log_norm`` and the trainer on ``pbb_cwmm_fit`` with one class
and one iteration (include/pbb.h).  NumPy in gives NumPy out; CUDA tensors in give CUDA tensors out.

Differences from the reference:
  - ``log_norm_1f1`` (and so ``log_pdf``) stays finite beyond kappa ~ 710, where scipy's ``hyp1f1`` overflows and
    the reference returns inf.  The trainer clamps kappa to ``max_concentration`` (500), so no fitted model gets
    there.
  - ``log_norm_low_concentration``, ``log_norm_medium_concentration`` and ``log_norm_high_concentration`` are
    computed; under NumPy 2 the reference's versions raise AttributeError (``np.asfarray`` was removed).
  - D is limited to 64.
"""
import math
from dataclasses import dataclass
from functools import cached_property

import numpy as np
import torch

from .. import _device, _lib
from .complex_circular_symmetric_gaussian import _as_device, _frames
from .mixture_model_utils import status_check
from .utils import _ProbabilisticModel

__all__ = ['ComplexWatson', 'ComplexWatsonTrainer']


def normalize_observation(observation):
    """(..., N, D) -> unit-norm (..., N, D) on the device: observation / max(norm over D, tiny)
    (complex_watson.py:16-29, complex_bingham.py:12-25; pbb_normalize_observation with swap = 0, the layout kept).
    Zero vectors stay zero.  Complex input; numpy in -> numpy out, CUDA tensor in -> CUDA tensor out."""
    like_numpy = not _device.is_tensor(observation)
    y = _device.to_device(observation)
    code = _device.complex_dtype_code(y)
    *independent, N, D = y.shape
    z = torch.empty(tuple(y.shape), dtype=y.dtype, device=y.device)
    if z.numel():
        _device.call('pbb_normalize_observation', y, z, math.prod(independent), N, D, code, 0)
    return _device.to_host(z, like_numpy)


@dataclass
class ComplexWatson(_ProbabilisticModel):
    mode: np.array = None  # (..., D)
    concentration: np.array = None  # (...)

    def pdf(self, y):
        """exp(log_pdf(y)) (complex_watson.py:61-71)."""
        p = self.log_pdf(y)
        return torch.exp(p) if _device.is_tensor(p) else np.exp(p)

    def log_pdf(self, y):
        """kappa |m^H y|^2 - log_norm_1f1(kappa, D) for y (..., N, D), used as given (not normalised); mode (..., D)
        and concentration (...) broadcast against y's leading dims (complex_watson.py:73-87)."""
        like_numpy = not _device.is_tensor(y)
        yd = _as_device(y)
        if not yd.is_complex():
            yd = yd.to(torch.complex128)
        mode = _as_device(self.mode, torch.complex128)
        kappa = _as_device(self.concentration, torch.float64)
        D = mode.shape[-1]
        assert yd.shape[-1] == D, (tuple(yd.shape), tuple(mode.shape))
        N = yd.shape[-2]
        lead = torch.broadcast_shapes(tuple(yd.shape[:-2]), tuple(mode.shape[:-1]), tuple(kappa.shape))
        M = int(np.prod(lead))
        out = _device.empty((M, N), torch.float64)
        if M and N:
            frames, stride = _frames(yd, lead)
            mode = mode.expand(*lead, D).reshape(M, D).contiguous()
            kappa = kappa.expand(lead).reshape(M).contiguous()
            _device.call('pbb_cw_log_pdf', frames, _device.complex_dtype_code(frames), stride, M, N, D, mode, kappa,
                         out)
        return _device.to_host(out.reshape(*lead, N), like_numpy)

    @staticmethod
    def log_norm_low_concentration(scale, dimension):
        """Mardia's Taylor series with 20 terms: good at low concentrations, drops off at 20 (:89-107)."""
        return _log_norm(scale, dimension, _lib.CW_NORM_LOW)

    @staticmethod
    def log_norm_medium_concentration(scale, dimension):
        """Mardia's closed form with kappa < 1e-2 clamped to 1e-2 (:109-138)."""
        return _log_norm(scale, dimension, _lib.CW_NORM_MEDIUM)

    @staticmethod
    def log_norm_high_concentration(scale, dimension):
        """The closed form without its correction term (:140-154)."""
        return _log_norm(scale, dimension, _lib.CW_NORM_HIGH)

    @staticmethod
    def log_norm_1f1(scale, dimension):
        """log(1F1(1; D; kappa) 2 pi^D / (D - 1)!) (:156-168), finite for every finite kappa >= 0."""
        return _log_norm(scale, dimension, _lib.CW_NORM_1F1)

    @staticmethod
    def log_norm_tran_vu(scale, dimension):
        """The low formula below kappa = 1 / D, the (unclamped) medium formula from there on (:170-214)."""
        return _log_norm(scale, dimension, _lib.CW_NORM_TRAN_VU)

    def log_norm(self):
        return self.log_norm_1f1(self.concentration, self.mode.shape[-1])


def _log_norm(scale, dimension, variant):
    """One ``pbb_cw_log_norm`` call over any array of kappa; NumPy in gives an array of the same shape (a NumPy
    scalar for log_norm_1f1 of a scalar, as scipy returns), a tensor in gives a tensor."""
    like_numpy = not _device.is_tensor(scale)
    k = _as_device(scale if not like_numpy else np.asarray(scale, dtype=float), torch.float64).contiguous()
    out = _device.empty(tuple(k.shape), torch.float64)
    if k.numel():
        _device.call('pbb_cw_log_norm', k, k.numel(), int(dimension), variant, out)
    out = _device.to_host(out, like_numpy)
    if like_numpy and variant == _lib.CW_NORM_1F1 and out.ndim == 0:
        return out[()]
    return out


class ComplexWatsonTrainer:
    def __init__(self, dimension=None, max_concentration=500,
                 spline_markers=1000):
        self.dimension = dimension
        self.max_concentration = max_concentration
        self.spline_markers = spline_markers

    def hypergeometric_ratio(self, concentration):
        """Largest eigenvalue of the Watson covariance as a function of the
        concentration (complex_watson.py:258-262)."""
        from scipy.special import hyp1f1
        D = self.dimension
        return hyp1f1(2, D + 1, concentration) / (D * hyp1f1(1, D, concentration))

    @cached_property
    def spline(self):
        """scipy interpolant eigenvalue -> concentration (complex_watson.py:237-256)."""
        from scipy.interpolate import interp1d
        assert self.dimension is not None, (
            'You need to specify dimension. This can be done at object '
            'instantiation or it can be inferred when using the fit function.')
        x = np.logspace(-3, np.log10(self.max_concentration), self.spline_markers)
        y = self.hypergeometric_ratio(x)
        return interp1d(y, x, kind='quadratic', assume_sorted=True,
                        bounds_error=False,
                        fill_value=(0, self.max_concentration))

    def hypergeometric_ratio_inverse(self, eigenvalues):
        return self.spline(eigenvalues)

    def fit(self, y, saliency=None) -> ComplexWatson:
        """Mode and concentration of y (..., N, D), normalised first (complex_watson.py:276-298).  Non-complex
        input or D = 1 raise AssertionError; the trainer takes its dimension from y, or asserts that it matches."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1
        if saliency is not None:
            saliency = _as_device(saliency, torch.float64)
            try:
                torch.broadcast_shapes(tuple(yd.shape[:-1]), tuple(saliency.shape))
            except RuntimeError:
                raise AssertionError((tuple(yd.shape), tuple(saliency.shape))) from None
        if self.dimension is None:
            self.dimension = yd.shape[-1]
        else:
            assert self.dimension == yd.shape[-1], (
                'You initialized the trainer with a different dimension than '
                'you are using to fit a model. Use a new trainer, when you '
                'change the dimension.')
        model = self._fit(yd, saliency=saliency)
        return ComplexWatson(mode=_device.to_host(model.mode, like_numpy),
                             concentration=_device.to_host(model.concentration, like_numpy))

    def _fit(self, y, saliency) -> ComplexWatson:
        """The top eigenpair of sum_n s y y^H / sum_n s (s = 1 without a saliency), kappa from the spline
        (complex_watson.py:300-315).  Runs as ``pbb_cwmm_fit`` with one class and one iteration, whose initial
        affiliations are the saliency.  The device normalises y, which leaves the unit-norm observations of
        ``fit`` unchanged; the reference uses other input as given.  Without frames the scatter sum is 0 / 0 and
        LinAlgError is raised, as in the reference."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        *_, N, D = yd.shape
        lead = tuple(yd.shape[:-2])
        if saliency is not None:
            saliency = _as_device(saliency, torch.float64)
            lead = torch.broadcast_shapes(lead, tuple(saliency.shape[:-1]))
        if N == 0:
            # the reference's scatter sum over no frames is 0 / 0, which its eigendecomposition rejects
            raise np.linalg.LinAlgError('Array must not contain infs or NaNs')
        F = int(np.prod(lead))
        mode = _device.empty((F, 1, D), torch.complex128)
        kappa = _device.empty((F, 1), torch.float64)
        if F:
            yf = yd.expand(*lead, N, D).reshape(F, N, D).contiguous()
            if saliency is None:
                init = torch.ones((F, 1, N), dtype=torch.float64, device=yd.device)
            else:
                init = saliency.expand(*lead, N).reshape(F, 1, N).contiguous()
            t_dev, c_dev = self.device_spline_table()
            w = _device.empty((F, 1), torch.float64)
            status = _device.empty((1,), torch.int32)
            lib = _lib.load()
            nbytes = lib.pbb_cwmm_workspace_bytes(F, N, D, 1)
            ws = _device.workspace(nbytes)
            _device.call('pbb_cwmm_fit', yf, _device.complex_dtype_code(yf), F, N, D, 1, init, None, 1,
                         _lib.WEIGHT_TIME, t_dev, c_dev, int(c_dev.numel()), float(self.max_concentration), mode, kappa,
                         w, ws, nbytes, status)
            status_check(status, 'ComplexWatsonTrainer.fit')
        return ComplexWatson(mode=_device.to_host(mode.reshape(*lead, D), like_numpy),
                             concentration=_device.to_host(kappa.reshape(lead), like_numpy))

    @cached_property
    def spline_table(self):
        """(knots t[n+3], coefficients c[n]) of the quadratic B-spline as numpy."""
        bs = self.spline._spline
        assert bs.k == 2, bs.k
        return np.ascontiguousarray(bs.t, dtype=np.float64), \
            np.ascontiguousarray(bs.c.ravel(), dtype=np.float64)

    def device_spline_table(self):
        """The table as CUDA tensors (cached per device)."""
        cache = self.__dict__.setdefault('_dev_tables', {})
        dev = _device.device()
        if dev.index not in cache:
            t, c = self.spline_table
            cache[dev.index] = (_device.to_device(t, torch.float64),
                                _device.to_device(c, torch.float64))
        return cache[dev.index]
