"""Gaussians over real embedding vectors (pb_bss/distribution/gaussian.py:19-193).

Diagonal and spherical covariances serve the integrated model (tied over all (bin, frame) observations, kernels
``pbb_gaussian_log_pdf`` / ``pbb_gaussian_fit``) and the GMM without independent dims.  ``Gaussian`` (full covariance)
holds any number of leading independent dims; its precision Cholesky factor, log pdf and fit are the batched kernels
``pbb_precision_cholesky``, ``pbb_gaussian_full_log_pdf`` and ``pbb_gaussian_full_fit``.  The observations are only
ever touched by the device kernels."""
import math
from dataclasses import dataclass, field

import numpy as np
import torch

from .. import _device, _lib
from .utils import _ProbabilisticModel

MAX_E = 64   # kIntMaxE of csrc/api_integration.cu
MAX_K = 6    # the posterior kernel (pbb_log_pdf_to_affiliation)
_ILL_DEFINED = ('Fitting the mixture model failed because some components have ill-defined empirical '
                'covariance (for instance caused by singleton or collapsed samples).')


def _np(x):
    return x.detach().cpu().numpy() if _device.is_tensor(x) else np.asarray(x)


def _dev(x):
    return _device.to_device(x, torch.float64).contiguous()


def _is_real(x):
    return not x.is_complex() if _device.is_tensor(x) else np.isrealobj(x)


def check_embedding_dim(E):
    if E > MAX_E:
        raise ValueError(f'embedding dimension E={E} > {MAX_E} is not supported by the device kernels')


def batched_layout(y, model_lead):
    """Lays out ``y (..., N, E)`` against models with batch shape ``model_lead`` as the kernels' (B, K) grid: when the
    last broadcast dim is the models' own (y has no or a singleton dim there) it becomes the class axis K and y is
    shared by the K models, else K = 1.  Returns (x (B, N, E) device, B, K, full broadcast shape)."""
    Y = tuple(y.shape[:-2])
    N, E = y.shape[-2:]
    L = tuple(np.broadcast_shapes(tuple(model_lead), Y))
    if L and (len(Y) == 0 or Y[-1] == 1) and L[-1] <= MAX_K:
        blead, K = L[:-1], L[-1]
        yy = y.reshape(Y[:-1] + (N, E)) if Y else y
    else:
        blead, K = L, 1
        yy = y
    B = math.prod(blead)
    return yy.expand(blead + (N, E)).reshape(B, N, E).contiguous(), B, K, L


def precision_cholesky(cov):
    """sklearn's _compute_precision_cholesky(cov, 'full') + _compute_log_det_cholesky on the device: cov (..., E, E)
    -> (U (..., E, E), log_det (...)).  A matrix that is not positive definite raises ValueError (at the end of an
    enclosing ``_device.deferred_status`` block)."""
    E = cov.shape[-1]
    check_embedding_dim(E)
    M = cov.numel() // (E * E)
    pc = _device.empty(cov.shape, torch.float64)
    ld = _device.empty(cov.shape[:-2], torch.float64)
    status = _device.empty((1,), torch.int32)
    _device.call('pbb_precision_cholesky', cov, M, E, pc, ld, status)

    def on_error(s):
        raise ValueError(_ILL_DEFINED)
    _device.check_status(status, on_error)
    return pc, ld


def full_log_pdf_bkn(x, mean, pc, ld):
    """x (B, N, E), mean (B, K, E), U (B, K, E, E), log_det (B, K) device -> log pdf (B, K, N)."""
    B, N, E = x.shape
    K = mean.shape[1]
    out = _device.empty((B, K, N), torch.float64)
    _device.call('pbb_gaussian_full_log_pdf', x, mean, pc, ld, B, N, E, K, out)
    return out


def full_fit_bkn(x, weight):
    """GaussianTrainer._fit, 'full' (gaussian.py:152-193): x (B, N, E), weights (B, K, N) device -> mean (B, K, E),
    covariance (B, K, E, E)."""
    B, N, E = x.shape
    K = weight.shape[1]
    check_embedding_dim(E)
    lib = _lib.load()
    mean = _device.empty((B, K, E), torch.float64)
    cov = _device.empty((B, K, E, E), torch.float64)
    scratch = _device.empty((int(lib.pbb_gaussian_full_fit_scratch_doubles(B, N, E, K)),), torch.float64)
    _device.call('pbb_gaussian_full_fit', x, weight, B, N, E, K, mean, cov, scratch)
    return mean, cov


@dataclass
class Gaussian(_ProbabilisticModel):
    """Full covariance (gaussian.py:19-56).  NumPy parameters stay NumPy, CUDA tensors stay on the device."""
    mean: np.array = None        # (..., E)
    covariance: np.array = None  # (..., E, E)
    precision_cholesky: np.array = field(init=False, default=None)          # (..., E, E)
    log_det_precision_cholesky: np.array = field(init=False, default=None)  # (...,)

    def __post_init__(self):
        like_numpy = not _device.is_tensor(self.covariance)
        pc, ld = precision_cholesky(_dev(self.covariance))
        self.precision_cholesky = _device.to_host(pc, like_numpy)
        self.log_det_precision_cholesky = _device.to_host(ld, like_numpy)

    @classmethod
    def _from_device(cls, mean, covariance, pc, ld, like_numpy):
        g = cls.__new__(cls)
        g.mean, g.covariance = _device.to_host(mean, like_numpy), _device.to_host(covariance, like_numpy)
        g.precision_cholesky = _device.to_host(pc, like_numpy)
        g.log_det_precision_cholesky = _device.to_host(ld, like_numpy)
        return g

    def log_pdf(self, y):
        """y (..., N, E) -> (..., N), broadcast against the model dims as the reference's einsums do.  White = U d
        (the reference's contraction, not sklearn's U^T d; include/pbb.h, pbb_gaussian_full_log_pdf)."""
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        E = yd.shape[-1]
        check_embedding_dim(E)
        mean = _dev(self.mean)
        x, B, K, L = batched_layout(yd, mean.shape[:-1])
        m = mean.expand(L + (E,)).reshape(B, K, E).contiguous()
        pc = _dev(self.precision_cholesky).expand(L + (E, E)).reshape(B, K, E, E).contiguous()
        ld = _dev(self.log_det_precision_cholesky).expand(L).reshape(B, K).contiguous()
        out = full_log_pdf_bkn(x, m, pc, ld)
        return _device.to_host(out.reshape(L + (yd.shape[-2],)), like_numpy)


@dataclass
class DiagonalGaussian(_ProbabilisticModel):
    mean: np.array = None        # (K, E)
    covariance: np.array = None  # (K, E)
    precision_cholesky: np.array = field(init=False, default=None)          # (K, E)
    log_det_precision_cholesky: np.array = field(init=False, default=None)  # (K,)

    def __post_init__(self):
        cov = _np(self.covariance)
        if np.any(cov <= 0.0):   # sklearn's _compute_precision_cholesky (gaussian.py:67)
            raise ValueError(_ILL_DEFINED)
        self.precision_cholesky = 1.0 / np.sqrt(cov)
        self.log_det_precision_cholesky = np.sum(np.log(self.precision_cholesky), axis=-1)

    def _device_params(self, E):
        return (_device.to_device(_np(self.mean), torch.float64).contiguous(),
                _device.to_device(np.ascontiguousarray(self.precision_cholesky), torch.float64),
                _device.to_device(np.ascontiguousarray(self.log_det_precision_cholesky), torch.float64))

    def log_pdf_fkt(self, embedding):
        """embedding (F, T, E) CUDA tensor -> log pdf (F, K, T)."""
        return _gaussian_log_pdf(self, embedding)

    def log_pdf(self, y):
        """y (..., N, E) -> (..., K, N) (gaussian.py:73-93, with its class-axis contraction)."""
        return _small_log_pdf(self, y)


@dataclass
class SphericalGaussian(_ProbabilisticModel):
    mean: np.array = None        # (K, E)
    covariance: np.array = None  # (K,)
    precision_cholesky: np.array = field(init=False, default=None)          # (K,)
    log_det_precision_cholesky: np.array = field(init=False, default=None)  # (K,)

    def __post_init__(self):
        cov = _np(self.covariance)
        if np.any(cov <= 0.0):
            raise ValueError(_ILL_DEFINED)
        E = _np(self.mean).shape[-1]
        self.precision_cholesky = 1.0 / np.sqrt(cov)
        self.log_det_precision_cholesky = E * np.log(self.precision_cholesky)   # gaussian.py:106

    def _device_params(self, E):
        pc = np.repeat(np.asarray(self.precision_cholesky)[:, None], E, axis=1)
        return (_device.to_device(_np(self.mean), torch.float64).contiguous(),
                _device.to_device(np.ascontiguousarray(pc), torch.float64),
                _device.to_device(np.ascontiguousarray(self.log_det_precision_cholesky), torch.float64))

    def log_pdf_fkt(self, embedding):
        return _gaussian_log_pdf(self, embedding)

    def log_pdf(self, y):
        """y (..., N, E) -> (..., K, N) (gaussian.py:110-130)."""
        return _small_log_pdf(self, y)


def _gaussian_log_pdf(model, embedding):
    F, T, E = embedding.shape
    mean, pc, ld = model._device_params(E)
    K = mean.shape[0]
    out = _device.empty((F, K, T), torch.float64)
    # DiagonalGaussian: the reference's einsum quirk (gaussian.py:79-87) is reproduced by the kernel, see include/pbb.h
    _device.call('pbb_gaussian_log_pdf', embedding, mean, pc, ld, F, T, E, K, int(isinstance(model, DiagonalGaussian)),
                 out)
    return out


def small_log_pdf_kn(model, x):
    """Diagonal / spherical model with K classes (one model, any singleton leading dims), x (N, E) device -> (K, N)."""
    N, E = x.shape
    mean = _dev(model.mean).reshape(-1, E)
    K = mean.shape[0]
    diagonal = isinstance(model, DiagonalGaussian)
    pc = _dev(model.precision_cholesky)
    pc = pc.reshape(K, E) if diagonal else pc.reshape(K, 1).expand(K, E).contiguous()
    ld = _dev(model.log_det_precision_cholesky).reshape(K).contiguous()
    out = _device.empty((1, K, N), torch.float64)
    _device.call('pbb_gaussian_log_pdf', x, mean, pc, ld, 1, N, E, K, int(diagonal), out)
    return out[0]


def _small_log_pdf(model, y):
    like_numpy = not _device.is_tensor(y)
    yd = _dev(y)
    N, E = yd.shape[-2:]
    check_embedding_dim(E)
    lead_m = tuple(np.shape(model.mean)[:-1])
    if math.prod(lead_m[:-1]) != 1 or math.prod(yd.shape[:-2]) != 1:
        # the reference's einsums only broadcast one model of K classes against one set of observations
        raise ValueError(f'operands could not be broadcast together: model {lead_m}, observations {tuple(yd.shape)}')
    out_shape = tuple(np.broadcast_shapes(lead_m, tuple(yd.shape[:-2]))) + (N,)
    out = small_log_pdf_kn(model, yd.reshape(N, E).contiguous())
    return _device.to_host(out.reshape(out_shape), like_numpy)


class GaussianTrainer:
    def fit(self, y, saliency=None, covariance_type='full'):
        """gaussian.py:134-150: y (..., N, E), saliency (..., N) or None -> Gaussian / DiagonalGaussian /
        SphericalGaussian with the leading dims of y and saliency broadcast."""
        assert _is_real(y), y.dtype
        if saliency is not None:
            ys, ss = tuple(y.shape[:-1]), tuple(saliency.shape)
            assert all(len({a, b} | {1}) <= 2 for a, b in zip(ys[::-1], ss[::-1])), (y.shape, saliency.shape)
        return self._fit(y, saliency=saliency, covariance_type=covariance_type)

    def _fit(self, y, saliency, covariance_type):
        if covariance_type not in ('full', 'diagonal', 'spherical'):
            raise ValueError(f"Unknown covariance type '{covariance_type}'.")
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        N, E = yd.shape[-2:]
        check_embedding_dim(E)
        sal = None if saliency is None else _dev(saliency)
        lead = tuple(yd.shape[:-2]) if sal is None else tuple(np.broadcast_shapes(yd.shape[:-2], sal.shape[:-1]))
        B = math.prod(lead)
        x = yd.expand(lead + (N, E)).reshape(B, N, E).contiguous()
        w = (torch.ones((B, 1, N), dtype=torch.float64, device=x.device) if sal is None
             else sal.expand(lead + (N,)).reshape(B, 1, N).contiguous())
        if covariance_type == 'full':
            mean, cov = full_fit_bkn(x, w)
            return Gaussian(mean=_device.to_host(mean.reshape(lead + (E,)), like_numpy),
                            covariance=_device.to_host(cov.reshape(lead + (E, E)), like_numpy))
        spherical = covariance_type == 'spherical'
        lib = _lib.load()
        mean = _device.empty((B, E), torch.float64)
        cov = _device.empty((B,) if spherical else (B, E), torch.float64)
        scratch = _device.empty((int(lib.pbb_gaussian_fit_scratch_doubles(1, E, 1)),), torch.float64)
        for b in range(B):   # one tied model per leading index: the kernels of the integrated model with F = K = 1
            _device.call('pbb_gaussian_fit', x[b], w[b], 1, N, E, 1, int(spherical), mean[b], cov[b], scratch)
        cls = SphericalGaussian if spherical else DiagonalGaussian
        return cls(mean=mean.reshape(lead + (E,)).cpu().numpy(),
                   covariance=cov.reshape(lead + (() if spherical else (E,))).cpu().numpy())


def gaussian_fit_fkt(embedding, weight_fkt, covariance_type):
    """GaussianTrainer._fit (gaussian.py:155-193) over the F*T embeddings with the weights (F, K, T)."""
    if covariance_type not in ('diagonal', 'spherical'):
        if covariance_type == 'full':
            raise NotImplementedError("covariance_type='full' is not on the device path (diagonal / spherical are)")
        raise ValueError(f"Unknown covariance type '{covariance_type}'.")
    F, T, E = embedding.shape
    K = weight_fkt.shape[1]
    spherical = covariance_type == 'spherical'
    mean = _device.empty((K, E), torch.float64)
    cov = _device.empty((K,) if spherical else (K, E), torch.float64)
    lib = _lib.load()
    scratch = _device.empty((int(lib.pbb_gaussian_fit_scratch_doubles(F, E, K)),), torch.float64)
    _device.call('pbb_gaussian_fit', embedding, weight_fkt, F, T, E, K, int(spherical), mean, cov, scratch)
    cls = SphericalGaussian if spherical else DiagonalGaussian
    return cls(mean=mean.cpu().numpy(), covariance=cov.cpu().numpy())
