"""Gaussian mixture model over embedding vectors (pb_bss/distribution/gmm.py:16-173), with any number of independent
leading dims: y (..., N, E), affiliations (..., K, N), one model (K, E[, E]) per leading index.

Same class / argument names, defaults and error types as the reference.  The EM loop is a per-iteration sequence of
launches on the caller's stream without a host synchronisation: class weights (``pbb_axis_sum`` /
``pbb_unit_norm``), the Gaussian fit (``pbb_gaussian_full_fit``, or ``pbb_gaussian_fit`` for the diagonal /
spherical model, which the reference only accepts without a leading dim > 1), the precision Cholesky factors
(``pbb_precision_cholesky``, status words read when the loop ends) and the posterior (``pbb_log_pdf_to_affiliation``
with the leading dims as its bin axis).  All arithmetic is float64.  NumPy in gives NumPy out, a CUDA tensor in gives
CUDA tensors out (the diagonal / spherical parameters are host arrays, as in the integrated model).

BinaryGMM / BinaryGMMTrainer (gmm.py:176-230) are the k-means baseline of deep clustering, sklearn's
``KMeans(n_clusters=K)`` on the device (``pbb_kmeans_fit`` / ``pbb_kmeans_predict``)."""
import math
import warnings
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from .. import _device, _lib, _nd
from .gaussian import (_ILL_DEFINED, MAX_K, DiagonalGaussian, Gaussian, SphericalGaussian, _dev, _is_real,
                       check_embedding_dim, full_fit_bkn, full_log_pdf_bkn, precision_cholesky, small_log_pdf_kn)
from .mixture_model_utils import (check_initialization, class_weight, initial_affiliation, masked_affiliation,
                                  saliency_bn)
from .utils import _ProbabilisticModel, _unit_norm


def weight_kind(weight_constant_axis):
    """estimate_mixture_weight (mixture_model_utils.py:178-201) as the trainers call it, always with a saliency:
    (-1,) -> one weight per (model, class); the int -2 -> the constant 1/K; the tuple (-2,) (not caught by the
    reference's int test) -> one weight per (model, observation)."""
    if isinstance(weight_constant_axis, list):
        weight_constant_axis = tuple(weight_constant_axis)
    if weight_constant_axis == (-1,):
        return 'class'
    if isinstance(weight_constant_axis, int) and not isinstance(weight_constant_axis, bool) \
            and weight_constant_axis == -2:
        return 'const'
    if weight_constant_axis == (-2,):
        return 'frame'
    raise NotImplementedError(f'weight_constant_axis={weight_constant_axis!r}: (-1,), -2 and (-2,) are supported')


def check_classes(K):
    if K > MAX_K:
        raise NotImplementedError(f'K={K} > {MAX_K} classes is not supported by the posterior kernel')


def mixture_weight(masked, kind):
    """masked affiliations (B, K, N) device -> (posterior weight mode, device weight or None)."""
    if kind == 'const':
        return _lib.WEIGHT_CONST, None
    if kind == 'class':
        return _lib.WEIGHT_TIME, class_weight(masked)
    # weight_constant_axis (-2,) with a saliency (mixture_model_utils.py:191-201): the sum over the classes,
    # L1-normalised over its singleton class axis -> s / |s|, and 0 where s == 0
    total = _nd.axis_sum(masked, (1,), True)
    return _lib.WEIGHT_FRAME, _unit_norm(total, ord=1, axis=-2, eps=1e-10, eps_style='where')[:, 0]


def weight_to_public(mode, w, lead, K, N, like_numpy):
    """The reference's weight shapes: (..., K, 1), (K, 1) of 1/K, (..., 1, N)."""
    if mode == _lib.WEIGHT_CONST:
        return np.full([K, 1], 1 / K)
    shape = lead + ((K, 1) if mode == _lib.WEIGHT_TIME else (1, N))
    return _device.to_host(w.reshape(shape), like_numpy)


def weight_from_public(weight, lead, K, N):
    """A model's weight -> (mode, device weight) for the posterior of (B, K, N) log pdfs."""
    shape = tuple(np.shape(weight))
    np.broadcast_shapes(shape, lead + (K, N))   # the reference's broadcast check (ValueError)
    B = math.prod(lead)
    if len(shape) >= 2 and shape[-1] == 1:
        return _lib.WEIGHT_TIME, _dev(weight).expand(lead + (K, 1)).reshape(B, K).contiguous()
    if len(shape) >= 2 and shape[-2] == 1:
        return _lib.WEIGHT_FRAME, _dev(weight).expand(lead + (1, N)).reshape(B, N).contiguous()
    raise NotImplementedError(f'mixture weight of shape {shape}: (..., K, 1) or (..., 1, N) expected')


def posterior(log_pdf, mode, w):
    """log_pdf_to_affiliation (mixture_model_utils.py:7-55), affiliation_eps = 0: (B, K, N) -> (B, K, N)."""
    B, K, N = log_pdf.shape
    aff = _device.empty((B, K, N), torch.float64)
    _device.call('pbb_log_pdf_to_affiliation', log_pdf, None, 1.0, 0.0, w, mode, None, 0.0, 0, B, K, N, aff, None)
    return aff


def _gaussian_log_pdf_bkn(gaussian, x, lead):
    """x (B, N, E) device with leading dims lead -> (B, K, N) for the GMM's Gaussian (model dims (..., K))."""
    B, N, E = x.shape
    if isinstance(gaussian, Gaussian):
        mean = _dev(gaussian.mean)
        K = mean.shape[-2]
        np.broadcast_shapes(tuple(mean.shape[:-2]), lead)   # the reference's broadcast check (ValueError)
        mean = mean.expand(lead + (K, E)).reshape(B, K, E).contiguous()
        pc = _dev(gaussian.precision_cholesky).expand(lead + (K, E, E)).reshape(B, K, E, E).contiguous()
        ld = _dev(gaussian.log_det_precision_cholesky).expand(lead + (K,)).reshape(B, K).contiguous()
        return full_log_pdf_bkn(x, mean, pc, ld)
    if B != 1 or math.prod(np.shape(gaussian.mean)[:-2]) != 1:
        raise ValueError(f'operands could not be broadcast together: {type(gaussian).__name__} with model shape '
                         f'{np.shape(gaussian.mean)} and {B} independent observation sets')
    return small_log_pdf_kn(gaussian, x[0])[None]


@dataclass
class GMM(_ProbabilisticModel):
    weight: Any = None    # (..., K, 1), (K, 1) or (..., 1, N)
    gaussian: Any = None  # Gaussian, DiagonalGaussian or SphericalGaussian

    def predict(self, x):
        """x (..., N, E) -> affiliation (..., K, N) (gmm.py:21-25)."""
        like_numpy = not _device.is_tensor(x)
        assert _is_real(x), x.dtype
        xd = _dev(x)
        N, E = xd.shape[-2:]
        check_embedding_dim(E)
        lead = tuple(xd.shape[:-2])
        K = np.shape(self.gaussian.mean)[-2]
        check_classes(K)
        lp = _gaussian_log_pdf_bkn(self.gaussian, xd.reshape(-1, N, E), lead)
        mode, w = weight_from_public(self.weight, lead, K, N)
        return _device.to_host(posterior(lp, mode, w).reshape(lead + (K, N)), like_numpy)


class GMMTrainer:
    def __init__(self, eps=1e-10):
        self.eps = eps
        self.log_likelihood_history = []

    def fit(self, y, initialization=None, num_classes=None, iterations=100, *, saliency=None,
            weight_constant_axis=(-1,), covariance_type='full', fixed_covariance=None):
        """EM of gmm.py:33-89: y (..., N, E), initialization (..., K, N), saliency (..., N)."""
        check_initialization(initialization, num_classes)
        assert _is_real(y), y.dtype
        return self._fit(y, initialization=initialization, num_classes=num_classes, iterations=iterations,
                         saliency=saliency, weight_constant_axis=weight_constant_axis,
                         covariance_type=covariance_type, fixed_covariance=fixed_covariance)

    def fit_predict(self, y, initialization=None, num_classes=None, iterations=100, *, saliency=None,
                    weight_constant_axis=(-2,), covariance_type='full', fixed_covariance=None):
        """Fit a model. Then just return the posterior affiliations (gmm.py:91-114)."""
        model = self.fit(y=y, initialization=initialization, num_classes=num_classes, iterations=iterations,
                         saliency=saliency, weight_constant_axis=weight_constant_axis,
                         covariance_type=covariance_type, fixed_covariance=fixed_covariance)
        return model.predict(y)

    def _fit(self, y, initialization, num_classes, iterations, saliency, weight_constant_axis, covariance_type,
             fixed_covariance):
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        N, E = yd.shape[-2:]
        lead = tuple(yd.shape[:-2])
        B = math.prod(lead)
        check_embedding_dim(E)
        kind = weight_kind(weight_constant_axis)
        K = num_classes if initialization is None else np.shape(initialization)[-2]
        check_classes(K)
        if covariance_type not in ('full', 'diagonal', 'spherical'):
            raise ValueError(f"Unknown covariance type '{covariance_type}'.")
        if covariance_type != 'full' and B != 1:
            # the reference's DiagonalGaussian / SphericalGaussian flatten their leading dims (gaussian.py:66-71,
            # 103-108), so the posterior's broadcast fails (gmm.py:22-25)
            raise ValueError(f'operands could not be broadcast together: covariance_type={covariance_type!r} with '
                             f'independent dims {lead}')
        x = yd.reshape(B, N, E)
        aff = initial_affiliation(initialization, num_classes, lead, N)
        sal = saliency_bn(saliency, lead, N)
        cov_shape = lead + {'full': (K, E, E), 'diagonal': (K, E), 'spherical': (K,)}[covariance_type]
        fixed = None
        if fixed_covariance is not None:
            assert tuple(fixed_covariance.shape) == cov_shape, f'{tuple(fixed_covariance.shape)} != {cov_shape}'
            fixed = _dev(fixed_covariance)
        state = None
        with _device.deferred_status():
            for _ in range(iterations):
                if state is not None:
                    aff = posterior(self._log_pdf(x, state), state['mode'], state['w'])
                state = self._m_step(x, aff, sal, kind, covariance_type, fixed)
        return self._to_model(state, lead, K, N, E, like_numpy)

    @staticmethod
    def _m_step(x, affiliation, sal, kind, covariance_type, fixed):
        """gmm.py:143-173 on device tensors."""
        B, N, E = x.shape
        K = affiliation.shape[1]
        masked = masked_affiliation(affiliation, sal)
        mode, w = mixture_weight(masked, kind)
        if covariance_type == 'full':
            mean, cov = full_fit_bkn(x, masked)
            if fixed is not None:
                cov = fixed.reshape(B, K, E, E)
            pc, ld = precision_cholesky(cov)
            return dict(type='full', mode=mode, w=w, mean=mean, cov=cov, pc=pc, ld=ld)
        spherical = covariance_type == 'spherical'
        lib = _lib.load()
        mean = _device.empty((K, E), torch.float64)
        cov = _device.empty((K,) if spherical else (K, E), torch.float64)
        scratch = _device.empty((int(lib.pbb_gaussian_fit_scratch_doubles(1, E, K)),), torch.float64)
        _device.call('pbb_gaussian_fit', x, masked, 1, N, E, K, int(spherical), mean, cov, scratch)
        if fixed is not None:
            cov = fixed.reshape(cov.shape)
        # sklearn's _compute_precision_cholesky(cov, 'diag') on the K x E parameters (gaussian.py:66-71, 103-108)
        status = (cov <= 0.0).any().to(torch.int32).reshape(1)

        def on_error(s):
            raise ValueError(_ILL_DEFINED)
        _device.check_status(status, on_error)
        pc = 1.0 / torch.sqrt(cov)
        ld = E * torch.log(pc) if spherical else torch.log(pc).sum(-1)
        return dict(type=covariance_type, mode=mode, w=w, mean=mean, cov=cov, pc=pc, ld=ld)

    @staticmethod
    def _log_pdf(x, state):
        if state['type'] == 'full':
            return full_log_pdf_bkn(x, state['mean'], state['pc'], state['ld'])
        K, E = state['mean'].shape
        pc = state['pc'] if state['type'] == 'diagonal' else state['pc'][:, None].expand(K, E).contiguous()
        out = _device.empty((1, K, x.shape[1]), torch.float64)
        _device.call('pbb_gaussian_log_pdf', x, state['mean'], pc, state['ld'], 1, x.shape[1], E, K,
                     int(state['type'] == 'diagonal'), out)
        return out

    @staticmethod
    def _to_model(state, lead, K, N, E, like_numpy):
        weight = weight_to_public(state['mode'], state['w'], lead, K, N, like_numpy)
        if state['type'] == 'full':
            gaussian = Gaussian._from_device(state['mean'].reshape(lead + (K, E)),
                                             state['cov'].reshape(lead + (K, E, E)),
                                             state['pc'].reshape(lead + (K, E, E)),
                                             state['ld'].reshape(lead + (K,)), like_numpy)
        else:
            cls = DiagonalGaussian if state['type'] == 'diagonal' else SphericalGaussian
            gaussian = cls(mean=state['mean'].reshape(lead + (K, E)).cpu().numpy(),
                           covariance=state['cov'].reshape(lead + state['cov'].shape).cpu().numpy())
        return GMM(weight=weight, gaussian=gaussian)


KMEANS_MAX_K = 16    # PBB_KMEANS_MAX_K
_KMEANS_MAX_ITER = 300


class ConvergenceWarning(UserWarning):
    """sklearn.exceptions.ConvergenceWarning, which the k-means fit issues for fewer distinct clusters than K."""


def _kmeans_draws(N, K, sklearn_dtype):
    """The draws of sklearn's _kmeans_plusplus from NumPy's global RandomState (random_state=None), in its order:
    the first centre's index, then (K - 1, n_local_trials) unscaled uniforms.  They do not depend on the data."""
    w = np.ones(N, dtype=sklearn_dtype)
    first = int(np.random.choice(N, p=w / w.sum()))
    L = 2 + int(np.log(K))
    u = np.array([np.random.uniform(size=L) for _ in range(K - 1)], dtype=np.float64).reshape(K - 1, L)
    return first, u


def _check_kmeans_input(x, K):
    """sklearn's validation of X and n_clusters, and the device limits; x is a CUDA tensor or an ndarray."""
    if x.ndim != 2:
        raise ValueError(f'Expected 2D array, got {x.ndim}D array instead.')
    if not _is_real(x):
        raise ValueError('Complex data not supported')
    N, E = x.shape
    if not 1 <= K <= KMEANS_MAX_K:
        raise ValueError(f'n_clusters={K}: the device k-means supports 1 <= K <= {KMEANS_MAX_K}')
    check_embedding_dim(E)
    if N < K:
        raise ValueError(f'n_samples={N} should be >= n_clusters={K}.')


def _kmeans_fit(x, K, init=None, max_ctas=0):
    """KMeans(n_clusters=K).fit(x) on the device, or KMeans(n_clusters=K, init=init, n_init=1).fit(x) with init (K, E)
    -- the latter only for tests, as is max_ctas > 0, a cap on the grid (the results do not depend on it).  x: a 2-D
    ndarray or CUDA tensor, already checked."""
    like_numpy = not _device.is_tensor(x)
    N, E = x.shape
    xd = _dev(x)
    dev_init, uniforms, first = None, None, 0
    if init is not None:
        dev_init = _dev(init)
    else:
        f32 = x.dtype == (np.float32 if like_numpy else torch.float32)
        first, u = _kmeans_draws(N, K, np.float32 if f32 else np.float64)
        if K > 1:
            uniforms = _device.to_device(u, torch.float64)
    lib = _lib.load()
    ws = _device.workspace(int(lib.pbb_kmeans_workspace_bytes(N, E, K)))
    centres = _device.empty((K, E), torch.float64)
    labels = _device.empty((N,), torch.int32)
    inertia = _device.empty((), torch.float64)
    n_iter = _device.empty((), torch.int32)
    status = _device.empty((1,), torch.int32)
    _device.call('pbb_kmeans_fit', xd, N, E, K, first, uniforms, dev_init, _KMEANS_MAX_ITER, ws, ws.numel(), centres,
                 labels, inertia, n_iter, status, max_ctas)

    def on_status(s):
        if s & 1:
            raise ValueError('Input X contains NaN or infinity.')
        warnings.warn(f'Number of distinct clusters ({s >> 8}) found smaller than n_clusters ({K}). Possibly due to '
                      'duplicate points in X.', ConvergenceWarning, stacklevel=3)
    _device.check_status(status, on_status)
    if like_numpy:
        return KMeans(K, centres.cpu().numpy(), labels.cpu().numpy(), float(inertia.item()), int(n_iter.item()))
    return KMeans(K, centres, labels, inertia, n_iter)


@dataclass
class KMeans:
    """The fitted attributes of sklearn.cluster.KMeans that BinaryGMM users read.  From NumPy input: ndarrays, a float
    inertia_ and an int n_iter_; from a CUDA tensor: CUDA tensors, inertia_ and n_iter_ 0-d (read without a host
    synchronisation only when asked for)."""
    n_clusters: int
    cluster_centers_: Any   # (K, E) float64
    labels_: Any            # (N_fit,) int32
    inertia_: Any
    n_iter_: Any

    def _labels_one_hot(self, x, one_hot):
        N, E = x.shape
        K = self.n_clusters
        if E != self.cluster_centers_.shape[1]:
            raise ValueError(f'X has {E} features, but KMeans is expecting {self.cluster_centers_.shape[1]} features '
                             'as input.')
        xd = _dev(x)
        labels = None if one_hot else _device.empty((N,), torch.int32)
        oh = _device.empty((K, N), torch.float64) if one_hot else None
        _device.call('pbb_kmeans_predict', xd, N, E, K, _dev(self.cluster_centers_), labels, oh)
        return oh if one_hot else labels

    def predict(self, x):
        """KMeans.predict: x (N, E) real -> the index of the closest centre (N,) int32."""
        like_numpy = not _device.is_tensor(x)
        if x.ndim != 2:
            raise ValueError(f'Expected 2D array, got {x.ndim}D array instead.')
        if not _is_real(x):
            raise ValueError('Complex data not supported')
        return _device.to_host(self._labels_one_hot(x, one_hot=False), like_numpy)


@dataclass
class BinaryGMM(_ProbabilisticModel):
    kmeans: KMeans

    def predict(self, x):
        """x (N, E) -> affiliation (K, N), the one-hot of the closest centre in x.dtype (gmm.py:180-198)."""
        like_numpy = not _device.is_tensor(x)
        N, D = x.shape
        assert _is_real(x), x.dtype
        check_embedding_dim(D)
        oh = self.kmeans._labels_one_hot(x, one_hot=True)
        if like_numpy:
            return oh.cpu().numpy().astype(x.dtype, copy=False)
        return oh if oh.dtype == x.dtype else oh.to(x.dtype)


class BinaryGMMTrainer:
    """k-means trainer (gmm.py:201-230): sklearn's ``KMeans(n_clusters=num_classes).fit`` on the device, with its
    k-means++ draws taken from NumPy's global RandomState in sklearn's order, so ``np.random.seed(s)`` reproduces the
    reference's fit.  Integer and float32 input are computed in float64 (sklearn computes float32 in float32).  With
    CUDA input the fit only enqueues work, except that a CUDA ``saliency`` selects its rows with a host
    synchronisation (``x[saliency]``); the non-finite check and the distinct-cluster warning come from a device
    status word, read at the end of a ``deferred_status()`` block."""

    def fit(self, x, num_classes, saliency=None):
        """x (N, E) real, num_classes K, saliency None or a boolean (N,) selecting the rows to fit."""
        if x.ndim != 2:
            raise ValueError(f'Expected 2D array, got {x.ndim}D array instead.')
        N, D = x.shape
        if saliency is not None:
            assert saliency.dtype in (bool, np.bool_, torch.bool), (
                'Only boolean saliency supported. '
                f'Current dtype: {saliency.dtype}.'
            )
            assert tuple(saliency.shape) == (N,)
            if _device.is_tensor(x):
                x = x[_device.to_device(saliency)]
            else:
                x = x[np.asarray(saliency.cpu() if _device.is_tensor(saliency) else saliency), :]
        _check_kmeans_input(x, num_classes)
        return BinaryGMM(kmeans=_kmeans_fit(x, num_classes))
