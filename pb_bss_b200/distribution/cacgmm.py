"""cACGMM: ``CACGMMTrainer.fit / fit_predict`` and ``CACGMM.predict /
log_likelihood`` with the signatures of pb_bss/distribution/cacgmm.py, executed
by the CUDA kernels behind ``pbb_cacgmm_fit`` / ``pbb_cacgmm_predict``.

numpy in -> numpy out (host buffers, copies included); CUDA tensors in -> CUDA
tensors out (everything stays resident in HBM).

Autograd: when grad mode is on and a CUDA tensor argument requires grad, ``cacgmm_m_step`` (and
``CACGMMTrainer._m_step``), ``CACGMM.predict``, ``CACGMM.log_likelihood`` and ``CACGMMTrainer.fit`` / ``fit_predict``
build a graph; otherwise every call runs the code path it runs without autograd.  The M-step is differentiable with
respect to y, the affiliation, the quadratic form and the saliency; predict and log_likelihood with respect to y and
the model's eigenvectors, eigenvalues and weight; the fit with respect to y, an affiliation initialisation, the
saliency and a warm-start model's tensors.  The backward passes are pbb_cacgmm_mstep_backward and
pbb_cacgmm_predict_backward (closed forms in include/pbb.h): gradients come back in the input's dtype, repeated
backward calls are bitwise identical, the backward only enqueues work, and double backward raises.  The floors and
clips pass no gradient where they are active, a zero frame has a zero gradient, the source activity mask is a
constant, a class whose affiliations sum to at most tiny passes no gradient, and a pair of floored model eigenvalues
contributes nothing through the eigenvectors, so rank-deficient scatter matrices give finite gradients.  Tied
unfloored eigenvalues take the Daleckii-Krein limit, and a floored and an unfloored eigenvalue within rounding of
each other (at the floor's kink) contribute nothing.  The eigenvector gradient is exact for every loss that sees the
model through B^-1 and log det B (predict, log_likelihood, the next E-step); for a loss on the eigenvectors
themselves it holds their phase fixed, and at a tie it is that convention.  A bin with a zero model eigenvalue or a non-finite sample gets NaN
gradients in that bin only.

The M-step, predict and log_likelihood with a graph launch what they launch without one, so their outputs are
bitwise unchanged.  A fit with a graph cannot run the persistent EM kernel, which keeps no per-iteration state: it
runs the reference's loop (cacgmm.py:252-278) as an M-step from the initialisation, then per iteration predict
(with affiliation_eps and the quadratic form) and an M-step, each a differentiable node.  Its model equals that loop
bitwise and agrees with the fit without a graph to the rounding of the persistent kernel's intermediate
Gauss-Jordan updates (about 1e-8 relative).  Autograd keeps every iteration's affiliation and quadratic form,
2 F K T float64 values per iteration (about 12 MB at F = 513, T = 500, K = 3).  Frequency-tied weights
(weight_constant_axis (-3,) / (-3, -1)), time-varying model weights and inline_permutation_aligner raise
NotImplementedError when a graph is needed.
"""
import ctypes
from dataclasses import dataclass, field

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _device, _lib
from . import complex_circular_symmetric_gaussian as _ccsg
from .complex_angular_central_gaussian import (
    ComplexAngularCentralGaussian,
    normalize_observation,
)
from .mixture_model_utils import (check_initialization, coupled_fit, fit_tied_leading, flatten_obs, initial_affiliation,
                                  model_to_host, saliency_bn, status_check, weight_mode, weight_to_device,
                                  weight_to_host)
from .utils import _ProbabilisticModel

__all__ = ['CACGMM', 'CACGMMTrainer', 'sample_cacgmm', 'normalize_observation']

_NORMS = {'eigenvalue': _lib.NORM_EIGENVALUE, 'trace': _lib.NORM_TRACE,
          False: _lib.NORM_NONE}


def _needs_graph(*ts):
    return torch.is_grad_enabled() and any(_device.is_tensor(t) and t.is_cuda and t.requires_grad for t in ts)


def _model_tensors(model):
    return model.weight, model.cacg.covariance_eigenvectors, model.cacg.covariance_eigenvalues


def _predict_launch(yd, V, lam, w, wmode, act, affiliation_eps, aff, q, ll):
    """pbb_cacgmm_predict of yd (..., N, D) into aff / q (F, K, N) and ll (F) (each may be None)."""
    _, F, N, D = flatten_obs(yd)
    K = V.shape[-3]
    status = _device.empty((1,), torch.int32)
    lib = _lib.load()
    nbytes = lib.pbb_cacgmm_workspace_bytes(F, N, D, K)
    ws = _device.workspace(nbytes)
    _device.call('pbb_cacgmm_predict', yd, _device.complex_dtype_code(yd), F, N, D, K, V, lam, w, wmode, act,
                 float(affiliation_eps), aff, q, ll, ws, nbytes, status)
    status_check(status, 'CACGMM.predict')


def _mstep_launch(yd, aff, q, sal, opts):
    """pbb_cacgmm_mstep of yd (..., N, D) from aff / q (F, K, N) and sal (F, N) -> V, lam, w (F, ...)"""
    _, F, N, D = flatten_obs(yd)
    K = aff.shape[-2]
    V = _device.empty((F, K, D, D), torch.complex128)
    lam = _device.empty((F, K, D), torch.float64)
    w = _device.empty((F, K), torch.float64)
    status = _device.empty((1,), torch.int32)
    lib = _lib.load()
    nbytes = lib.pbb_cacgmm_workspace_bytes(F, N, D, K)
    ws = _device.workspace(nbytes)
    _device.call('pbb_cacgmm_mstep', yd, _device.complex_dtype_code(yd), F, N, D, K, aff, q, sal, ctypes.byref(opts), V,
                 lam, w, ws, nbytes, status)
    status_check(status, 'cacgmm_m_step')
    return V, lam, w


def _flat(t, *shape):
    return None if t is None else t.contiguous().reshape(*shape)


class _Predict(torch.autograd.Function):
    """One E-step of y (F, N, D) under the model V (F, K, D, D), lam (F, K, D), w (F, K) by pbb_cacgmm_predict ->
    affiliation, quadratic form (F, K, N) and, with want_ll, the per-bin log-likelihood (F) (else an empty tensor);
    backward: pbb_cacgmm_predict_backward."""

    @staticmethod
    def forward(ctx, y, V, lam, w, act, affiliation_eps, want_ll):
        F, N, _ = y.shape
        K = V.shape[1]
        aff = _device.empty((F, K, N), torch.float64)
        q = _device.empty((F, K, N), torch.float64)
        ll = _device.empty((F,), torch.float64) if want_ll else _device.empty((0,), torch.float64)
        _predict_launch(y, V, lam, w, _lib.WEIGHT_TIME, act, affiliation_eps, aff, q, ll if want_ll else None)
        ctx.save_for_backward(y, V, lam, w, act, aff, q)
        ctx.affiliation_eps = affiliation_eps
        return aff, q, ll

    @staticmethod
    @once_differentiable
    def backward(ctx, gaff, gq, gll):
        y, V, lam, w, act, aff, q = ctx.saved_tensors
        F, N, D = y.shape
        K = V.shape[1]
        gy = _device.empty((F, N, D), torch.complex128)
        gV = _device.empty((F, K, D, D), torch.complex128)
        glam = _device.empty((F, K, D), torch.float64)
        gw = _device.empty((F, K), torch.float64)
        gll = gll if gll is not None and gll.numel() else None
        lib = _lib.load()
        nbytes = lib.pbb_cacgmm_predict_backward_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cacgmm_predict_backward', y, _device.complex_dtype_code(y), F, N, D, K, V, lam, w, act,
                     float(ctx.affiliation_eps), aff, q, _flat(gaff, F, K, N), _flat(gq, F, K, N), _flat(gll, F), gy,
                     gV, glam, gw, ws, nbytes)
        return gy.to(y.dtype), gV.to(V.dtype), glam, gw, None, None, None


class _MStep(torch.autograd.Function):
    """One M-step of y (F, N, D) from the affiliation (F, K, N), the quadratic form (F, K, N) or None and the
    saliency (F, N) or None by pbb_cacgmm_mstep -> V, lam, w; backward: pbb_cacgmm_mstep_backward."""

    @staticmethod
    def forward(ctx, y, aff, q, sal, opts):
        V, lam, w = _mstep_launch(y, aff, q, sal, opts)
        ctx.save_for_backward(y, aff, q, sal, V, lam)
        ctx.opts = opts
        return V, lam, w

    @staticmethod
    @once_differentiable
    def backward(ctx, gV, glam, gw):
        y, aff, q, sal, V, lam = ctx.saved_tensors
        F, N, D = y.shape
        K = aff.shape[1]
        gy = _device.empty((F, N, D), torch.complex128)
        gaff = _device.empty((F, K, N), torch.float64)
        gq = _device.empty((F, K, N), torch.float64) if q is not None else None
        gsal = _device.empty((F, N), torch.float64) if sal is not None else None
        lib = _lib.load()
        nbytes = lib.pbb_cacgmm_mstep_backward_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cacgmm_mstep_backward', y, _device.complex_dtype_code(y), F, N, D, K, aff, q, sal,
                     ctypes.byref(ctx.opts), V, lam, _flat(gV, F, K, D, D), _flat(glam, F, K, D), _flat(gw, F, K), gy,
                     gaff, gq, gsal, ws, nbytes)
        return gy.to(y.dtype), gaff, gq, gsal, None


def sample_cacgmm(size, weight, covariance, return_label=False):
    """``size`` samples (size, D) of a cACGMM (cacgmm.py:27-55): labels from ``np.random.choice(range(K), size,
    p=weight)``, then, class by class, ``from_covariance(covariance[l]).sample((count_l,))`` -- the same draws from
    NumPy's global stream in the same order, so the result equals that loop exactly.  The K models come from one
    ``pbb_cacg_from_covariance`` and all samples from one ``pbb_ccsg_sample`` launch.  The argument checks are
    assertions, as in the reference."""
    assert weight.ndim == 1, weight
    assert isinstance(size, int), size
    assert covariance.ndim == 3, covariance.shape
    num_classes, = weight.shape
    D = covariance.shape[-1]
    assert tuple(covariance.shape) == (num_classes, D, D), (covariance.shape, num_classes, D)
    p = weight.cpu().numpy() if _device.is_tensor(weight) else weight
    labels = np.random.choice(range(num_classes), size=size, p=p)
    model = ComplexAngularCentralGaussian.from_covariance(_device.to_device(covariance, torch.complex128))
    draws, dest = [], []
    for k in range(num_classes):
        rows = np.flatnonzero(labels == k)
        draws.append((np.random.normal(size=(rows.size, D)), np.random.normal(size=(rows.size, D))))
        dest.append(rows)
    x = _ccsg.sample_classes(model.covariance_eigenvectors, model.covariance_eigenvalues, draws, True,
                             not _device.is_tensor(covariance), dest=np.concatenate(dest))
    if return_label:
        return x, labels
    return x


@dataclass
class CACGMM(_ProbabilisticModel):
    weight: np.array = None  # (..., K, 1), or (K, 1) for weight_constant_axis=-2
    cacg: ComplexAngularCentralGaussian = field(
        default_factory=ComplexAngularCentralGaussian)

    # -- device views of the model ------------------------------------------------
    def _device_model(self, independent, F, N):
        V = _device.to_device(self.cacg.covariance_eigenvectors, torch.complex128)
        lam = _device.to_device(self.cacg.covariance_eigenvalues, torch.float64)
        K, D = V.shape[-3], V.shape[-1]
        V = V.expand(*independent, K, D, D).reshape(F, K, D, D).contiguous()
        lam = lam.expand(*independent, K, D).reshape(F, K, D).contiguous()
        return V, lam, *weight_to_device(self.weight, independent, F, K, N), K

    def _run_predict(self, y, source_activity_mask, affiliation_eps,
                     want_aff=True, want_q=False, want_ll=False):
        graph = _needs_graph(y, *_model_tensors(self))
        like_numpy = not _device.is_tensor(y) and not graph
        yd = _device.to_device(y)
        independent, F, N, D = flatten_obs(yd)
        V, lam, w, wmode, K = self._device_model(independent, F, N)
        assert V.shape[-1] == D, (V.shape, D)
        act = None
        if source_activity_mask is not None:
            assert source_activity_mask.dtype in (bool, np.bool_, torch.bool), source_activity_mask.dtype
            act = _device.to_device(source_activity_mask).to(torch.uint8)
            act = act.expand(*independent, K, N).reshape(F, K, N).contiguous()
        shape = (*independent, K, N)
        if graph:
            if wmode != _lib.WEIGHT_TIME:
                raise NotImplementedError('CACGMM.predict with a graph: only per-bin weights (..., K, 1) are '
                                          'differentiable, not time-varying or frequency-tied ones')
            aff, q, ll = _Predict.apply(yd.reshape(F, N, D), V, lam, w, act, float(affiliation_eps), want_ll)
            return (aff.reshape(shape) if want_aff else None, q.reshape(shape) if want_q else None,
                    ll if want_ll else None, False)
        aff = _device.empty((F, K, N), torch.float64) if want_aff else None
        q = _device.empty((F, K, N), torch.float64) if want_q else None
        ll = _device.empty((F,), torch.float64) if want_ll else None
        _predict_launch(yd, V, lam, w, wmode, act, affiliation_eps, aff, q, ll)
        if aff is not None:
            aff = _device.to_host(aff.reshape(shape), like_numpy)
        if q is not None:
            q = _device.to_host(q.reshape(shape), like_numpy)
        return aff, q, ll, like_numpy

    def predict(self, y, return_quadratic_form=False, source_activity_mask=None):
        """Posterior affiliations (..., K, N) for observations y (..., N, D).

        cacgmm.py:64-71: normalise, one E-step, affiliation_eps = 0.  Differentiable with respect to y and the
        model's tensors (see the module's docstring)."""
        aff, q, _, _ = self._run_predict(y, source_activity_mask, 0.,
                                         want_q=return_quadratic_form)
        return (aff, q) if return_quadratic_form else aff

    def log_likelihood(self, y):
        """sum_{f,t} logsumexp_k log_pdf (without weights), cacgmm.py:97-138.  Differentiable with respect to y and
        the model's eigenvectors and eigenvalues (see the module's docstring)."""
        _, _, ll, like_numpy = self._run_predict(y, None, 0., want_aff=False,
                                                 want_ll=True)
        total = ll.sum()
        return np.float64(total.item()) if like_numpy else total


class CACGMMTrainer:
    def fit(
            self,
            y,
            initialization=None,
            num_classes=None,
            iterations=100,
            *,
            saliency=None,
            source_activity_mask=None,
            weight_constant_axis=(-1,),
            hermitize=True,
            covariance_norm='eigenvalue',
            affiliation_eps=1e-10,
            eigenvalue_floor=1e-10,
            inline_permutation_aligner=None,
            frames_per_block=0,
            multi_kernel=False,
            total_bins=None,
            bin_group=None,
    ):
        """EM for the cACGMM, signature of cacgmm.py:142-157.

        Args:
            y: (..., N, D) complex64/128; numpy array or CUDA tensor.
            initialization: affiliations (..., K, N) (singleton independent
                dims broadcast) or a ``CACGMM`` (warm start).
            num_classes: K, if no initialization is given (the init is then
                drawn from NumPy's global RNG exactly like cacgmm.py:206-209).
            saliency: (..., N); source_activity_mask: bool (..., K, N).
            weight_constant_axis: (-1,) or -2 on the device.
            covariance_norm: 'eigenvalue', 'trace' or False.
            frames_per_block: tuning knob of the multi-kernel EM path (0 = default).
            multi_kernel: force the one-kernel-pair-per-iteration path instead
                of the persistent kernel (A/B testing; same results).
            total_bins, bin_group: bin-sharded multi-GPU use (pb_bss_b200.parallel):
                ``y`` holds this rank's contiguous slice of ``total_bins`` bins.  Only
                the couplings across bins (frequency-tied weights, inline alignment)
                communicate, once per iteration.
        Returns: CACGMM.  With a graph (a CUDA tensor argument that requires grad) the fit runs the reference's
        loop of differentiable E- and M-steps and returns CUDA tensors (see the module's docstring).
        """
        check_initialization(initialization, num_classes)
        assert covariance_norm in _NORMS, covariance_norm
        like_numpy = not _device.is_tensor(y)
        mode = weight_mode(weight_constant_axis, y.ndim)
        tied = mode in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED)
        coupled = inline_permutation_aligner is not None or tied
        graph = _needs_graph(y, initialization, saliency,
                             *(_model_tensors(initialization) if isinstance(initialization, CACGMM) else ()))
        if graph:
            if coupled:
                raise NotImplementedError('CACGMMTrainer.fit with a graph: frequency-tied weights and '
                                          'inline_permutation_aligner are not differentiable')
            return self._fit_graph(y, initialization, num_classes, iterations, saliency, source_activity_mask,
                                   weight_constant_axis, covariance_norm, affiliation_eps, eigenvalue_floor,
                                   total_bins, bin_group)
        # pinned host tensors stay where they are: pbb_cacgmm_fit streams them in while it computes
        yd = _device.to_device(y, keep_pinned=not coupled)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1, yd.shape
        assert iterations > 0, iterations
        code = _device.complex_dtype_code(yd)
        independent, F, N, D = flatten_obs(yd)
        assert D < 35, f'Channels: {D}, sure?'

        init_dev = None
        model_in = None
        if initialization is None:
            K = num_classes
            init_dev = initial_affiliation(None, K, independent, N)
        elif isinstance(initialization, CACGMM):
            model_in = initialization
            K = initialization.cacg.covariance_eigenvectors.shape[-3]
        elif isinstance(initialization, (np.ndarray, torch.Tensor)):
            K = initialization.shape[-2]
            assert K > 1, K
            shape = (*independent, K, N)
            assert initialization.ndim == len(shape), (initialization.shape, shape)
            assert tuple(initialization.shape[-2:]) == shape[-2:], (initialization.shape, shape)
            init_dev = _device.to_device(initialization, torch.float64, keep_pinned=yd.device.type == 'cpu')
            init_dev = init_dev.expand(shape).reshape(F, K, N)
            if not init_dev.is_contiguous():
                # broadcast singleton dims materialise a new tensor: keep it where the library can read it
                init_dev = init_dev.contiguous()
                if init_dev.device.type == 'cpu':
                    init_dev = init_dev.pin_memory()
        else:
            raise TypeError('No sufficient initialization.')
        assert K < 20, f'num_classes: {K}, sure?'
        sal = saliency_bn(saliency, independent, N)
        if tied and len(independent) > 1:
            assert model_in is None, 'warm start with tied weights: one leading dim only'
            model = fit_tied_leading(
                self.fit, independent[:-1], y=yd, initialization=init_dev.reshape(*independent, K, N),
                iterations=iterations, saliency=saliency, source_activity_mask=source_activity_mask,
                weight_constant_axis=weight_constant_axis, hermitize=hermitize, covariance_norm=covariance_norm,
                affiliation_eps=affiliation_eps, eigenvalue_floor=eigenvalue_floor,
                inline_permutation_aligner=inline_permutation_aligner)
            return model_to_host(model) if like_numpy else model
        if coupled:
            # frequency-tied weights and the inline permutation alignment couple the bins inside the
            # EM loop (cacgmm.py:252-278): one E-step / alignment / M-step round trip per iteration
            mask = source_activity_mask
            if mask is not None and not _device.is_tensor(mask):
                mask = _device.to_device(mask)   # uploaded once, not per iteration
            model = coupled_fit(
                yd, init_dev, model_in, iterations, weight_constant_axis, sal, inline_permutation_aligner,
                predict=lambda m: m._run_predict(yd, mask, affiliation_eps, want_q=True)[:2],
                m_step=lambda aff, q: cacgmm_m_step(yd, q, aff, saliency=sal, hermitize=hermitize,
                                                    covariance_norm=covariance_norm, eigenvalue_floor=eigenvalue_floor),
                saliency_form=sal is not None, total_bins=total_bins, bin_group=bin_group)
            return model_to_host(model) if like_numpy else model

        act = None
        if source_activity_mask is not None:
            assert source_activity_mask.dtype in (bool, np.bool_, torch.bool), source_activity_mask.dtype
            assert tuple(source_activity_mask.shape[-2:]) == (K, N), (source_activity_mask.shape, K, N)
            if isinstance(initialization, (np.ndarray, torch.Tensor)):
                assert source_activity_mask.shape == initialization.shape, (
                    source_activity_mask.shape, initialization.shape)
            act = _device.to_device(source_activity_mask).to(torch.uint8)
            act = act.expand(*independent, K, N).reshape(F, K, N).contiguous()

        if model_in is not None:
            V, lam, w, wm_in, _ = model_in._device_model(independent, F, N)
            assert wm_in == _lib.WEIGHT_TIME, 'warm start with frequency-tied weights goes through the coupled loop'
            V, lam, w = V.clone(), lam.clone(), w.clone()
        elif yd.device.type == 'cpu':
            # pinned observation in, pinned model out: the final update kernel writes it over PCIe
            V = torch.empty((F, K, D, D), dtype=torch.complex128, pin_memory=True)
            lam = torch.empty((F, K, D), dtype=torch.float64, pin_memory=True)
            w = torch.empty((F, K), dtype=torch.float64, pin_memory=True)
        else:
            V = _device.empty((F, K, D, D), torch.complex128)
            lam = _device.empty((F, K, D), torch.float64)
            w = _device.empty((F, K), torch.float64)
        status = _device.empty((1,), torch.int32)
        opts = _lib.CacgmmOptions(
            iterations=int(iterations), covariance_norm=_NORMS[covariance_norm],
            weight_mode=mode, hermitize=int(bool(hermitize)),
            affiliation_eps=float(affiliation_eps),
            eigenvalue_floor=float(eigenvalue_floor),
            frames_per_block=int(frames_per_block),
            reserved=1 if multi_kernel else 0)
        lib = _lib.load()
        nbytes = lib.pbb_cacgmm_workspace_bytes(F, N, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_cacgmm_fit', yd, code, F, N, D, K, init_dev, sal, act, ctypes.byref(opts), V, lam, w, ws,
                     nbytes, status)
        status_check(status, 'CACGMMTrainer.fit')
        return CACGMM(
            weight=weight_to_host(mode, w, independent, K, like_numpy),
            cacg=ComplexAngularCentralGaussian(
                covariance_eigenvectors=_device.to_host(
                    V.reshape(*independent, K, D, D), like_numpy),
                covariance_eigenvalues=_device.to_host(
                    lam.reshape(*independent, K, D), like_numpy)))

    def _fit_graph(self, y, initialization, num_classes, iterations, saliency, source_activity_mask,
                   weight_constant_axis, covariance_norm, affiliation_eps, eigenvalue_floor, total_bins, bin_group):
        """The fit with a graph: the reference's loop (cacgmm.py:252-278) through coupled_fit, every E-step and
        M-step a differentiable node; frames_per_block and multi_kernel do not apply."""
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1, yd.shape
        assert iterations > 0, iterations
        independent, F, N, D = flatten_obs(yd)
        assert D < 35, f'Channels: {D}, sure?'
        model_in, aff = None, None
        if initialization is None:
            K = num_classes
            aff = initial_affiliation(None, K, independent, N).reshape(*independent, K, N)
        elif isinstance(initialization, CACGMM):
            model_in = initialization
            K = initialization.cacg.covariance_eigenvectors.shape[-3]
        elif isinstance(initialization, (np.ndarray, torch.Tensor)):
            K = initialization.shape[-2]
            assert K > 1, K
            shape = (*independent, K, N)
            assert initialization.ndim == len(shape), (initialization.shape, shape)
            assert tuple(initialization.shape[-2:]) == shape[-2:], (initialization.shape, shape)
            aff = _device.to_device(initialization, torch.float64).expand(shape)
        else:
            raise TypeError('No sufficient initialization.')
        assert K < 20, f'num_classes: {K}, sure?'
        mask = source_activity_mask
        if mask is not None:
            assert mask.dtype in (bool, np.bool_, torch.bool), mask.dtype
            assert tuple(mask.shape[-2:]) == (K, N), (mask.shape, K, N)
            mask = _device.to_device(mask)
        sal = None if saliency is None else _device.to_device(saliency, torch.float64)
        return coupled_fit(
            yd, aff, model_in, iterations, weight_constant_axis, None, None,
            predict=lambda m: m._run_predict(yd, mask, affiliation_eps, want_q=True)[:2],
            m_step=lambda a, q: cacgmm_m_step(yd, q, a, saliency=sal, covariance_norm=covariance_norm,
                                              eigenvalue_floor=eigenvalue_floor,
                                              weight_constant_axis=weight_constant_axis),
            saliency_form=False, total_bins=total_bins, bin_group=bin_group)

    def fit_predict(self, y, initialization=None, num_classes=None,
                    iterations=100, **kwargs):
        """Fit, then return the posterior affiliations (cacgmm.py:282-313)."""
        model = self.fit(y=y, initialization=initialization,
                         num_classes=num_classes, iterations=iterations,
                         **kwargs)
        return model.predict(y)

    def _m_step(self, x, quadratic_form, affiliation, saliency, hermitize,
                covariance_norm, eigenvalue_floor, weight_constant_axis):
        """One M-step, signature of cacgmm.py:315-345; ``x`` is the normalised
        observation in the reference's internal (..., D, N) layout."""
        if _device.is_tensor(x):
            y = x.transpose(-1, -2)
        else:
            y = np.swapaxes(x, -1, -2)
        return cacgmm_m_step(
            y, quadratic_form, affiliation, saliency=saliency,
            hermitize=hermitize, covariance_norm=covariance_norm,
            eigenvalue_floor=eigenvalue_floor,
            weight_constant_axis=weight_constant_axis)


def cacgmm_m_step(y, quadratic_form, affiliation, *, saliency=None,
                  hermitize=True, covariance_norm='eigenvalue',
                  eigenvalue_floor=1e-10, weight_constant_axis=(-1,)):
    """One M-step from given affiliations / quadratic forms (``pbb_cacgmm_mstep``).

    estimate_mixture_weight (mixture_model_utils.py:133-203) +
    ComplexAngularCentralGaussianTrainer._fit (cacg.py:253-342).
    y: (..., N, D); affiliation, quadratic_form: (..., K, N);
    quadratic_form=None means ones (the first EM iteration, cacgmm.py:210).
    """
    graph = _needs_graph(y, quadratic_form, affiliation, saliency)
    like_numpy = not _device.is_tensor(y) and not graph
    yd = _device.to_device(y)
    independent, F, N, D = flatten_obs(yd)
    aff = _device.to_device(affiliation, torch.float64)
    K = aff.shape[-2]
    aff = aff.expand(*independent, K, N).reshape(F, K, N).contiguous()
    q = None
    if quadratic_form is not None:
        q = _device.to_device(quadratic_form, torch.float64)
        q = q.expand(*independent, K, N).reshape(F, K, N).contiguous()
    sal = None
    if saliency is not None:
        sal = _device.to_device(saliency, torch.float64)
        sal = sal.expand(*independent, N).reshape(F, N).contiguous()
    mode = weight_mode(weight_constant_axis, len(independent) + 2)
    opts = _lib.CacgmmOptions(
        iterations=1, covariance_norm=_NORMS[covariance_norm],
        weight_mode=mode, hermitize=int(bool(hermitize)),
        affiliation_eps=0., eigenvalue_floor=float(eigenvalue_floor),
        frames_per_block=0, reserved=0)
    if graph:
        if mode not in (_lib.WEIGHT_TIME, _lib.WEIGHT_CONST):
            raise NotImplementedError('cacgmm_m_step with a graph: frequency-tied weights (weight_constant_axis '
                                      '(-3,) / (-3, -1)) are not differentiable')
        V, lam, w = _MStep.apply(yd.reshape(F, N, D), aff, q, sal, opts)
    else:
        V, lam, w = _mstep_launch(yd, aff, q, sal, opts)
    return CACGMM(
        weight=weight_to_host(mode, w, independent, K, like_numpy),
        cacg=ComplexAngularCentralGaussian(
            covariance_eigenvectors=_device.to_host(
                V.reshape(*independent, K, D, D), like_numpy),
            covariance_eigenvalues=_device.to_host(
                lam.reshape(*independent, K, D), like_numpy)))
