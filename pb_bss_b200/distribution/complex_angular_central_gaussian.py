"""Complex angular central Gaussian -- ``ComplexAngularCentralGaussian``, its trainer and
``sample_complex_angular_central_gaussian`` with the names, arguments, defaults and error types of
pb_bss/distribution/complex_angular_central_gaussian.py.

The model is stored as eigenvectors / eigenvalues of the covariance (:78-79); ``covariance`` (:140-148) and
``log_determinant`` (:150-152) are derived properties.  NumPy in gives NumPy out; CUDA tensors in give CUDA tensors
out.  The arithmetic runs in fp64 on the device:
  - ``from_covariance``: ``pbb_cacg_from_covariance`` (Jacobi eigendecomposition, norm and floor);
  - ``log_pdf`` / ``_log_pdf``: the quadratic form of ``pbb_cacgmm_predict`` and ``pbb_cacg_log_pdf_floor``;
  - ``ComplexAngularCentralGaussianTrainer.fit``: ``pbb_cacgmm_fit`` with one class, all-ones affiliations and
    affiliation_eps = 0, so every posterior is 1 and each M-step is the reference's ``_fit``;
  - ``ComplexAngularCentralGaussianTrainer._fit``: ``pbb_cacgmm_mstep``;
  - ``sample``: ``pbb_ccsg_sample``, the draws from NumPy's global stream on the host.

Differences from the reference:
  - ``ComplexAngularCentralGaussianTrainer.fit`` fits every leading index of y independently; the reference raises
    TypeError for any y with leading dims (``np.ones(*independent, N)``).
  - ``from_covariance(covariance_norm='trace')`` leaves the caller's array as it is; the reference divides it in
    place.
  - The eigenvalues come from a Jacobi solver, the eigenvectors' phases from it too: compare models through
    ``covariance``.
  - D is limited to 34 for ``log_pdf`` and the trainer, like the mixture model, and to 64 for ``from_covariance``.
"""
import ctypes
from dataclasses import dataclass

import numpy as np
import torch

from .. import _device, _lib
from . import complex_circular_symmetric_gaussian as _ccsg
from .mixture_model_utils import status_check
from .utils import _ProbabilisticModel

__all__ = [
    'ComplexAngularCentralGaussian',
    'ComplexAngularCentralGaussianTrainer',
    'sample_complex_angular_central_gaussian',
    'normalize_observation',
]

_NORMS = {'eigenvalue': _lib.NORM_EIGENVALUE, 'trace': _lib.NORM_TRACE, False: _lib.NORM_NONE}
_MAX_GRID_Y = 65535  # pbb_cacg_log_pdf_floor launches one CTA row per (bin, class)
_MAX_CLASSES = 19    # pbb_cacgmm_predict takes K < 20 classes (kMaxK, cacgmm.py:249)


def normalize_observation(observation):
    """(..., N, D) -> unit-norm (..., D, N) on the device.

    complex_angular_central_gaussian.py:34-55 (zero vectors stay zero).
    numpy in -> numpy out, CUDA tensor in -> CUDA tensor out.
    """
    like_numpy = not _device.is_tensor(observation)
    y = _device.to_device(observation)
    code = _device.complex_dtype_code(y)
    *independent, N, D = y.shape
    F = int(np.prod(independent)) if independent else 1
    z = torch.empty((*independent, D, N), dtype=y.dtype, device=y.device)
    _device.call('pbb_normalize_observation', y, z, F, N, D, code, 1)
    return _device.to_host(z, like_numpy)


def sample_complex_angular_central_gaussian(size, covariance):
    """Circular-symmetric Gaussian samples (*size, D) of ``covariance`` (D, D), scaled to unit norm
    (complex_angular_central_gaussian.py:58-65).  Errors as ``ComplexCircularSymmetricGaussian.sample``."""
    return _ccsg.sample(size, covariance, None, unit_norm=True)


def _tiny(dtype):
    """np.finfo(y.dtype).tiny of the observation's torch dtype."""
    single = dtype in (torch.complex64, torch.float32)
    return float(np.finfo(np.float32 if single else np.float64).tiny)


def _check_norm(covariance_norm):
    if covariance_norm != 'trace':
        assert covariance_norm in ['eigenvalue', False]


@dataclass
class ComplexAngularCentralGaussian(_ProbabilisticModel):
    covariance_eigenvectors: np.array = None  # (..., D, D)
    covariance_eigenvalues: np.array = None  # (..., D)

    @classmethod
    def from_covariance(cls, covariance, eigenvalue_floor=0., covariance_norm='eigenvalue'):
        """Eigendecomposition of covariance (..., D, D) with the reference's norm and floor
        (complex_angular_central_gaussian.py:81-132): 'trace' divides by the trace first, 'eigenvalue' scales the
        largest eigenvalue to 1 and floors at ``eigenvalue_floor``, False floors at the largest eigenvalue times
        it.  Eigenvalues ascend.  An unknown norm or non-finite eigenvalues raise AssertionError; a non-finite
        covariance raises what the reference's eigh fallback raises (RuntimeError for eigenvalue_floor = 0, else
        LinAlgError).  The input is not changed."""
        _check_norm(covariance_norm)
        like_numpy = not _device.is_tensor(covariance)
        c = _ccsg._as_device(covariance, torch.complex128).contiguous()
        *lead, D, _ = c.shape
        n = int(np.prod(lead))
        V = _device.empty((n, D, D), torch.complex128)
        lam = _device.empty((n, D), torch.float64)
        if n:
            status = _device.empty((1,), torch.int32)
            _device.call('pbb_cacg_from_covariance', c, n, D, _NORMS[covariance_norm], float(eigenvalue_floor), V, lam,
                         status)

            def on_error(s):
                if torch.isfinite(torch.view_as_real(c[s - 1])).all():
                    raise AssertionError(f'non-finite eigenvalues (matrix {s - 1})')
                # np.linalg.eigh and eig fail on non-finite input; the reference reraises (:94-110)
                if eigenvalue_floor == 0:
                    raise RuntimeError(
                        'When you set the eigenvalue_floor to zero it can happen that the eigenvalues get zero and '
                        f'the reciprocal eigenvalue that is used in {cls.__name__}._log_pdf gets infinity.')
                raise np.linalg.LinAlgError(f'non-finite covariance (matrix {s - 1})')
            _device.check_status(status, on_error)
        return cls(covariance_eigenvalues=_device.to_host(lam.reshape(*lead, D), like_numpy),
                   covariance_eigenvectors=_device.to_host(V.reshape(*lead, D, D), like_numpy))

    def sample(self, size):
        """Samples (*size, D) of unit norm (complex_angular_central_gaussian.py:134-138); the covariance
        V diag(lambda) V^H is formed on the device.  Errors as ``ComplexCircularSymmetricGaussian.sample``."""
        return _ccsg.sample(size, self.covariance_eigenvectors, self.covariance_eigenvalues, unit_norm=True)

    @property
    def covariance(self):
        """V diag(lambda) V^H -- a derived view for inspection, not on the hot
        path (complex_angular_central_gaussian.py:140-148)."""
        V, lam = self.covariance_eigenvectors, self.covariance_eigenvalues
        if _device.is_tensor(V):
            return torch.einsum('...wx,...x,...zx->...wz', V, lam.to(V.dtype), V.conj())
        return np.einsum('...wx,...x,...zx->...wz', V, lam, V.conj())

    @property
    def log_determinant(self):
        lam = self.covariance_eigenvalues
        if _device.is_tensor(lam):
            return torch.sum(torch.log(lam), dim=-1)
        return np.sum(np.log(lam), axis=-1)

    def log_pdf(self, y):
        """log pdf (..., N) of observations y (..., N, D), normalised first (:154-165)."""
        log_pdf, _ = self._device_log_pdf(y, swapped=False)
        return log_pdf

    def _log_pdf(self, y):
        """(log_pdf, quadratic_form), both (..., N), of y (..., D, N) (:167-203).  q = max(|z^H B^-1 z|, tiny of
        y's dtype), log_pdf = -D log q - log det.  The model's leading dims broadcast against y's, e.g. a model
        (F, K, D, D) with y (F, 1, D, N).  The device normalises y again, which leaves the unit-norm observations
        the reference expects unchanged (zero vectors stay zero)."""
        return self._device_log_pdf(y, swapped=True)

    def _device_log_pdf(self, y, swapped):
        like_numpy = not _device.is_tensor(y)
        yd = _ccsg._as_device(y)
        tiny = _tiny(yd.dtype)
        if not yd.is_complex():
            yd = yd.to(torch.complex128)
        if swapped:
            yd = yd.transpose(-1, -2)
        V = _ccsg._as_device(self.covariance_eigenvectors, torch.complex128)
        lam = _ccsg._as_device(self.covariance_eigenvalues, torch.float64)
        D = V.shape[-1]
        N = yd.shape[-2]
        assert yd.shape[-1] == D, (tuple(yd.shape), tuple(V.shape))
        try:
            lead = torch.broadcast_shapes(tuple(yd.shape[:-2]), tuple(V.shape[:-2]), tuple(lam.shape[:-1]))
        except RuntimeError:
            raise AssertionError((tuple(yd.shape), tuple(V.shape))) from None
        # the last leading dim becomes the class axis K of pbb_cacgmm_predict when y is broadcast along it and it
        # fits the kernel's class limit; otherwise every model is its own bin (K = 1) and y is expanded
        ylead = (1,) * (len(lead) - (yd.dim() - 2)) + tuple(yd.shape[:-2])
        yd = yd.reshape(*ylead, N, D)
        if lead and ylead[-1] == 1 and 1 < lead[-1] <= _MAX_CLASSES:
            outer, K = tuple(lead[:-1]), lead[-1]
            yd = yd[..., 0, :, :]
        else:
            outer, K = tuple(lead), 1
        F = int(np.prod(outer))
        q_raw = _device.empty((F, K, N), torch.float64)
        q = _device.empty((F, K, N), torch.float64)
        out = _device.empty((F, K, N), torch.float64)
        if F and N:
            yf = yd.expand(*outer, N, D).reshape(F, N, D).contiguous()
            Vf = V.expand(*lead, D, D).reshape(F, K, D, D).contiguous()
            lamf = lam.expand(*lead, D).reshape(F, K, D).contiguous()
            status = _device.empty((1,), torch.int32)
            lib = _lib.load()
            nbytes = lib.pbb_cacgmm_workspace_bytes(F, N, D, K)
            ws = _device.workspace(nbytes)
            _device.call('pbb_cacgmm_predict', yf, _device.complex_dtype_code(yf), F, N, D, K, Vf, lamf, None,
                         _lib.WEIGHT_CONST, None, 0., None, q_raw, None, ws, nbytes, status)
            status_check(status, 'ComplexAngularCentralGaussian.log_pdf')
            step = max(1, _MAX_GRID_Y // K)
            for f0 in range(0, F, step):
                f1 = min(F, f0 + step)
                _device.call('pbb_cacg_log_pdf_floor', q_raw[f0:f1], lamf[f0:f1], f1 - f0, K, N, D, tiny, q[f0:f1],
                             out[f0:f1])
        shape = (*lead, N)
        return (_device.to_host(out.reshape(shape), like_numpy), _device.to_host(q.reshape(shape), like_numpy))


class ComplexAngularCentralGaussianTrainer:
    def fit(self, y, saliency=None, hermitize=True, covariance_norm='eigenvalue', eigenvalue_floor=1e-10,
            iterations=10):
        """Fixed-point iterations from q = 1 (complex_angular_central_gaussian.py:207-251) for y (..., N, D).

        Every leading index of y is fitted independently and equals the reference's 2-D fit of that slice (the
        reference itself raises TypeError for leading dims).  A saliency raises NotImplementedError, non-complex
        input or D = 1 AssertionError.  Runs as ``CACGMMTrainer.fit`` with one class: all-ones affiliations,
        affiliation_eps = 0, so every posterior is 1 and each M-step is ``_fit`` with denominator N.  Without frames
        the scatter matrix is zero, and the model is ``from_covariance`` of it, as in the reference."""
        *independent, N, D = y.shape
        assert np.iscomplexobj(y) if not _device.is_tensor(y) else y.is_complex(), y.dtype
        assert y.shape[-1] > 1
        if saliency is not None:
            raise NotImplementedError
        assert iterations > 0, iterations
        _check_norm(covariance_norm)
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        if N == 0:
            return _from_empty_scatter((*independent, D, D), eigenvalue_floor, covariance_norm, like_numpy)
        F = int(np.prod(independent))
        V = _device.empty((F, 1, D, D), torch.complex128)
        lam = _device.empty((F, 1, D), torch.float64)
        if F:
            w = _device.empty((F, 1), torch.float64)
            init = torch.ones((F, 1, N), dtype=torch.float64, device=yd.device)
            status = _device.empty((1,), torch.int32)
            opts = _lib.CacgmmOptions(
                iterations=int(iterations), covariance_norm=_NORMS[covariance_norm], weight_mode=_lib.WEIGHT_TIME,
                hermitize=int(bool(hermitize)), affiliation_eps=0., eigenvalue_floor=float(eigenvalue_floor),
                frames_per_block=0, reserved=0)
            lib = _lib.load()
            nbytes = lib.pbb_cacgmm_workspace_bytes(F, N, D, 1)
            ws = _device.workspace(nbytes)
            _device.call('pbb_cacgmm_fit', yd, _device.complex_dtype_code(yd), F, N, D, 1, init, None, None,
                         ctypes.byref(opts), V, lam, w, ws, nbytes, status)
            status_check(status, 'ComplexAngularCentralGaussianTrainer.fit')
        return ComplexAngularCentralGaussian(
            covariance_eigenvectors=_device.to_host(V.reshape(*independent, D, D), like_numpy),
            covariance_eigenvalues=_device.to_host(lam.reshape(*independent, D), like_numpy))

    def _fit(self, y, saliency, quadratic_form, hermitize=True, covariance_norm='eigenvalue',
             eigenvalue_floor=1e-10) -> ComplexAngularCentralGaussian:
        """One step of ``fit`` (complex_angular_central_gaussian.py:253-342): y (..., D, N) broadcast against
        quadratic_form (..., K, N) -> K covariances D sum_n s y y^H / q / (N, or sum_n s), then ``from_covariance``.
        Runs as ``pbb_cacgmm_mstep``, whose scatter sum is Hermitian by construction, so ``hermitize`` changes
        nothing.  The device normalises y again, which leaves the unit-norm observations the reference expects
        unchanged.  Without frames the scatter matrix is zero (``fit``)."""
        _check_norm(covariance_norm)
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        q = _ccsg._as_device(quadratic_form, torch.float64)
        try:
            lead = torch.broadcast_shapes(tuple(yd.shape[:-2]), tuple(q.shape[:-1]))
        except RuntimeError:
            raise AssertionError((tuple(yd.shape), tuple(q.shape))) from None
        D, N = yd.shape[-2], q.shape[-1]
        if saliency is None:
            aff = torch.ones((*lead, N), dtype=torch.float64, device=yd.device)
        else:
            assert yd.dim() == saliency.ndim + 1, (tuple(yd.shape), saliency.ndim)
            aff = _ccsg._as_device(saliency, torch.float64)
        if N == 0:
            return _from_empty_scatter((*lead, D, D), eigenvalue_floor, covariance_norm, like_numpy)
        F = int(np.prod(lead))
        y_nd = yd.expand(*lead, D, N).transpose(-1, -2).reshape(F, N, D).contiguous()
        from .cacgmm import cacgmm_m_step
        model = cacgmm_m_step(y_nd, q.expand(*lead, N).reshape(F, 1, N), aff.expand(*lead, N).reshape(F, 1, N),
                              hermitize=hermitize, covariance_norm=covariance_norm,
                              eigenvalue_floor=eigenvalue_floor).cacg
        return ComplexAngularCentralGaussian(
            covariance_eigenvectors=_device.to_host(model.covariance_eigenvectors.reshape(*lead, D, D), like_numpy),
            covariance_eigenvalues=_device.to_host(model.covariance_eigenvalues.reshape(*lead, D), like_numpy))


def _from_empty_scatter(shape, eigenvalue_floor, covariance_norm, like_numpy):
    """The model of zero frames: the reference's scatter sum is zero and its denominator max(0, tiny), so the fit is
    ``from_covariance`` of zero matrices (identity eigenvectors, eigenvalues max(0, floor) or 0)."""
    zeros = np.zeros(shape, dtype=np.complex128)
    return ComplexAngularCentralGaussian.from_covariance(
        zeros if like_numpy else _device.to_device(zeros), eigenvalue_floor=eigenvalue_floor,
        covariance_norm=covariance_norm)
