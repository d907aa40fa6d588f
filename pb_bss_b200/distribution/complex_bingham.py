"""Complex Bingham distribution -- ``ComplexBingham`` and ``ComplexBinghamTrainer`` with the names, arguments,
defaults and error types of pb_bss/distribution/complex_bingham.py, executed by the kernels behind
``pbb_bingham_log_norm``, ``pbb_bingham_log_pdf``, ``pbb_bingham_parameters`` and ``pbb_cbmm_fit``
(include/pbb.h).

Numerics that differ from the reference on purpose (see include/pbb.h):
  - the normaliser c(lambda) = 2 pi^D exp[lambda] is evaluated as a divided difference of exp, which stays
    exact for repeated eigenvalues (the reference's term-by-term sum is accurate to ~3e-8 there);
  - ``find_eigenvalues_v3`` solves its equations to convergence (residual <= 1e-12) instead of stopping
    where scipy's least squares does (~1e-7), so parameters differ from the reference's by up to ~2e-4.
Only D = 2..6 is supported, like the reference's gradient table (KeyError otherwise).
"""
from dataclasses import dataclass

import numpy as np
import torch

from .. import _device, _lib
from .mixture_model_utils import flatten_obs
from .complex_watson import normalize_observation  # noqa: F401  (complex_bingham.py:12-25, the same function)
from .utils import _ProbabilisticModel, force_hermitian  # noqa: F401  (complex_bingham.py:597)

__all__ = ['ComplexBingham', 'ComplexBinghamTrainer']

_MAX_INDEX = (1 << 29) - 1


def _check_dimension(D):
    """The reference's gradient table covers D = 2..6 (complex_bingham_utils.py:342-348)."""
    if not 2 <= D <= 6:
        raise KeyError(D)


def _status_error(what, K=None):
    """Decodes the status word of the Bingham entry points (include/pbb.h) into the reference's exception."""
    def on_error(s):
        kind, index = 4 - (s & 3), _MAX_INDEX - (s >> 2)
        where = f'problem {index}' if K is None else f'bin {index // K}, class {index % K}'
        if kind == 1:
            raise AssertionError(f'{what}: a scatter eigenvalue is negative or numerically zero ({where})')
        if kind == 2:
            raise ValueError(f'{what}: infeasible start of the parameter solve, a zero or negative scatter '
                             f'eigenvalue ({where})')
        raise AssertionError(f'{what}: non-finite scatter, parameters or normaliser ({where})')
    return on_error


def _as_device(x, dtype):
    if not _device.is_tensor(x):
        x = np.asarray(x)
    return _device.to_device(x, dtype)


@dataclass
class ComplexBingham(_ProbabilisticModel):
    covariance_eigenvectors: np.array = None  # (..., D, D), columns
    covariance_eigenvalues: np.array = None  # (..., D)

    def __post_init__(self):
        if self.covariance_eigenvectors is not None and not _device.is_tensor(self.covariance_eigenvectors):
            self.covariance_eigenvectors = np.array(self.covariance_eigenvectors)
        if not _device.is_tensor(self.covariance_eigenvalues):
            self.covariance_eigenvalues = np.array(self.covariance_eigenvalues)

    @property
    def covariance(self):
        """B = V diag(lambda) V^H (complex_bingham.py:37-45)."""
        like_numpy = not _device.is_tensor(self.covariance_eigenvectors)
        V = _as_device(self.covariance_eigenvectors, torch.complex128)
        lam = _as_device(self.covariance_eigenvalues, torch.float64)
        B = torch.einsum('...wx,...x,...zx->...wz', V, lam.to(V.dtype), V.conj())
        return _device.to_host(B, like_numpy)

    def pdf(self, y):
        return np.exp(self.log_pdf(y)) if not _device.is_tensor(y) else torch.exp(self.log_pdf(y))

    def log_pdf(self, y):
        """Re(y^H B y) - log c(lambda) for y (..., T, D), as given (complex_bingham.py:59-78)."""
        like_numpy = not _device.is_tensor(y)
        yd = _as_device(y, None)
        if not yd.is_complex():
            yd = yd.to(torch.complex128)
        V = _as_device(self.covariance_eigenvectors, torch.complex128)
        lam = _as_device(self.covariance_eigenvalues, torch.float64)
        D = lam.shape[-1]
        _check_dimension(D)
        lead = torch.broadcast_shapes(tuple(yd.shape[:-2]), tuple(V.shape[:-2]), tuple(lam.shape[:-1]))
        T = yd.shape[-2]
        M = int(np.prod(lead)) if lead else 1
        yd = yd.expand(*lead, T, D).reshape(M, T, D).contiguous()
        V = V.expand(*lead, D, D).reshape(M, D, D).contiguous()
        lam = lam.expand(*lead, D).reshape(M, D).contiguous()
        ld = self._log_norm_device(lam, 1e-8)
        out = _device.empty((M, T), torch.float64)
        _device.call('pbb_bingham_log_pdf', yd, _device.complex_dtype_code(yd), M, T, D, V, lam, ld, out)
        return _device.to_host(out.reshape(*lead, T), like_numpy)

    @staticmethod
    def _log_norm_device(lam, eps):
        D = lam.shape[-1]
        _check_dimension(D)
        n = lam.numel() // D
        out = _device.empty((n,), torch.float64)
        _device.call('pbb_bingham_log_norm', lam, n, D, float(eps), out)
        return out

    def log_norm(self, remove_duplicate_eigenvalues=True):
        return self._log_norm(remove_duplicate_eigenvalues, 1e-8)

    def norm(self, remove_duplicate_eigenvalues=True, eps=1e-8):
        """c(lambda) = 2 pi^D exp[lambda_1, ..., lambda_D] (complex_bingham.py:83-164).  With
        ``remove_duplicate_eigenvalues`` the sorted eigenvalues are first forced at least ``eps`` apart
        (:167-203); without it repeated eigenvalues give the exact limit."""
        ln = self._log_norm(remove_duplicate_eigenvalues, eps)
        return np.exp(ln) if not _device.is_tensor(ln) else torch.exp(ln)

    def _log_norm(self, remove_duplicate_eigenvalues, eps):
        like_numpy = not _device.is_tensor(self.covariance_eigenvalues)
        lam = _as_device(self.covariance_eigenvalues, torch.float64)
        out = self._log_norm_device(lam.contiguous(), eps if remove_duplicate_eigenvalues else 0.0)
        out = _device.to_host(out.reshape(lam.shape[:-1]), like_numpy)
        return out[()] if like_numpy else out


class ComplexBinghamTrainer:
    def __init__(self, dimension=None, max_concentration=np.inf, eignevalue_eps=1e-8):
        """``eignevalue_eps`` keeps the reference's spelling (complex_bingham.py:207-223)."""
        self.dimension = dimension
        assert max_concentration > 0, max_concentration
        self.max_concentration = max_concentration
        self.eignevalue_eps = eignevalue_eps

    @classmethod
    def find_eigenvalues_v3(cls, scatter_eigenvalues, eps=1e-8, max_concentration=np.inf):
        """Bingham parameters (largest 0) from scatter eigenvalues (..., D), batched over the leading dims
        (complex_bingham.py:304-425).  A zero or negative scatter eigenvalue raises ValueError."""
        like_numpy = not _device.is_tensor(scatter_eigenvalues)
        s = _as_device(scatter_eigenvalues, torch.float64)
        D = s.shape[-1]
        _check_dimension(D)
        assert max_concentration > 0, max_concentration
        n = s.numel() // D
        lam = _device.empty(tuple(s.shape), torch.float64)
        status = _device.empty((1,), torch.int32)
        _device.call('pbb_bingham_parameters', s, n, D, float(eps), float(max_concentration), lam, status)
        _device.check_status(status, _status_error('find_eigenvalues_v3'))
        return _device.to_host(lam, like_numpy)

    def fit(self, y, saliency=None) -> ComplexBingham:
        """complex_bingham.py:541-565: normalises y (..., N, D), then ``_fit``."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        assert yd.is_complex(), yd.dtype
        assert yd.shape[-1] > 1
        if saliency is not None:
            sal = _as_device(saliency, torch.float64)
            torch.broadcast_shapes(tuple(yd.shape[:-1]), tuple(sal.shape))
            saliency = sal
        if self.dimension is None:
            self.dimension = yd.shape[-1]
        else:
            assert self.dimension == yd.shape[-1], (
                'You initialized the trainer with a different dimension than '
                'you are using to fit a model. Use a new trainer, when you '
                'change the dimension.')
        model = self._fit(yd, saliency=saliency)
        if like_numpy:
            model = ComplexBingham(_device.to_host(model.covariance_eigenvectors, True),
                                   _device.to_host(model.covariance_eigenvalues, True))
        return model

    def _fit(self, y, saliency) -> ComplexBingham:
        """Scatter sum_n sal y y^H / sum_n sal, hermitian eigh, eigenvalue check and find_eigenvalues_v3
        (complex_bingham.py:567-594).  The device normalises y first, which leaves the unit-norm
        observations of fit() and of the mixture model unchanged."""
        like_numpy = not _device.is_tensor(y)
        yd = _device.to_device(y)
        independent, F, N, D = flatten_obs(yd)
        _check_dimension(D)
        if saliency is None:
            aff = torch.ones((F, 1, N), dtype=torch.float64, device=yd.device)
        else:
            aff = _as_device(saliency, torch.float64).expand(*independent, N).reshape(F, 1, N).contiguous()
        V, lam, _ = _cbmm_fit_device(yd, aff, None, 1, 1, _lib.WEIGHT_CONST, 0.0, self.eignevalue_eps,
                                     self.max_concentration, 'ComplexBinghamTrainer.fit')
        return ComplexBingham(
            covariance_eigenvectors=_device.to_host(V.reshape(*independent, D, D), like_numpy),
            covariance_eigenvalues=_device.to_host(lam.reshape(*independent, D), like_numpy))


def _cbmm_fit_device(yd, init, sal, K, iterations, weight_mode, affiliation_eps, eigenvalue_eps,
                     max_concentration, what):
    """One ``pbb_cbmm_fit`` call: (eigenvectors (F, K, D, D), eigenvalues (F, K, D), weight (F, K)) tensors."""
    independent, F, N, D = flatten_obs(yd)
    _check_dimension(D)
    code = _device.complex_dtype_code(yd)
    V = _device.empty((F, K, D, D), torch.complex128)
    lam = _device.empty((F, K, D), torch.float64)
    w = _device.empty((F, K), torch.float64)
    status = _device.empty((1,), torch.int32)
    lib = _lib.load()
    nbytes = lib.pbb_cbmm_workspace_bytes(F, N, D, K)
    ws = _device.workspace(nbytes)
    _device.call('pbb_cbmm_fit', yd, code, F, N, D, K, init, sal, int(iterations), weight_mode, float(affiliation_eps),
                 float(eigenvalue_eps), float(max_concentration), V, lam, w, ws, nbytes, status)
    _device.check_status(status, _status_error(what, K))
    return V, lam, w
