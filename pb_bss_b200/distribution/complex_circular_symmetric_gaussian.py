"""Complex circular-symmetric Gaussian -- ``ComplexCircularSymmetricGaussian`` and its trainer with the names,
arguments, defaults and error types of pb_bss/distribution/complex_circular_symmetric_gaussian.py, executed by the
kernels behind ``pbb_ccsg_log_pdf``, ``pbb_ccsg_sample`` and ``pbb_ccsg_fit`` (include/pbb.h).

NumPy in gives NumPy out; CUDA tensors in give CUDA tensors out.  The random draws of ``sample`` stay on the host:
``np.random.normal`` from NumPy's global stream, real parts first, in the reference's call order, so a seeded run
reproduces the reference's draws and leaves the stream where the reference leaves it.  The device does the
Cholesky factorisation and the transform.

Differences from the reference:
  - ``sample`` raises ValueError for a ``size`` with two or more dims; the reference's ``(L @ x.T).T`` raises there
    too, or, when a size happens to equal D, returns samples mixed across axes.  The check comes before the draws.
  - D is limited to 64 (``log_pdf``, ``sample``) and to 34 (the trainer).
"""
from dataclasses import dataclass

import numpy as np
import torch

from .. import _device, _lib
from .utils import _ProbabilisticModel

__all__ = ['ComplexCircularSymmetricGaussian', 'ComplexCircularSymmetricGaussianTrainer']


def _as_device(x, dtype=None):
    if not _device.is_tensor(x):
        x = np.asarray(x)
    return _device.to_device(x, dtype)


def _frames(yd, lead):
    """y (..., N, D) -> (y on the device as (M, N, D) or, when every model shares it, (N, D); the model stride)."""
    N, D = yd.shape[-2:]
    if int(np.prod(yd.shape[:-2])) == 1:
        return yd.reshape(N, D).contiguous(), 0
    M = int(np.prod(lead))
    return yd.expand(*lead, N, D).reshape(M, N, D).contiguous(), N * D


def _linalg_error(message):
    def on_error(s):
        raise np.linalg.LinAlgError(f'{message} (matrix {s - 1})')
    return on_error


def _draw(size, D):
    """The reference's draws for ``size`` samples of dimension D: real parts, then imaginary parts
    (complex_circular_symmetric_gaussian.py:66-67).  ``(*size, D)`` raises TypeError for a plain int, as there."""
    shape = (*size, D)
    if len(shape) > 2:
        raise ValueError(f'size must have at most one dim, got {tuple(size)}: the reference transforms the samples '
                         f'with (L @ x.T).T, which mixes the axes of a larger size')
    return np.random.normal(size=shape), np.random.normal(size=shape)


def sample_classes(a, eigenvalues, draws, unit_norm, like_numpy, dest=None):
    """One ``pbb_ccsg_sample`` launch for C classes.

    a: (C, D, D) covariances, or eigenvectors when ``eigenvalues`` (C, D) is given (then the covariance is
    V diag(lambda) V^H); draws: per class in order, the pair (real, imag) of (n_c, D) standard normals; dest: (S,)
    int64 output row of every sample, or None for the concatenation order.  Returns (S, D) complex128.
    """
    a = _as_device(a, torch.complex128)
    C, D = a.shape[0], a.shape[-1]
    counts = [re.shape[0] for re, _ in draws]
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    S = int(offsets[-1])
    lam = None if eigenvalues is None else _as_device(eigenvalues, torch.float64).contiguous()
    normals = None
    if S:
        normals = _as_device(np.concatenate([np.concatenate([re.reshape(-1, D) for re, _ in draws]).ravel(),
                                             np.concatenate([im.reshape(-1, D) for _, im in draws]).ravel()]),
                             torch.float64)
    off = _as_device(offsets)
    dst = None if dest is None else _as_device(np.asarray(dest, dtype=np.int64))
    out = _device.empty((S, D), torch.complex128)
    status = _device.empty((1,), torch.int32)
    lib = _lib.load()
    nbytes = lib.pbb_ccsg_workspace_bytes(C, D)
    ws = _device.workspace(nbytes)
    _device.call('pbb_ccsg_sample', a.contiguous(), lam, C, D, normals, off, dst, S, int(bool(unit_norm)), out, ws,
                 nbytes, status)
    _device.check_status(status, _linalg_error('Matrix is not positive definite'))
    return _device.to_host(out, like_numpy)


def sample(size, a, eigenvalues, unit_norm):
    """``size`` samples of one class (see ``sample_classes``), shape (*size, D)."""
    like_numpy = not _device.is_tensor(a)
    if a.ndim > 2:
        # TODO of the reference: what is the correct generalization?
        raise NotImplementedError('Not quite clear how the correct broadcasting would look like.')
    D = a.shape[-1]
    re, im = _draw(size, D)
    x = sample_classes(a[None], None if eigenvalues is None else eigenvalues[None], [(re, im)], unit_norm,
                       like_numpy)
    return x.reshape(re.shape)


@dataclass
class ComplexCircularSymmetricGaussian(_ProbabilisticModel):
    covariance: np.array  # (..., D, D)

    def log_pdf(self, y):
        """-D log pi - log|det S| - Re(y^H S^-1 y) for y (..., N, D), complex or real; the model's leading dims
        broadcast against y's (complex_circular_symmetric_gaussian.py:26-48).  S may be any invertible matrix
        (LU with partial pivoting, like the reference's solve / slogdet); a singular S raises LinAlgError."""
        like_numpy = not _device.is_tensor(y)
        yd = _as_device(y)
        if not yd.is_complex():
            yd = yd.to(torch.complex128)
        S = _as_device(self.covariance, torch.complex128)
        D = S.shape[-1]
        assert yd.shape[-1] == D, (yd.shape, S.shape)
        N = yd.shape[-2]
        lead = torch.broadcast_shapes(tuple(yd.shape[:-2]), tuple(S.shape[:-2]))
        M = int(np.prod(lead))
        out = _device.empty((M, N), torch.float64)
        if M and N:
            frames, stride = _frames(yd, lead)
            S = S.expand(*lead, D, D).reshape(M, D, D).contiguous()
            status = _device.empty((1,), torch.int32)
            lib = _lib.load()
            nbytes = lib.pbb_ccsg_workspace_bytes(M, D)
            ws = _device.workspace(nbytes)
            _device.call('pbb_ccsg_log_pdf', frames, _device.complex_dtype_code(frames), stride, M, N, D, S, out, ws,
                         nbytes, status)
            _device.check_status(status, _linalg_error('Singular matrix'))
        return _device.to_host(out.reshape(*lead, N), like_numpy)

    def sample(self, size):
        """Samples of shape (*size, D) (complex_circular_symmetric_gaussian.py:50-72): a covariance with more than
        two dims raises NotImplementedError, a plain int ``size`` TypeError, a ``size`` with two or more dims
        ValueError."""
        return sample(size, self.covariance, None, unit_norm=False)


class ComplexCircularSymmetricGaussianTrainer:
    def fit(self, y, saliency=None, covariance_type='full'):
        """Maximum-likelihood covariance of y (..., N, D) (complex_circular_symmetric_gaussian.py:76-92)."""
        like_numpy = not _device.is_tensor(y)
        yd = _as_device(y)
        assert yd.is_complex(), yd.dtype
        if saliency is not None:
            saliency = _as_device(saliency, torch.float64)
            try:
                torch.broadcast_shapes(tuple(yd.shape[:-1]), tuple(saliency.shape))
            except RuntimeError:
                raise AssertionError((tuple(yd.shape), tuple(saliency.shape))) from None
        model = self._fit(yd, saliency=saliency, covariance_type=covariance_type)
        return ComplexCircularSymmetricGaussian(covariance=_device.to_host(model.covariance, like_numpy))

    def _fit(self, y, saliency, covariance_type):
        """sum_n s y y^H / (N, or max(sum_n s, tiny of y's dtype)), without hermitisation or normalisation of y
        (:94-116).  Without frames that is 0 / 0 = NaN, or 0 with a saliency, as in the reference."""
        if covariance_type != 'full':
            raise ValueError(f"Unknown covariance type '{covariance_type}'.")
        like_numpy = not _device.is_tensor(y)
        yd = _as_device(y)
        *_, N, D = yd.shape
        lead = tuple(yd.shape[:-2])
        if saliency is not None:
            saliency = _as_device(saliency, torch.float64)
            lead = torch.broadcast_shapes(lead, tuple(saliency.shape[:-1]))
        F = int(np.prod(lead))
        cov = _device.empty((F, D, D), torch.complex128)
        if F and N == 0:
            cov.fill_(complex('nan+nanj') if saliency is None else 0)
        elif F:
            # the PSD accumulation reads the observation as (F, D, N)
            obs = yd.expand(*lead, N, D).reshape(F, N, D).transpose(-1, -2).contiguous()
            sal = None if saliency is None else saliency.expand(*lead, N).reshape(F, N).contiguous()
            lib = _lib.load()
            nbytes = lib.pbb_psd_workspace_bytes(F, N, D, 1)
            ws = _device.workspace(nbytes)
            _device.call('pbb_ccsg_fit', obs, _device.complex_dtype_code(obs), F, D, N, sal,
                         float(np.finfo(np.float32 if yd.dtype == torch.complex64 else np.float64).tiny), cov, ws,
                         nbytes)
        return ComplexCircularSymmetricGaussian(covariance=_device.to_host(cov.reshape(*lead, D, D), like_numpy))
