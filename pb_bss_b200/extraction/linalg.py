"""Batched small-matrix linear algebra on the device (thin ctypes wrappers)."""
import numpy as np
import torch

from .. import _device


def eigh(a):
    """Batched Hermitian eigendecomposition (..., D, D) -> (w (..., D) ascending,
    v (..., D, D) with eigenvectors as columns), like ``np.linalg.eigh``
    (complex_angular_central_gaussian.py:95, pb_bss/utils.py:154)."""
    like_numpy = not _device.is_tensor(a)
    ad = _device.to_device(a, torch.complex128)
    *lead, D, D2 = ad.shape
    assert D == D2, ad.shape
    n = int(np.prod(lead)) if lead else 1
    w = _device.empty((n, D), torch.float64)
    v = _device.empty((n, D, D), torch.complex128)
    status = torch.zeros(1, dtype=torch.int32, device=ad.device)
    _device.call('pbb_heig_batched', ad, n, D, w, v, status)
    def on_error(s):
        raise np.linalg.LinAlgError(f'eigh: non-finite input or no convergence in matrix {s - 1}')
    _device.check_status(status, on_error)
    return (_device.to_host(w.reshape(*lead, D), like_numpy),
            _device.to_host(v.reshape(*lead, D, D), like_numpy))


def stable_solve(A, B, hermitize=False):
    """``pb_bss.math.solve.stable_solve`` (math/solve.py:20-114): np.linalg.solve over the independent dimensions;
    an exactly singular matrix gets its minimum-norm least-squares solution (np.linalg.lstsq) instead of a
    LinAlgError.  A (..., D, D), B (..., D, R) -> X (..., D, R).  The reference falls back matrix by matrix on the
    host; here the fallback lives in the same kernel (linalg_kernels.cuh: solve_kernel)."""
    like_numpy = not _device.is_tensor(A)
    ad = _device.to_device(A, torch.complex128)
    bd = _device.to_device(B, torch.complex128)
    assert ad.shape[:-2] == bd.shape[:-2], (ad.shape, bd.shape)
    assert ad.shape[-1] == bd.shape[-2], (ad.shape, bd.shape)
    *lead, D, _ = ad.shape
    R = bd.shape[-1]
    n = int(np.prod(lead)) if lead else 1
    x = _device.empty((n, D, R), torch.complex128)
    status = torch.zeros(1, dtype=torch.int32, device=ad.device)
    _device.call('pbb_solve_batched', ad.reshape(n, D, D).contiguous(), bd.reshape(n, D, R).contiguous(), n, D, R,
                 1 if hermitize else 0, x, status)
    def on_error(s):
        raise np.linalg.LinAlgError(f'stable_solve: singular matrix {s - 1} (D > 40: no lstsq fallback)')
    _device.check_status(status, on_error)
    return _device.to_host(x.reshape(*lead, D, R), like_numpy)


solve = stable_solve
