"""von Mises-Fisher distribution over real embedding vectors (pb_bss/distribution/von_mises_fisher.py:31-144): tied
over all (bin, frame) observations, as the integrated model vmfcacgmm.py uses it (``log_pdf_fkt``), and with any
number of independent leading dims (``log_pdf``, ``VonMisesFisherTrainer``, the VMFMM).  The normaliser (scipy's
exponentially scaled Bessel function on one scalar per model) and the final K x E parameter math stay on the host;
the observations are only touched by the device kernels."""
import math
from dataclasses import dataclass

import numpy as np
import torch
from scipy.special import ive

from .. import _device, _lib
from .gaussian import _dev, _is_real, _np, batched_layout, check_embedding_dim
from .utils import _ProbabilisticModel


@dataclass
class VonMisesFisher(_ProbabilisticModel):
    mean: np.array = None           # (K, E)
    concentration: np.array = None  # (K,)

    def log_norm(self):
        """von_mises_fisher.py:36-46."""
        D = self.mean.shape[-1]
        kappa = np.asarray(self.concentration)
        return ((D / 2) * np.log(2 * np.pi) + np.log(ive(D / 2 - 1, kappa))
                + (np.abs(kappa) - (D / 2 - 1) * np.log(kappa)))

    def norm(self):
        """exp(log_norm) (von_mises_fisher.py:62-63; the reference applies np.exp to the bound method and raises
        TypeError, this evaluates the normaliser it means)."""
        return np.exp(self.log_norm())

    def sample(self, size):
        """von_mises_fisher.py:85-91."""
        raise NotImplementedError(
            'A sampling method is not yet implemented. '
            'Feel free to make a pull request.')

    def pdf(self, y):
        """exp(log_pdf(y)) (von_mises_fisher.py:82-90), in the same device pass as the log-pdf (pbb_vmf_pdf)."""
        return self.log_pdf(y, _exp=True)

    def log_pdf(self, y, _exp=False):
        """y (..., N, E) (any norm: normalised inside) -> (..., N), broadcast against the model dims
        (von_mises_fisher.py:65-79)."""
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        E = yd.shape[-1]
        check_embedding_dim(E)
        mean = _np(self.mean)
        kappa = _np(self.concentration)
        x, B, K, L = batched_layout(yd, mean.shape[:-1])
        log_norm = VonMisesFisher(mean=mean, concentration=kappa).log_norm()
        m = _dev(np.broadcast_to(mean, L + (E,)).reshape(B, K, E))
        kap = _dev(np.broadcast_to(kappa, L).reshape(B, K))
        ln = _dev(np.broadcast_to(log_norm, L).reshape(B, K))
        out = vmf_log_pdf_bkn(x, m, kap, ln, exp=_exp)
        return _device.to_host(out.reshape(L + (yd.shape[-2],)), like_numpy)

    def log_pdf_fkt(self, embedding):
        """embedding (F, T, E) CUDA tensor (any norm: normalised inside, von_mises_fisher.py:75-77) -> (F, K, T)."""
        F, T, E = embedding.shape
        K = self.mean.shape[0]
        mean = _device.to_device(np.ascontiguousarray(self.mean), torch.float64)
        kap = _device.to_device(np.ascontiguousarray(np.repeat(np.asarray(self.concentration)[:, None], E, axis=1)),
                                torch.float64)
        ln = _device.to_device(np.ascontiguousarray(self.log_norm()), torch.float64)
        out = _device.empty((F, K, T), torch.float64)
        _device.call('pbb_gaussian_log_pdf', embedding, mean, kap, ln, F, T, E, K, 2, out)
        return out


def vmf_fit_fkt(embedding, weight_fkt, min_concentration, max_concentration):
    """VonMisesFisherTrainer._fit (von_mises_fisher.py:122-144) over the F*T embeddings with weights (F, K, T): the
    weighted resultant comes from the first pass of pbb_gaussian_fit (sum w x, sum w), the K x E rest is host math."""
    F, T, E = embedding.shape
    K = weight_fkt.shape[1]
    mean = _device.empty((K, E), torch.float64)
    cov = _device.empty((K,), torch.float64)
    lib = _lib.load()
    scratch = _device.empty((int(lib.pbb_gaussian_fit_scratch_doubles(F, E, K)),), torch.float64)
    _device.call('pbb_gaussian_fit', embedding, weight_fkt, F, T, E, K, 1, mean, cov, scratch)
    total = scratch[F * K * (E + 1):F * K * (E + 1) + K].cpu().numpy()        # sum of the weights per class
    r = mean.cpu().numpy() * total[:, None]                                   # Banerjee2005vMF eq. 2.4
    norm = np.linalg.norm(r, axis=-1)
    direction = r / np.maximum(norm, np.finfo(np.float64).tiny)[..., None]
    r_bar = norm / total                                                      # eq. 2.5
    concentration = (r_bar * E - r_bar ** 3) / (1 - r_bar ** 2)               # eq. 4.4
    concentration = np.clip(concentration, min_concentration, max_concentration)
    return VonMisesFisher(mean=direction, concentration=concentration)


def vmf_log_pdf_bkn(x, mean, concentration, log_norm, exp=False):
    """x (B, N, E), mean (B, K, E), concentration / log_norm (B, K) device -> (B, K, N); exp: the pdf."""
    B, N, E = x.shape
    K = mean.shape[1]
    out = _device.empty((B, K, N), torch.float64)
    name = 'pbb_vmf_pdf' if exp else 'pbb_vmf_log_pdf'
    _device.call(name, x, mean, concentration, log_norm, B, N, E, K, out)
    return out


def vmf_fit_bkn(x, weight, min_concentration, max_concentration):
    """VonMisesFisherTrainer._fit (von_mises_fisher.py:122-144) of x (B, N, E) (normalised by the kernel) with weights
    (B, K, N) device -> host mean (B, K, E), concentration (B, K)."""
    B, N, E = x.shape
    K = weight.shape[1]
    check_embedding_dim(E)
    lib = _lib.load()
    r = _device.empty((B, K, E), torch.float64)
    total = _device.empty((B, K), torch.float64)
    scratch = _device.empty((int(lib.pbb_gaussian_full_fit_scratch_doubles(B, N, E, K)),), torch.float64)
    _device.call('pbb_vmf_resultant', x, weight, B, N, E, K, r, total, scratch)
    r, total = r.cpu().numpy(), total.cpu().numpy()
    norm = np.linalg.norm(r, axis=-1)                                                 # Banerjee2005vMF eq. 2.4
    mean = r / np.maximum(norm, np.finfo(np.float64).tiny)[..., None]
    r_bar = norm / total                                                              # eq. 2.5
    concentration = (r_bar * E - r_bar ** 3) / (1 - r_bar ** 2)                       # eq. 4.4
    concentration = np.clip(concentration, min_concentration, max_concentration)
    return mean, concentration


class VonMisesFisherTrainer:
    def fit(self, y, saliency=None, min_concentration=1e-10, max_concentration=500) -> VonMisesFisher:
        """von_mises_fisher.py:93-120: y (..., N, E), saliency (..., N) or None."""
        assert _is_real(y), y.dtype
        if saliency is not None:
            ys, ss = tuple(y.shape[:-1]), tuple(saliency.shape)
            assert all(len({a, b} | {1}) <= 2 for a, b in zip(ys[::-1], ss[::-1])), (y.shape, saliency.shape)
        like_numpy = not _device.is_tensor(y)
        yd = _dev(y)
        N, E = yd.shape[-2:]
        sal = None if saliency is None else _dev(saliency)
        lead = tuple(yd.shape[:-2]) if sal is None else tuple(np.broadcast_shapes(yd.shape[:-2], sal.shape[:-1]))
        B = math.prod(lead)
        x = yd.expand(lead + (N, E)).reshape(B, N, E).contiguous()
        w = (torch.ones((B, 1, N), dtype=torch.float64, device=x.device) if sal is None
             else sal.expand(lead + (N,)).reshape(B, 1, N).contiguous())
        mean, concentration = vmf_fit_bkn(x, w, min_concentration, max_concentration)
        mean, concentration = mean.reshape(lead + (E,)), concentration.reshape(lead)
        if not like_numpy:
            mean, concentration = _dev(mean), _dev(concentration)
        return VonMisesFisher(mean=mean, concentration=concentration)
