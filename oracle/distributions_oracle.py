"""NumPy restatement of the single distributions of pb_bss.distribution and the inputs of their fixture cases.

The restatement follows the formulas, not the reference's code: the complex angular central Gaussian (Tyler 1987,
Ito et al. 2016), the complex Watson distribution with Mardia's normalisers (Mardia & Dryden 1999, Eq. 3 and 4), the
complex circular-symmetric Gaussian (Gallager), and the samplers built on it.  Where the reference fixes an order of
operations that changes the float64 result (normalisation by max(., tiny), the clamps, NumPy's complex division by a
real scalar as a multiplication by its reciprocal), the restatement keeps that order.  Used by
oracle/make_golden_distributions.py and tests/test_distributions_oracle.py.

Every case input is regenerated from a seed by ``case_input``; only outputs are stored in the fixture.
"""
import math

import numpy as np

TINY = np.finfo(np.float64).tiny
KAPPAS = np.array([0.0, 1e-3, None, 19.9, 20.1, 100.0, 500.0, 800.0], dtype=object)  # None: 1 / D
NORM_DIMS = (2, 3, 4, 5, 6, 7, 8)
FIT_DIMS = (2, 3, 4, 5, 6, 7, 8)
VARIANTS = ('1f1', 'low', 'medium', 'high', 'tran_vu')


def kappas(D):
    return np.array([1.0 / D if k is None else k for k in KAPPAS], dtype=np.float64)


# ---- inputs -------------------------------------------------------------------------------------------------------
def _crandn(rng, *shape):
    return rng.normal(size=shape) + 1j * rng.normal(size=shape)


def hermitian_pd(rng, *lead, D, cond=10.0):
    """Hermitian positive definite matrices (*lead, D, D) with eigenvalues spread over [1, cond]."""
    q, _ = np.linalg.qr(_crandn(rng, *lead, D, D))
    lam = np.exp(rng.uniform(0.0, np.log(cond), size=(*lead, D)))
    return np.einsum('...dx,...x,...ex->...de', q, lam, q.conj())


def directional(rng, N, D, lead=()):
    """Observations (*lead, N, D) around a few directions, not normalised: a well-conditioned fit."""
    base = _crandn(rng, *lead, 1, D) * np.array([3.0] + [1.0] * (D - 1))
    return base + 0.5 * _crandn(rng, *lead, N, D)


def case_input(name, D=None):
    """The inputs of a fixture case, regenerated from its seed."""
    rng = np.random.default_rng({'cov': 1, 'logpdf': 2, 'fit': 3, 'batch': 4, 'step': 5, 'watson': 6, 'wfit': 7,
                                 'ccsg': 8, 'ccsg_fit': 9}[name] * 1000 + (D or 0))
    if name == 'cov':
        return hermitian_pd(rng, 3, D=5, cond=1e4)
    if name == 'logpdf':
        cov = hermitian_pd(rng, 3, 2, D=4)
        y = directional(rng, 50, 4, lead=(3, 1))
        y[0, 0, 7] = 0.0  # a zero frame: q = tiny
        return cov, y
    if name == 'fit':
        return directional(rng, 200, D)
    if name == 'batch':
        return directional(rng, 120, 4, lead=(2, 3))
    if name == 'step':
        y = directional(rng, 60, 4)
        z = y / np.linalg.norm(y, axis=-1, keepdims=True)
        q = rng.uniform(0.5, 4.0, size=(2, 60))
        sal = rng.uniform(0.0, 1.0, size=(2, 60))
        return np.ascontiguousarray(z.T)[None], q, sal
    if name == 'watson':
        mode = _crandn(rng, 3, 4)
        mode /= np.linalg.norm(mode, axis=-1, keepdims=True)
        kappa = np.array([0.5, 7.0, 40.0])
        y = 0.7 * _crandn(rng, 3, 40, 4)  # not unit norm: log_pdf uses y as given
        return mode, kappa, y
    if name == 'wfit':
        y = directional(rng, 150, D)
        sal = rng.uniform(0.0, 1.0, size=150)
        sal[::7] = 0.0
        return y, sal
    if name == 'ccsg':
        D = 4
        herm = hermitian_pd(rng, D=D)
        nonherm = _crandn(rng, D, D) + 3.0 * np.eye(D)
        classes = hermitian_pd(rng, 3, D=D)
        y = _crandn(rng, 30, D)
        yreal = rng.normal(size=(30, D))
        return herm, nonherm, classes, y, yreal
    if name == 'ccsg_fit':
        y = _crandn(rng, 2, 80, 3)
        sal = rng.uniform(0.0, 1.0, size=(2, 80))
        sal[:, ::5] = 0.0
        return y, sal
    raise KeyError(name)


SAMPLE_SEED = 20261016
SAMPLE_COV_SEED = 11


def sample_inputs():
    rng = np.random.default_rng(SAMPLE_COV_SEED)
    return hermitian_pd(rng, D=3), hermitian_pd(rng, 3, D=3), np.array([0.5, 0.0, 0.5])


# ---- complex angular central Gaussian -----------------------------------------------------------------------------
def unit_rows(y):
    n = np.linalg.norm(y, axis=-1, keepdims=True)
    return np.where(n > 0, y / np.maximum(n, np.finfo(y.dtype).tiny), 0)


def cacg_from_covariance(cov, floor=0.0, norm='eigenvalue'):
    """Eigenvalues (ascending) and eigenvectors of the (optionally trace-normalised) covariance, the eigenvalues
    scaled to a largest of 1 and floored ('eigenvalue'), or floored relative to the largest (other norms)."""
    cov = np.array(cov, dtype=np.complex128)
    if norm == 'trace':
        tr = np.einsum('...dd->...', cov).real
        cov = cov * (1.0 / np.maximum(tr, TINY))[..., None, None]
    lam, V = np.linalg.eigh(cov)
    top = lam.max(axis=-1, keepdims=True)
    if norm == 'eigenvalue':
        lam = np.maximum(lam / np.maximum(top, TINY), floor)
    else:
        lam = np.maximum(lam, top * floor)
    return V, lam


def covariance(V, lam):
    return np.einsum('...dx,...x,...ex->...de', V, lam, V.conj())


def cacg_log_pdf(z, V, lam, tiny=TINY):
    """(log_pdf, q) of unit-norm z (..., D, N): q = max(|z^H V diag(1/lam) V^H z|, tiny), -D log q - log det."""
    D = z.shape[-2]
    w = np.einsum('...de,...dn->...en', V.conj(), z)  # V^H z
    q = np.maximum(np.abs(np.einsum('...en,...e->...n', np.abs(w) ** 2, 1.0 / lam)), tiny)
    return -D * np.log(q) - np.sum(np.log(lam), axis=-1)[..., None], q


def cacg_step(z, q, saliency=None, floor=1e-10, norm='eigenvalue'):
    """One fixed-point step: D sum_n s z z^H / q / (N or sum s), then from_covariance."""
    D = z.shape[-2]
    N = q.shape[-1]
    q = np.maximum(q, 10 * TINY)
    s = 1.0 if saliency is None else saliency
    den = N if saliency is None else np.sum(saliency, axis=-1)[..., None, None]
    cov = D * np.einsum('...dn,...en,...n->...de', z, z.conj(), s / q) / np.maximum(den, TINY)
    return cacg_from_covariance(cov, floor, norm)


def cacg_fit(y, iterations=10, floor=1e-10, norm='eigenvalue'):
    z = np.swapaxes(unit_rows(y), -1, -2)
    q = np.ones(z.shape[:-2] + z.shape[-1:])
    for _ in range(iterations):
        V, lam = cacg_step(z, q, None, floor, norm)
        _, q = cacg_log_pdf(z, V, lam)
    return V, lam


# ---- complex Watson -----------------------------------------------------------------------------------------------
def _log_base(D):
    return np.log(2.0) + D * np.log(np.pi)


def cw_log_norm(variant, kappa, D):
    """The five normalisers, restated with np.asarray(kappa, float) (np.asfarray is gone in NumPy 2)."""
    k = np.asarray(kappa, dtype=float)
    shape = k.shape
    k = k.ravel()
    low = (_log_base(D) - np.log(math.factorial(D - 1))
           + np.log(1 + np.sum(np.cumprod(k[:, None] / np.arange(D, D + 20)[None, :], -1), -1)))

    def closed(k, series=True):
        with np.errstate(divide='ignore', invalid='ignore'):
            v = _log_base(D) + (1.0 - D) * np.log(k) + k
            if not series:
                return v
            r = np.arange(D - 1)
            terms = k[:, None] ** r * np.exp(-k[:, None]) / np.array([math.factorial(i) for i in r])
            return v + np.log(1.0 - np.sum(terms, -1))

    if variant == 'low':
        out = low
    elif variant == 'medium':
        out = closed(np.where(k < 1e-2, 1e-2, k))
    elif variant == 'high':
        out = closed(k, series=False)
    elif variant == 'tran_vu':
        out = np.where(k >= 1.0 / D, closed(k), low)
    elif variant == '1f1':
        # 1F1(1; D; k) = (D-1)! e^k k^(1-D) (1 - e^-k sum_{r<D-1} k^r / r!): the closed form, with the Taylor series
        # where it cancels
        out = np.where(k < 20.0, _series_1f1(k, D), closed(k))
    else:
        raise KeyError(variant)
    return out.reshape(shape)


def _series_1f1(k, D):
    s = np.ones_like(k)
    t = np.ones_like(k)
    for n in range(1, 400):
        t = t * k / (D + n - 1)
        s = s + t
    return _log_base(D) - np.log(math.factorial(D - 1)) + np.log(s)


def cw_log_norm_spread(variant, kappa, D):
    """Absolute float64 spread of a normaliser: the correction log(1 - S) of the medium formula cancels when
    S = e^-k sum_{r<D-1} k^r / r! is close to 1, and a rounding of S by a few ulp moves it by ~ eps S / (1 - S)."""
    k = np.asarray(kappa, dtype=float)
    if variant == 'medium':
        k = np.where(k < 1e-2, 1e-2, k)
    if variant not in ('medium', 'tran_vu'):
        return np.zeros_like(k)
    r = np.arange(D - 1)
    S = np.sum(k[..., None] ** r * np.exp(-k[..., None]) / np.array([math.factorial(i) for i in r]), -1)
    with np.errstate(divide='ignore', invalid='ignore'):
        spread = 8 * D * np.finfo(float).eps * S / np.abs(1.0 - S)
    if variant == 'tran_vu':
        spread = np.where(k >= 1.0 / D, spread, 0.0)
    return np.where(np.isfinite(spread), spread, np.inf)


def cw_log_pdf(y, mode, kappa):
    d = np.einsum('...nd,...d->...n', y, mode.conj())
    return (d.real ** 2 + d.imag ** 2) * kappa[..., None] - cw_log_norm('1f1', kappa, mode.shape[-1])[..., None]


def cw_scatter(y, saliency=None):
    """The saliency-weighted scatter sum s y y^H / sum s of y (..., N, D) as given."""
    s = np.ones(y.shape[:-1]) if saliency is None else saliency
    return np.einsum('...n,...nd,...ne->...de', s, y, y.conj()) / np.sum(s, axis=-1)[..., None, None]


# ---- complex circular-symmetric Gaussian --------------------------------------------------------------------------
def ccsg_log_pdf(y, cov):
    D = cov.shape[-1]
    _, logdet = np.linalg.slogdet(cov)
    x = np.linalg.solve(cov[..., None, :, :], y[..., :, None])[..., 0]
    return -D * np.log(np.pi) - logdet[..., None] - np.einsum('...nd,...nd->...n', y.conj(), x).real


def ccsg_fit(y, saliency=None):
    if saliency is None:
        return np.einsum('...nd,...ne->...de', y, y.conj()) * (1.0 / y.shape[-2])
    den = np.maximum(np.sum(saliency, axis=-1), TINY)
    return np.einsum('...n,...nd,...ne->...de', saliency, y, y.conj()) * (1.0 / den)[..., None, None]


def ccsg_transform(re, im, cov, unit_norm):
    """L (re + i im) / sqrt 2 per row, optionally scaled to unit norm; re, im (n, D) standard normals."""
    x = (re + 1j * im) * (1.0 / np.sqrt(2))
    y = x @ np.linalg.cholesky(cov).T
    if unit_norm:
        y = y * (1.0 / np.linalg.norm(y, axis=-1, keepdims=True))
    return y


def ccsg_sample(size, cov, unit_norm=False):
    D = cov.shape[-1]
    re = np.random.normal(size=(*size, D))
    im = np.random.normal(size=(*size, D))
    return ccsg_transform(re.reshape(-1, D), im.reshape(-1, D), cov, unit_norm).reshape(re.shape)


def sample_cacgmm(size, weight, cov):
    K, D = weight.shape[0], cov.shape[-1]
    labels = np.random.choice(range(K), size=size, p=weight)
    x = np.zeros((size, D), dtype=np.complex128)
    for k in range(K):
        V, lam = cacg_from_covariance(cov[k])
        x[labels == k] = ccsg_sample((int(np.sum(labels == k)),), covariance(V, lam), unit_norm=True)
    return x, labels
