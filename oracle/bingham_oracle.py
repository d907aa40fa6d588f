"""NumPy restatement of the complex Bingham mixture model (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows pb_bss/distribution/complex_bingham.py and cbmm.py line by line, with the two numerical choices the
device makes (include/pbb.h): the normaliser and its derivatives are divided differences of exp (entries of exp()
of the bidiagonal Opitz matrix, scaling and squaring), and find_eigenvalues_v3's equations are solved to
convergence by projected Gauss-Newton in the reference's difference coordinates, from the reference's start.
"""
import numpy as np

from .pb_bss_oracle import estimate_mixture_weight, log_pdf_to_affiliation, normalize_observation_cw

NORM_EPS = 1e-8     # norm()'s default eps, used by log_pdf (complex_bingham.py:83)
UPPER = -1e-8       # upper bound of the differences (complex_bingham.py:404)
ZERO = 1e-12        # scatter eigenvalue <= ZERO * largest: numerically zero
TOL = 1e-12
MAX_STEPS, MAX_HALVINGS, TAYLOR = 100, 40, 24


def dd_exp(x):
    """exp() of the upper bidiagonal matrix with diagonal x and unit superdiagonal: E[i, j] = exp[x_i..x_j]."""
    x = np.asarray(x, dtype=np.float64)
    N = len(x)
    xm = np.max(np.abs(x))
    s = int(np.frexp(xm)[1]) + 1 if xm > 0.5 else 0   # xm / 2^s <= 1/2
    h = 2.0 ** -s
    A = np.diag(x * h) + np.diag(np.full(N - 1, h), 1)
    E = np.eye(N)
    for k in range(TAYLOR, 0, -1):
        E = np.eye(N) + (A @ E) / k
    for _ in range(s):
        E = E @ E
    return E


def gap_rule(v, eps):
    """ComplexBingham._remove_duplicate_eigenvalues (complex_bingham.py:167-203): (inverse permutation, sorted
    values with neighbours at least eps apart)."""
    v = np.array(v, dtype=np.float64)
    perm = np.argsort(v, axis=-1, kind='stable')
    v = np.take_along_axis(v, perm, axis=-1)
    diff = np.maximum(np.diff(v, axis=-1), eps)
    v[..., 1:] = v[..., :1] + np.cumsum(diff, axis=-1)
    inv = np.argsort(perm, axis=-1, kind='stable')
    return inv, v


def log_norm(lam, eps=NORM_EPS):
    """log c(lambda) = log(2 pi^D exp[lambda]) after the gap rule (complex_bingham.py:80-164); eps <= 0: none."""
    lam = np.asarray(lam, dtype=np.float64)
    out = np.empty(lam.shape[:-1])
    for idx in np.ndindex(out.shape):
        v = np.sort(lam[idx], kind='stable')
        if eps > 0:
            v = gap_rule(v, eps)[1]
        top = v[-1]
        D = len(v)
        out[idx] = np.log(2) + D * np.log(np.pi) + top + np.log(dd_exp(v - top)[0, -1])
    return out


def derivatives(lam):
    """grad log c and its Hessian at lam (complex_bingham.py:552-564 differentiate the same c)."""
    D = len(lam)
    g = np.empty(D)
    H = np.empty((D, D))
    c0 = dd_exp(lam)[0, -1]
    for k in range(D):
        for l in range(k, D):
            E = dd_exp(np.concatenate([lam, [lam[k], lam[l]]]))
            if k == l:
                g[k] = E[0, D] / c0
            H[k, l] = (2.0 if k == l else 1.0) * E[0, D + 1] / c0
    for k in range(D):
        for l in range(k, D):
            H[k, l] -= g[k] * g[l]
            H[l, k] = H[k, l]
    return g, H


def _lambda_from_diff(x):
    # np.cumsum(np.array([*x, 0])[::-1])[::-1] (complex_bingham.py:411)
    return np.cumsum(np.array([*x, 0.0])[::-1])[::-1]


def residual_norm(lam, s):
    """max |grad log c(lam) - s| -- the equations of find_eigenvalues_v3 (complex_bingham.py:374-376)."""
    lam = np.asarray(lam, dtype=np.float64)
    return np.max(np.abs(derivatives(lam - lam.max())[0] - np.asarray(s)))


def find_eigenvalues_v3(scatter_eigenvalues, eps=1e-8, max_concentration=np.inf):
    """complex_bingham.py:304-425 for one problem (D values), solved to convergence."""
    inv, s = gap_rule(scatter_eigenvalues, eps)
    D = len(s)
    lb, ub = -max_concentration, UPPER
    with np.errstate(divide='ignore', invalid='ignore'):
        x0 = -1 / s
    x0[-1] = 0
    if np.isfinite(max_concentration):
        x0 = np.maximum(x0, [-(max_concentration - d) for d in range(D)])
    with np.errstate(invalid='ignore'):
        x = -np.diff(x0)
    if not np.all((x >= lb) & (x <= ub) & np.isfinite(x)):
        raise ValueError(x, s)

    def evaluate(x):
        lam = _lambda_from_diff(x)
        g, H = derivatives(lam)
        r = g - s
        return lam, H, r, np.sum(r * r)

    lam, H, r, phi = evaluate(x)
    for _ in range(MAX_STEPS):
        if not np.max(np.abs(r)) > TOL:
            break
        J = np.cumsum(H[:, :D - 1], axis=1)
        grad = J.T @ r
        free = ~(((x <= lb) & (grad > 0)) | ((x >= ub) & (grad < 0)))
        step = np.zeros(D - 1)
        if free.any():
            step[free] = np.linalg.lstsq(J[:, free], -r, rcond=None)[0]
        alpha, accepted = 1.0, False
        for _ in range(MAX_HALVINGS):
            xt = np.clip(x + alpha * step, lb, ub)
            if np.array_equal(xt, x):
                break
            t = evaluate(xt)
            if t[3] < phi:
                x, (lam, H, r, phi), accepted = xt, t, True
                break
            alpha *= 0.5
        if not accepted:
            break
    est = lam[inv]
    if np.isfinite(max_concentration):
        est = np.maximum(est, -max_concentration)
        inv2, est = gap_rule(est, eps)
        est = est[inv2]
    return est


def scatter(y, saliency):
    """complex_bingham.py:567-579: sum_n sal y y^H / sum_n sal, hermitised; y (..., N, D), saliency (..., N)."""
    cov = np.einsum('...n,...nd,...nD->...dD', saliency, y, y.conj())
    cov /= np.einsum('...n->...', saliency)[..., None, None]
    return (cov + np.swapaxes(cov.conj(), -1, -2)) / 2


def bingham_fit(y, saliency, eps=1e-8, max_concentration=np.inf):
    """ComplexBinghamTrainer._fit (complex_bingham.py:567-594) with the device's eigenvalue check."""
    s_all, V = np.linalg.eigh(scatter(y, saliency))
    lam = np.empty_like(s_all)
    for idx in np.ndindex(s_all.shape[:-1]):
        s = s_all[idx]
        assert s[0] > ZERO * s[-1], s
        lam[idx] = find_eigenvalues_v3(s, eps, max_concentration)
    return V, lam


def log_pdf(y, V, lam):
    """ComplexBingham.log_pdf (complex_bingham.py:59-78), y (..., T, D) against (..., D, D) / (..., D)."""
    B = np.einsum('...wx,...x,...zx->...wz', V, lam, V.conj())
    return np.einsum('...td,...dD,...tD->...t', y.conj(), B, y).real - log_norm(lam)[..., None]


def cbmm_predict(y, model, affiliation_eps=0.):
    """CBMM.predict (cbmm.py:26-55)."""
    z = normalize_observation_cw(y)
    return log_pdf_to_affiliation(model['weight'], log_pdf(z[..., None, :, :], model['V'], model['lam']),
                                  affiliation_eps=affiliation_eps)


def cbmm_m_step(z, affiliation, saliency, weight_constant_axis=(-1,), eps=1e-8, max_concentration=np.inf):
    """CBMMTrainer._m_step (cbmm.py:215-237)."""
    weight = estimate_mixture_weight(affiliation, saliency, weight_constant_axis)
    V, lam = bingham_fit(z[..., None, :, :], affiliation * saliency[..., None, :], eps, max_concentration)
    return dict(weight=weight, V=V, lam=lam)


def cbmm_fit(y, initialization, iterations, *, saliency=None, weight_constant_axis=(-1,), affiliation_eps=0.,
             eps=1e-8, max_concentration=np.inf):
    """CBMMTrainer.fit / _fit (cbmm.py:79-205), without inline permutation alignment."""
    z = normalize_observation_cw(y)
    if saliency is None:
        saliency = np.ones_like(initialization[..., 0, :])
    affiliation = initialization
    model = None
    for _ in range(iterations):
        if model is not None:
            affiliation = cbmm_predict(z, model, affiliation_eps)
        model = cbmm_m_step(z, affiliation, saliency, weight_constant_axis, eps, max_concentration)
    return model


def model_covariance(V, s):
    """V diag(s) V^H: compares eigenvector sets independently of their phases."""
    return np.einsum('...wx,...x,...zx->...wz', V, s, V.conj())
