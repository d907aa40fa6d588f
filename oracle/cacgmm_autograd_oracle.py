"""float64 torch restatement of the cACGMM's M-step, E-step, predict, log_likelihood and EM loop that torch autograd
differentiates (TEST INFRASTRUCTURE, see oracle/__init__.py).

The values follow oracle/pb_bss_oracle.py (cacgmm_m_step, cacgmm_e_step, cacgmm_fit, cacgmm_log_likelihood), which
pins pb_bss/distribution/cacgmm.py and complex_angular_central_gaussian.py.  The gradient conventions are those stated
in include/pbb.h for pbb_cacgmm_mstep_backward / pbb_cacgmm_predict_backward: floors and clips pass no gradient where
they are active, a zero frame has a zero gradient, a class whose affiliations sum to at most tiny passes none.

The model of an M-step reaches its consumers only as B^-1 = V diag(1 / lam) V^H and log det B = sum log lam, formed
from the covariance by ``SpectralModel``, whose backward is the Loewner (divided-difference) formula: a pair of floored
model eigenvalues contributes zero and a pair of unfloored ones the closed form -lam' / (lam_i lam_j), so floored bins
and tied eigenvalues have a finite, correct reference, where torch.linalg.eigh's own backward divides by the vanishing
gaps.  ``mp_loss`` is an independent reference: the same forward at 40 digits in mpmath, differentiated by central
differences.

Tensors: y (..., N, D) complex, affiliations / quadratic forms (..., K, N), saliency (..., N); a model is a dict with
``binv`` (..., K, D, D), ``logdet`` (..., K), ``weight`` (..., K, 1) and, from an M-step, the values ``eigenvectors``
/ ``eigenvalues`` (no graph).
"""
import numpy as np
import torch

TINY = torch.finfo(torch.float64).tiny
KINK_GAP = 64 * 2.0 ** -52   # kKinkGap of em_backward.cuh


def _keep(cond, x):
    """x where cond, else x without a gradient (a clamp that is active passes none)"""
    return torch.where(cond, x, x.detach())


def normalize(y):
    """y / |y| per frame (the reference's 'where' normalisation); an all-zero frame stays zero with zero gradient"""
    y = y.to(torch.complex128)
    n = torch.linalg.vector_norm(y, dim=-1, keepdim=True)
    nz = n != 0
    return y / torch.where(nz, n, torch.ones_like(n)) * nz


def model_eigenvalues(mu, m, floor, norm):
    """The floored model eigenvalues from the raw ones mu (..., D) and the top one m (..., 1)"""
    if norm == 'eigenvalue':
        return torch.clamp(mu / torch.clamp(m, min=TINY), min=floor)
    return torch.maximum(mu, m * floor)


class SpectralModel(torch.autograd.Function):
    """(C Hermitian (..., D, D), m (..., 1)) -> (B^-1 = V diag(1 / lam) V^H, sum log lam) with lam =
    model_eigenvalues(eigh(C), m).  Backward (Daleckii-Krein): Cbar = V (L o (V^H Bbar V) + diag(ldbar lam' / lam)) V^H
    with lam'_i = d lam_i / d mu_i, L_ii = -lam'_i / lam_i^2 and, for i != j, the divided differences
    L_ij = (1/lam_i - 1/lam_j) / (mu_i - mu_j): -lam' / (lam_i lam_j) where neither eigenvalue is floored (also at a
    tie mu_i == mu_j), 0 where both are; and mbar from d lam / d m.  m is an input, so a caller that forms it as the
    Rayleigh quotient of the top eigenvector (m_step) gets the gradient of the loss with that eigenvector held fixed:
    the derivative of mu_max where the top eigenvalue is simple, and that convention where it is tied."""

    @staticmethod
    def forward(ctx, C, m, floor, norm):
        mu, V = torch.linalg.eigh(C)
        lam = model_eigenvalues(mu, m, floor, norm)
        binv = (V / lam[..., None, :].to(V.dtype)) @ V.mH
        ctx.save_for_backward(V, mu, m, lam)
        ctx.floor, ctx.norm = floor, norm
        return binv, torch.log(lam).sum(-1)

    @staticmethod
    def backward(ctx, gb, gld):
        V, mu, m, lam = ctx.saved_tensors
        floor, norm = ctx.floor, ctx.norm
        if norm == 'eigenvalue':
            mm = torch.clamp(m, min=TINY)
            pass_ = lam > floor
            dlam = torch.where(pass_, 1 / mm, torch.zeros_like(mu))
            dlam_m = torch.where(pass_, -mu / mm ** 2, torch.zeros_like(mu)) * (m > TINY)
        else:
            pass_ = mu > m * floor            # the side of the maximum that lam took (not lam > lam_max floor:
            #                                   m is a Rayleigh quotient, lam_max = mu_max may differ from it in the last bit)
            dlam = pass_.to(mu.dtype)
            dlam_m = (~pass_).to(mu.dtype) * floor
        gb = torch.zeros_like(V) if gb is None else gb
        gld = torch.zeros_like(mu[..., 0]) if gld is None else gld
        P = V.mH @ ((gb + gb.mH) / 2) @ V
        f = 1 / lam
        diff_mu = mu[..., :, None] - mu[..., None, :]
        off = ~torch.eye(mu.shape[-1], dtype=torch.bool, device=mu.device)   # the diagonal is dg below
        both = pass_[..., :, None] & pass_[..., None, :] & off
        none = ~(pass_[..., :, None] | pass_[..., None, :]) | ~off
        # unfloored pairs: (1/lam_i - 1/lam_j) / (mu_i - mu_j) = -lam' / (lam_i lam_j) exactly (lam' = d lam / d mu is
        # the same for both), which is also the limit -lam'_i / lam_i^2 at a tie and has no cancellation near one;
        # a floored pair (1/lam constant) gives 0; a mixed pair the divided difference, but 0 where the gap is within
        # KINK_GAP D mu_max (both at the floor's kink, the convention of pbb.h)
        kink = diff_mu.abs() <= KINK_GAP * mu.shape[-1] * mu[..., -1:, None]
        mixed = (f[..., :, None] - f[..., None, :]) / torch.where(kink, torch.ones_like(diff_mu), diff_mu)
        mixed = torch.where(kink, torch.zeros_like(mixed), mixed)
        L = torch.where(both, -dlam[..., :, None] * f[..., :, None] * f[..., None, :],
                        torch.where(none, torch.zeros_like(diff_mu), mixed))
        # d/d mu_i of (sum_j P_jj / lam_j + ldbar sum_j log lam_j) through lam_i
        dg = (-P.diagonal(dim1=-2, dim2=-1).real / lam ** 2 + gld[..., None] / lam)
        M = L.to(V.dtype) * P + torch.diag_embed((dg * dlam).to(V.dtype))
        gC = V @ M @ V.mH
        gm = (dg * dlam_m).sum(-1, keepdim=True)
        return gC, gm, None, None


def m_step(y, quadratic_form, affiliation, saliency=None, covariance_norm='eigenvalue', eigenvalue_floor=1e-10,
           weight_constant_axis=(-1,)):
    """cacgmm.py:315-345: the model of one M-step.  quadratic_form None means ones."""
    z = normalize(y)                                     # (..., N, D)
    D = z.shape[-1]
    gamma = affiliation.to(torch.float64)
    g = gamma if saliency is None else gamma * saliency.to(torch.float64)[..., None, :]
    S = g.sum(-1)                                        # (..., K)
    live = S > TINY
    g = _keep(live[..., None], g)
    gamma = _keep(live[..., None], gamma)
    S = g.sum(-1)
    if quadratic_form is None:
        c = g
    else:
        q = quadratic_form.to(torch.float64)
        c = g / torch.where(q > 10 * TINY, q, torch.full_like(q, 10 * TINY))
    # a class with S <= tiny passes no gradient at all: its covariance D psi / tiny is a constant
    psi = _keep(live[..., None, None], torch.einsum('...kn,...nd,...ne->...kde', c.to(torch.complex128), z, z.conj()))
    C = D * psi / torch.where(live, S, torch.full_like(S, TINY))[..., None, None]
    C = (C + C.mH) / 2
    if covariance_norm == 'trace':
        tr = C.diagonal(dim1=-2, dim2=-1).real.sum(-1)
        C = C / torch.where(tr > TINY, tr, torch.full_like(tr, TINY))[..., None, None]
    norm = covariance_norm if covariance_norm in ('eigenvalue', 'trace') else False
    with torch.no_grad():
        mu, V = torch.linalg.eigh(C)
    top = V[..., -1:]                                    # the top eigenvector: m = Re v^H C v
    m = (top.mH @ C @ top).real[..., 0]
    binv, logdet = SpectralModel.apply(C, m, eigenvalue_floor, norm)
    K = gamma.shape[-2]
    if isinstance(weight_constant_axis, int) and weight_constant_axis % gamma.dim() - gamma.dim() == -2:
        weight = torch.full((K, 1), 1 / K, dtype=torch.float64, device=gamma.device)
    elif saliency is None:
        weight = gamma.mean(-1, keepdim=True)
    else:
        n = S.abs().sum(-1, keepdim=True)
        weight = (S / torch.where(n == 0, torch.full_like(n, 1e-10), n))[..., None]
    return dict(weight=weight, binv=binv, logdet=logdet, eigenvectors=V.detach(),
                eigenvalues=model_eigenvalues(mu, mu[..., -1:], eigenvalue_floor, norm).detach())


def from_eig(eigenvectors, eigenvalues, weight):
    """A model dict from eigenvectors, eigenvalues and weight, differentiable in all three"""
    V = eigenvectors.to(torch.complex128)
    lam = eigenvalues.to(torch.float64)
    return dict(weight=weight.to(torch.float64), binv=(V / lam[..., None, :].to(V.dtype)) @ V.mH,
                logdet=torch.log(lam).sum(-1))


def e_step(y, model, source_activity_mask=None, affiliation_eps=0.):
    """cacgmm.py:73-95: (affiliation, quadratic form, log pdf), each (..., K, N)"""
    z = normalize(y)
    D = z.shape[-1]
    qr = torch.einsum('...nd,...kde,...ne->...kn', z.conj(), model['binv'], z).real
    aq = qr.abs()
    q = torch.where(aq > TINY, aq, torch.full_like(aq, TINY))
    lp = -D * torch.log(q) - model['logdet'][..., None]
    a = torch.exp(lp - lp.max(-2, keepdim=True).values.detach()) * model['weight']
    if source_activity_mask is not None:
        a = a * source_activity_mask
    den = a.sum(-2, keepdim=True)
    gamma = a / torch.where(den > TINY, den, torch.full_like(den, TINY))
    if affiliation_eps != 0:
        inside = (gamma > affiliation_eps) & (gamma < 1 - affiliation_eps)
        gamma = torch.where(inside, gamma, gamma.clamp(affiliation_eps, 1 - affiliation_eps).detach())
    return gamma, q, lp


def predict(y, model, return_quadratic_form=False, source_activity_mask=None):
    """cacgmm.py:64-71 (affiliation_eps = 0)"""
    gamma, q, _ = e_step(y, model, source_activity_mask, 0.)
    return (gamma, q) if return_quadratic_form else gamma


def log_likelihood_per_bin(y, model):
    """sum_t logsumexp_k log pdf per bin (..., ) (cacgmm.py:97-138, without the weights)"""
    _, _, lp = e_step(y, model)
    m = lp.max(-2, keepdim=True).values.detach()
    return (m[..., 0, :] + torch.log(torch.exp(lp - m).sum(-2))).sum(-1)


def log_likelihood(y, model):
    return log_likelihood_per_bin(y, model).sum()


def fit(y, initialization, iterations, saliency=None, source_activity_mask=None, weight_constant_axis=(-1,),
        covariance_norm='eigenvalue', affiliation_eps=1e-10, eigenvalue_floor=1e-10):
    """cacgmm.py:252-278: an M-step from the initial affiliations (quadratic form ones), then per iteration an E-step
    and an M-step; ``initialization`` may be a model dict (warm start)."""
    model, gamma, q = None, None, None
    if isinstance(initialization, dict):
        model = initialization
    else:
        gamma = initialization
    for _ in range(iterations):
        if model is not None:
            gamma, q, _ = e_step(y, model, source_activity_mask, affiliation_eps)
        model = m_step(y, q, gamma, saliency, covariance_norm, eigenvalue_floor, weight_constant_axis)
    return model


def tie_data(D, weights, probe_T=6, seed=0):
    """One bin, one frame per basis vector e_d (times 3 + 4j, so |y| = 5 and every z z^H is the same float64 matrix up
    to its position) and K classes whose affiliations put weights[k][d] on e_d: C_k = D diag(weights[k]) / S_k holds
    exactly the ties of weights[k] in float64 too.  Returns (y, init, probe, R): probe frames are random, so the loss
    sees every direction of B^-1."""
    K = len(weights)
    y = (3 + 4j) * np.eye(D, dtype=np.complex128)[None]
    init = np.asarray(weights, dtype=np.float64)[None]
    rng = np.random.RandomState(seed)
    probe = rng.standard_normal((1, probe_T, D)) + 1j * rng.standard_normal((1, probe_T, D))
    R = rng.standard_normal((1, K, probe_T))
    return y, init, probe, R


# ---- mpmath reference ------------------------------------------------------------------------------------------------
DPS = 40


def mp_loss(x, covariance_norm='eigenvalue', eigenvalue_floor=1e-10, affiliation_eps=1e-10, weight_constant_axis=-1,
            mask=None, iterations=1, probe=None, R=None, c_ll=0.1, top=None, dps=DPS):
    """The scalar loss sum R * predict(probe, model) + c_ll * log_likelihood(probe, model) at ``dps`` digits, where the
    model comes from ``iterations`` M-steps as in ``fit``: from x['init'] (F, K, T) (with x['q'] as the first
    quadratic form, ones without), or from x['V'] (F, K, D, D), x['lam'] (F, K, D), x['w'] (F, K[, 1]) (then iterations
    may be 0: predict / log_likelihood of that model).  x['y'] (F, T, D), x['saliency'] (F, T) optional; every entry of
    x is a numpy array of mpmath numbers or floats.  probe defaults to y (the same numbers), R (F, K, Tp) to zeros.
    ``top`` (F, K, D): the forward's top eigenvectors of the first M-step; where given, that M-step's m is their
    Rayleigh quotient instead of mu_max (the gradient convention at a tied top eigenvalue).  Returns an mpf."""
    import mpmath as mp
    with mp.workdps(dps):
        tiny = mp.mpf(TINY)
        y = x['y']
        F, T, D = y.shape
        total = mp.mpf(0)
        for f in range(F):
            z = [_mp_normalize(mp, y[f, t]) for t in range(T)]
            if 'V' in x:
                K = x['V'].shape[1]
                model = [_mp_from_eig(mp, x['V'][f, k], x['lam'][f, k], D) for k in range(K)]
                weight = list(np.reshape(x['w'][f], -1))
                gamma, q, first = None, None, False
            else:
                K = x['init'].shape[1]
                model, gamma = None, x['init'][f]
                q = x['q'][f] if 'q' in x else None
                first = True
            sal = x['saliency'][f] if 'saliency' in x else None
            for _ in range(iterations):
                if model is not None:
                    gamma, q, _ = _mp_e_step(mp, z, model, weight, None if mask is None else mask[f], affiliation_eps,
                                             tiny)
                model, weight = _mp_m_step(mp, z, gamma, q, sal, covariance_norm, eigenvalue_floor,
                                           weight_constant_axis, tiny, top[f] if (first and top is not None) else None)
                first = False
            zp = z if probe is None else [_mp_normalize(mp, probe[f, t]) for t in range(probe.shape[1])]
            gamma, _, lp = _mp_e_step(mp, zp, model, weight, None, 0.0, tiny)
            if R is not None:
                total += mp.fsum(mp.mpf(float(R[f, k, t])) * gamma[k][t] for k in range(K) for t in range(len(zp)))
            if c_ll:
                for t in range(len(zp)):
                    m = max(lp[k][t] for k in range(K))
                    total += mp.mpf(c_ll) * (m + mp.log(mp.fsum(mp.exp(lp[k][t] - m) for k in range(K))))
        return +total


def _mp_normalize(mp, v):
    n = mp.sqrt(mp.fsum(abs(e) ** 2 for e in v))
    return [e / n for e in v] if n != 0 else [mp.mpc(0) for _ in v]


def _mp_from_eig(mp, V, lam, D):
    """(B^-1 as a D x D list, log det) of V diag(lam) V^H"""
    binv = [[mp.fsum(V[d, i] * mp.conj(V[e, i]) / lam[i] for i in range(D)) for e in range(D)] for d in range(D)]
    return binv, mp.fsum(mp.log(lam[i]) for i in range(D))


def _mp_m_step(mp, z, gamma, q, sal, norm, floor, wca, tiny, top):
    K, T, D = len(gamma), len(z), len(z[0])
    g = [[gamma[k][t] * (sal[t] if sal is not None else 1) for t in range(T)] for k in range(K)]
    S = [mp.fsum(g[k]) for k in range(K)]
    model = []
    for k in range(K):
        c = [g[k][t] / (max(q[k][t], 10 * tiny) if q is not None else 1) for t in range(T)]
        C = mp.matrix(D, D)
        for d in range(D):
            for e in range(D):
                C[d, e] = mp.fsum(c[t] * z[t][d] * mp.conj(z[t][e]) for t in range(T)) * D / max(S[k], tiny)
        if norm == 'trace':
            tr = max(mp.re(mp.fsum(C[d, d] for d in range(D))), tiny)
            C = C / tr
        w, Q = mp.eighe(C)
        order = sorted(range(D), key=lambda i: mp.re(w[i]))
        mu = [mp.re(w[i]) for i in order]
        V = [[Q[d, i] for i in order] for d in range(D)]
        if top is None:
            m = mu[-1]
        else:
            v = [mp.mpc(complex(top[k][d, -1])) for d in range(D)]
            m = mp.re(mp.fsum(mp.conj(v[d]) * C[d, e] * v[e] for d in range(D) for e in range(D)))
        if norm == 'eigenvalue':
            lam = [max(u / max(m, tiny), floor) for u in mu]
        else:
            lam = [max(u, m * floor) for u in mu]
        Vm = np.empty((D, D), dtype=object)
        for d in range(D):
            for i in range(D):
                Vm[d, i] = V[d][i]
        model.append(_mp_from_eig(mp, Vm, lam, D))
    if wca == -2:
        weight = [mp.mpf(1) / K] * K
    elif sal is None:
        weight = [mp.fsum(gamma[k]) / T for k in range(K)]
    else:
        n = mp.fsum(abs(s) for s in S)
        weight = [s / (n if n != 0 else mp.mpf(1e-10)) for s in S]
    return model, weight


def _mp_e_step(mp, z, model, weight, mask, eps, tiny):
    K, T, D = len(model), len(z), len(z[0])
    q = [[None] * T for _ in range(K)]
    lp = [[None] * T for _ in range(K)]
    for k in range(K):
        binv, ld = model[k]
        for t in range(T):
            qr = mp.re(mp.fsum(mp.conj(z[t][d]) * binv[d][e] * z[t][e] for d in range(D) for e in range(D)))
            q[k][t] = max(abs(qr), tiny)
            lp[k][t] = -D * mp.log(q[k][t]) - ld
    gamma = [[None] * T for _ in range(K)]
    for t in range(T):
        m = max(lp[k][t] for k in range(K))
        a = [mp.exp(lp[k][t] - m) * weight[k] * (1 if mask is None or mask[k, t] else 0) for k in range(K)]
        den = max(mp.fsum(a), tiny)
        for k in range(K):
            gk = a[k] / den
            if eps != 0:
                gk = min(max(gk, mp.mpf(eps)), 1 - mp.mpf(eps))
            gamma[k][t] = gk
    return gamma, q, lp


def mp_directional(inputs, dirs, h=1e-15, dps=DPS, **kw):
    """d/ds mp_loss(inputs + s dirs) at s = 0 by a central difference at ``dps`` digits (float).  inputs / dirs: dicts
    of numpy arrays (dirs a subset of the keys); the truncation error is ~h^2 times the third derivative, the rounding
    error ~10^-dps / h."""
    import mpmath as mp
    with mp.workdps(dps):
        hh = mp.mpf(h)

        def at(s):
            x = {}
            for key, v in inputs.items():
                cplx = np.iscomplexobj(v) or (key in dirs and np.iscomplexobj(dirs[key]))
                conv = (lambda a: mp.mpc(complex(a))) if cplx else (lambda a: mp.mpf(float(a)))
                a = np.vectorize(conv, otypes=[object])(v)
                if key in dirs:
                    a = a + np.vectorize(conv, otypes=[object])(dirs[key]) * s
                x[key] = a
            return mp_loss(x, dps=dps, **kw)
        return float((at(hh) - at(-hh)) / (2 * hh))


def directional(grads, dirs):
    """sum over the inputs of Re <grad, dir> (grad z = dL/dRe z + i dL/dIm z for complex inputs)"""
    return sum(float(np.real(np.sum(np.conj(np.asarray(grads[k])) * dirs[k]))) for k in dirs)
