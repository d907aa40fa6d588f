"""float64 torch restatement of the cACGMM's M-step, E-step, predict, log_likelihood and EM loop that torch autograd
differentiates (TEST INFRASTRUCTURE, see oracle/__init__.py).

The values follow oracle/pb_bss_oracle.py (cacgmm_m_step, cacgmm_e_step, cacgmm_fit, cacgmm_log_likelihood), which
pins pb_bss/distribution/cacgmm.py and complex_angular_central_gaussian.py.  The gradient conventions are those stated
in include/pbb.h for pbb_cacgmm_mstep_backward / pbb_cacgmm_predict_backward: floors and clips pass no gradient where
they are active, a zero frame has a zero gradient, a class whose affiliations sum to at most tiny passes none.

The model of an M-step reaches its consumers only as B^-1 = V diag(1 / lam) V^H and log det B = sum log lam, formed
from the covariance by ``SpectralModel``, whose backward is the Loewner (divided-difference) formula: a pair of equal
model eigenvalues (a floored block) contributes zero, so floored bins have a finite, correct reference, where
torch.linalg.eigh's own backward divides by the vanishing gaps.

Tensors: y (..., N, D) complex, affiliations / quadratic forms (..., K, N), saliency (..., N); a model is a dict with
``binv`` (..., K, D, D), ``logdet`` (..., K), ``weight`` (..., K, 1) and, from an M-step, the values ``eigenvectors``
/ ``eigenvalues`` (no graph).
"""
import torch

TINY = torch.finfo(torch.float64).tiny


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
    model_eigenvalues(eigh(C), m).  Backward: Cbar = V (L o (V^H Bbar V) + diag(ldbar lam' / lam)) V^H with the
    divided differences L_ij = (1/lam_i - 1/lam_j) / (mu_i - mu_j), zero where lam_i == lam_j, L_ii = -lam'_i / lam_i^2,
    lam'_i = d lam_i / d mu_i; and mbar from d lam / d m."""

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
            pass_ = lam > lam[..., -1:] * floor
            dlam = pass_.to(mu.dtype)
            dlam_m = (~pass_).to(mu.dtype) * floor
        gb = torch.zeros_like(V) if gb is None else gb
        gld = torch.zeros_like(mu[..., 0]) if gld is None else gld
        P = V.mH @ ((gb + gb.mH) / 2) @ V
        f = 1 / lam
        diff_mu = mu[..., :, None] - mu[..., None, :]
        same = lam[..., :, None] == lam[..., None, :]
        L = torch.where(same, torch.zeros_like(diff_mu),
                        (f[..., :, None] - f[..., None, :]) / torch.where(same, torch.ones_like(diff_mu), diff_mu))
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
    psi = torch.einsum('...kn,...nd,...ne->...kde', c.to(torch.complex128), z, z.conj())
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
