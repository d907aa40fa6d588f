"""Pure-torch restatements of the get_bf_vector beamformers of pb_bss_b200 (GEV, PCA, MVDR, blind analytic
normalisation, the rank-1 estimate and the matvec of the scaled GEV ATF), so that torch's own autograd gives the
reference gradients of their device backward passes; the closed forms of those gradients (include/pbb.h); and
long-double references with per-bin bounds of the kind autograd_oracle.souden_grad_ref uses.  Runs on CPU or CUDA
tensors in complex128.  Test infrastructure only, like the rest of oracle/."""
import numpy as np
import torch

from .autograd_oracle import C_G, CLD, LD, U, U32, _err, _ratio, _rounded, gamma  # noqa: F401


# Restatements in torch (complex128), so that torch's autograd gives the reference gradients.  The eigenvector ones fix
# the phase: w~ = w |p| / p with p = w.detach()^H B.detach() w, which equals w at the point and removes the component
# i Im(w^H B dw) w from dw -- the phase-held convention of the device backward (Im(w^H B dw) = 0), and a loss of w~ no
# longer depends on the phase, which torch's eigh backward requires.

def _herm(A):
    return (A + A.conj().transpose(-1, -2)) / 2


def fix_phase(w, B=None, ref=None):
    """w |p| / p, p = r^H B.detach() w with r = w.detach() (B None: the identity).  With ref (a constant vector of the
    same phase class, such as the device's output) r = ref: the result then also takes ref's phase, so that a
    phase-dependent loss of it matches the device's forward, and Im(ref^H B dw~) = 0 holds for its derivative."""
    Bw = w if B is None else (B.detach() @ w[..., None])[..., 0]
    r = w.detach() if ref is None else ref.detach().to(w.dtype)
    p = (r.conj() * Bw).sum(-1, keepdim=True)
    return w * (p.abs() / p)


def _gev_basis(A, B):
    """(eigenvalues ascending, generalised eigenvectors W as columns, W^H B W = I) of the Hermitian parts of (A, B):
    B = L L^H, C = L^-1 A L^-H, eigh(C) = (lam, Y), W = L^-H Y (zhegvd ITYPE = 1, as gev_kernel)."""
    L = torch.linalg.cholesky(_herm(B))
    C = torch.linalg.solve_triangular(L, _herm(A), upper=False)
    C = torch.linalg.solve_triangular(L, C.conj().transpose(-1, -2), upper=False).conj().transpose(-1, -2)
    lam, Y = torch.linalg.eigh(_herm(C))
    W = torch.linalg.solve_triangular(L.conj().transpose(-1, -2), Y, upper=True)
    return lam, W


def gev_vector(A, B, ref=None):
    """(top generalised eigenvector with w^H B w = 1, phase fixed (to ref's, if given); its eigenvalue) of the
    Hermitian parts."""
    lam, W = _gev_basis(A, B)
    return fix_phase(W[..., -1], _herm(B), ref), lam[..., -1]


def pca(A, ref=None):
    """(top eigenvalue, its unit eigenvector, phase fixed (to ref's, if given)) of the Hermitian part of A."""
    lam, V = torch.linalg.eigh(_herm(A))
    return lam[..., -1], fix_phase(V[..., -1], None, ref)


def mvdr_vector(atf, noise):
    """w = N_h^-1 a / (a^H N_h^-1 a), N_h = (N + N^H) / 2."""
    x = torch.linalg.solve(_herm(noise), atf[..., None])[..., 0]
    return x / (atf.conj() * x).sum(-1, keepdim=True)


def blind_analytic_normalization(w, noise):
    """w sqrt|w^H N N w| / |w^H N w|, N as given."""
    r = (noise @ w[..., None])[..., 0]
    l = (noise.conj().transpose(-1, -2) @ w[..., None])[..., 0]
    nu = (l.conj() * r).sum(-1)
    de = (w.conj() * r).sum(-1)
    return w * (torch.sqrt(nu.abs()) / de.abs())[..., None]


def rank_one_estimate(a, cov):
    """a a^H tr(C) / |a|^2 with the complex trace."""
    tr = torch.diagonal(cov, dim1=-2, dim2=-1).sum(-1)
    na = (a.abs() ** 2).sum(-1)
    return a[..., :, None] * a.conj()[..., None, :] * (tr / na)[..., None, None]


def matvec(M, x):
    return (M @ x[..., None])[..., 0]


# ---- closed forms of the gradients (restated from include/pbb.h) ----

def _outer(x, y):
    return x[..., :, None] * y.conj()[..., None, :]


def eig_grad(A, B, w, g, g_lambda=None):
    """(grad A, grad B) of the top eigenpair for the forward's vector w (any phase) and the incoming g (and g_lambda):
    u = sum_{j != top} w_j (w_j^H g) / (lambda - lambda_j), grad A = (u w^H + w u^H) / 2 + g_lambda w w^H,
    grad B = -lambda (u w^H + w u^H) / 2 - (Re(w^H g) / 2 + lambda g_lambda) w w^H (None for B None)."""
    if B is None:
        lam, W = torch.linalg.eigh(_herm(A))
    else:
        lam, W = _gev_basis(A, B)
    D = lam.shape[-1]
    lt = lam[..., -1:]
    coef = (W.conj().transpose(-1, -2) @ g[..., None])[..., 0]
    keep = torch.arange(D, device=lam.device) < D - 1
    den = torch.where(keep, lt - lam, torch.ones_like(lam))
    u = (W @ torch.where(keep, coef / den, torch.zeros_like(coef))[..., None])[..., 0]
    sym = (_outer(u, w) + _outer(w, u)) / 2
    ww = _outer(w, w)
    gl = torch.zeros_like(lt[..., 0]) if g_lambda is None else g_lambda.to(lam.dtype)
    gA = sym + gl[..., None, None] * ww
    if B is None:
        return gA, None
    rho = (w.conj() * g).sum(-1).real
    lt = lt[..., 0]
    gB = -lt[..., None, None] * sym - (rho / 2 + lt * gl)[..., None, None] * ww
    return gA, gB


def mvdr_grad(atf, noise, g):
    """(grad a, grad N): t = w^H g, q = (g - t a) / conj(s), p = N_h^-1 q, grad a = p - conj(t) w,
    grad N = -(p x^H + x p^H) / 2."""
    Nh = _herm(noise)
    x = torch.linalg.solve(Nh, atf[..., None])[..., 0]
    s = (atf.conj() * x).sum(-1, keepdim=True)
    w = x / s
    t = (w.conj() * g).sum(-1, keepdim=True)
    p = torch.linalg.solve(Nh, ((g - t * atf) / s.conj())[..., None])[..., 0]
    return p - t.conj() * w, -(_outer(p, x) + _outer(x, p)) / 2


def _ban_parts(w, N, g):
    r = (N @ w[..., None])[..., 0]
    l = (N.conj().transpose(-1, -2) @ w[..., None])[..., 0]
    nu = (l.conj() * r).sum(-1)
    de = (w.conj() * r).sum(-1)
    c = nu.abs() ** 0.5 / de.abs()
    rho = (w.conj() * g).sum(-1).real
    alpha = rho * c * nu.conj() / (2 * nu.abs() ** 2)
    beta = -rho * c * de.conj() / de.abs() ** 2
    return r, l, c, alpha, beta


def ban_grad(w, N, g):
    """(grad w, grad N): grad w = c g + alpha N r + conj(alpha) N^H l + beta r + conj(beta) l,
    grad N = conj(alpha) (w r^H + l w^H) + conj(beta) w w^H."""
    r, l, c, alpha, beta = _ban_parts(w, N, g)
    Nr = (N @ r[..., None])[..., 0]
    NHl = (N.conj().transpose(-1, -2) @ l[..., None])[..., 0]
    a, b = alpha[..., None], beta[..., None]
    gw = c[..., None] * g + a * Nr + a.conj() * NHl + b * r + b.conj() * l
    gN = a.conj()[..., None] * (_outer(w, r) + _outer(l, w)) + b.conj()[..., None] * _outer(w, w)
    return gw, gN


def rank_one_grad(a, cov, G):
    """(grad a, grad C): (conj(t) G a + t G^H a) / nu - 2 Re(t conj(q)) / nu^2 a and (q / nu) I, q = a^H G a."""
    tr = torch.diagonal(cov, dim1=-2, dim2=-1).sum(-1)[..., None]
    na = (a.abs() ** 2).sum(-1)[..., None]
    Ga = (G @ a[..., None])[..., 0]
    GHa = (G.conj().transpose(-1, -2) @ a[..., None])[..., 0]
    q = (a.conj() * Ga).sum(-1, keepdim=True)
    ga = (tr.conj() * Ga + tr * GHa) / na - 2 * (tr * q.conj()).real / na ** 2 * a
    eye = torch.eye(a.shape[-1], dtype=a.dtype, device=a.device)
    return ga, (q / na)[..., None] * eye


def matvec_grad(M, x, g):
    """(grad M, grad x) = (g x^H, M^H g)."""
    return _outer(g, x), (M.conj().transpose(-1, -2) @ g[..., None])[..., 0]


# ---- long-double references and bounds (per bin, Frobenius; error / bound <= 1 passes) ----
C_EIG = 16.0
C_MVDR = 8.0
C_BAN = 4.0


def _fro(x, axes):
    return np.sqrt((np.abs(np.asarray(x)).astype(np.float64) ** 2).sum(axes))


def eig_grad_ref(A, B, w, g, g_lambda=None):
    """(grad A*, grad B* (None for B None), bound A, bound B) per bin for A, B (n, D, D), the device's w and g (n, D)
    and g_lambda (n) or None.

    The projector comes from float64 LAPACK (scipy.linalg.eigh of the Hermitian parts, ITYPE = 1 for a pencil); u, the
    outer products and the sums are formed in long double with the device's w, whose phase the gradient is tied to.
    Bound: the device recomputes the projector P = sum_{j != top} w_j w_j^H / (lambda - lambda_j) from its own
    reduction and Jacobi solver.  A backward error of order u D kappa(B) ||C|| in C = L^-1 A L^-H moves P by
    ||C|| / gap times ||P|| <= ||B^-1|| / gap (gap = min_j |lambda - lambda_j|), so
      ||u - u*|| <= C_EIG u D kappa(B) (||C|| / gap) ||B^-1|| ||g|| / gap,
      ||grad A - grad A*|| <= (||u - u*|| + C_EIG u D |g_lambda| ||w||) ||w||,
      ||grad B - grad B*|| <= |lambda| ||grad A - grad A*|| + C_EIG u D (kappa(B) ||C|| ||u*|| + |Re(w^H g)| ||w||
                               + |lambda g_lambda| ||w||) ||w||.
    The float64 projector's own error is of the same order and inside the bound.  A tied top eigenvalue (gap = 0)
    gives an infinite bound."""
    import scipy.linalg
    A = np.asarray(A, dtype=np.complex128)
    n, D = A.shape[0], A.shape[-1]
    Bm = None if B is None else np.asarray(B, dtype=np.complex128)
    w = np.asarray(w, dtype=np.complex128)
    g = np.asarray(g, dtype=np.complex128)
    gl = np.zeros(n) if g_lambda is None else np.asarray(g_lambda, dtype=np.float64)
    gA = np.empty((n, D, D), dtype=CLD)
    gB = None if Bm is None else np.empty((n, D, D), dtype=CLD)
    bA, bB = np.empty(n), np.empty(n)
    for m in range(n):
        Ah = (A[m] + A[m].conj().T) / 2
        if Bm is None:
            lam, W = np.linalg.eigh(Ah)
            kappa, binv = 1.0, 1.0
        else:
            Bh = (Bm[m] + Bm[m].conj().T) / 2
            lam, W = scipy.linalg.eigh(Ah, Bh)
            sv = np.linalg.svd(Bh, compute_uv=False)
            kappa, binv = sv[0] / sv[-1], 1 / sv[-1]
        lt = LD(lam[-1])
        Wl = W.astype(CLD)
        coef = Wl.conj().T @ g[m].astype(CLD)
        den = lt - lam[:-1].astype(LD)
        u = Wl[:, :-1] @ (coef[:-1] / den) if D > 1 else np.zeros(D, dtype=CLD)
        wl = w[m].astype(CLD)
        sym = (np.outer(u, wl.conj()) + np.outer(wl, u.conj())) / 2
        ww = np.outer(wl, wl.conj())
        gA[m] = sym + LD(gl[m]) * ww
        normC = float(np.max(np.abs(lam)))  # ||L^-1 A L^-H||_2: its eigenvalues are the pencil's
        gap = float(np.min(np.abs(lam[-1] - lam[:-1]))) if D > 1 else np.inf
        nw, ng = float(np.linalg.norm(w[m])), float(np.linalg.norm(g[m]))
        err_u = 0.0 if D == 1 else C_EIG * U * D * kappa * normC / gap * binv * ng / gap
        bA[m] = (err_u + C_EIG * U * D * abs(gl[m]) * nw) * nw
        if Bm is not None:
            rho = LD((np.conj(w[m]) * g[m]).sum().real)
            gB[m] = -lt * sym - (rho / 2 + lt * LD(gl[m])) * ww
            nu = float(np.sqrt((np.abs(u).astype(np.float64) ** 2).sum()))
            bB[m] = abs(float(lt)) * bA[m] + C_EIG * U * D * (kappa * normC * nu + abs(float(rho)) * nw
                                                              + abs(float(lt) * gl[m]) * nw) * nw
        else:
            bB[m] = 0.0
    return gA, gB, bA, (None if Bm is None else bB)


def normwise_ratio(got, ref, bound):
    """Per-bin Frobenius error / bound over the trailing axes after the first."""
    err = np.sqrt((_err(got, ref).astype(np.float64) ** 2).reshape(len(bound), -1).sum(-1))
    return _ratio(err, bound)


def mvdr_grad_ref(atf, noise, g):
    """(grad a*, grad N*, bound a, bound N) per bin: mvdr_grad's closed form in long double from float64 solves with
    N_h.  With kappa = kappa(N_h), S_q = (||g|| + |t| ||a||) / |s| (the size of q before g - t a cancels):
      ||grad a - grad a*|| <= C_MVDR u D kappa (||N_h^-1|| S_q + ||p|| + ||g|| ||w||^2),
      ||grad N - grad N*|| <= C_MVDR u D kappa (||N_h^-1|| S_q + ||p||) ||x||."""
    a = np.asarray(atf, dtype=np.complex128)
    N = np.asarray(noise, dtype=np.complex128)
    g = np.asarray(g, dtype=np.complex128)
    n, D = a.shape
    ga = np.empty((n, D), dtype=CLD)
    gN = np.empty((n, D, D), dtype=CLD)
    ba, bN = np.empty(n), np.empty(n)
    for m in range(n):
        Nh = (N[m] + N[m].conj().T) / 2
        x = np.linalg.solve(Nh, a[m]).astype(CLD)
        al, gm = a[m].astype(CLD), g[m].astype(CLD)
        s = (al.conj() * x).sum()
        w = x / s
        t = (w.conj() * gm).sum()
        q = (gm - t * al) / np.conj(s)
        p = np.linalg.solve(Nh, q.astype(np.complex128)).astype(CLD)
        ga[m] = p - np.conj(t) * w
        gN[m] = -(np.outer(p, x.conj()) + np.outer(x, p.conj())) / 2
        sv = np.linalg.svd(Nh, compute_uv=False)
        kappa, ninv = sv[0] / sv[-1], 1 / sv[-1]
        nrm = lambda v: float(np.sqrt((np.abs(v).astype(np.float64) ** 2).sum()))  # noqa: E731
        sq = (nrm(gm) + abs(complex(t)) * nrm(al)) / abs(complex(s))
        ba[m] = C_MVDR * U * D * kappa * (ninv * sq + nrm(p) + nrm(gm) * nrm(w) ** 2)
        bN[m] = C_MVDR * U * D * kappa * (ninv * sq + nrm(p)) * nrm(x)
    return ga, gN, ba, bN


def ban_grad_ref(w, noise, g):
    """(grad w*, grad N*, bound w, bound N) per bin: ban_grad's closed form in long double.  The device forms r, l, nu,
    delta and rho by plain sums, so with the absolute sums r+ = |N| |w|, l+ = |N|^T |w|, nu+ = l+ . r+, delta+ =
    |w| . r+, rho+ = |w| . |g| the relative errors are e_nu = gamma(2D) nu+ / |nu|, e_delta = gamma(2D) delta+ / |delta|,
    e_c = e_nu / 2 + e_delta, and
      d alpha <= |alpha| (e_c + 2 e_nu) + gamma(D) rho+ c / (2 |nu|),  d beta <= |beta| (e_c + 2 e_delta)
               + gamma(D) rho+ c / |delta|;
      ||d grad w|| <= C_BAN (e_c c ||g|| + d alpha (||N r|| + ||N^H l||) + d beta (||r|| + ||l||)
                    + gamma(2D) (|alpha| (|| |N| r+ || + || |N|^T l+ ||) + |beta| (||r+|| + ||l+||)) + 4 u ||grad w*||),
      ||d grad N|| <= C_BAN ((d alpha (||r|| + ||l||) + gamma(D) |alpha| (||r+|| + ||l+||)) ||w|| + d beta ||w||^2
                    + 4 u ||grad N*||).
    Bins with delta = 0 have zero references (bound 0: the device must give exactly 0); nu = 0 ones NaN."""
    w = np.asarray(w, dtype=np.complex128)
    N = np.asarray(noise, dtype=np.complex128)
    g = np.asarray(g, dtype=np.complex128)
    D = w.shape[-1]
    gw, gN = ban_grad(torch.from_numpy(w), torch.from_numpy(N), torch.from_numpy(g))  # float64 sizes for the bound
    wl, Nl, gl = w.astype(CLD), N.astype(CLD), g.astype(CLD)
    r = np.einsum('nij,nj->ni', Nl, wl)
    l = np.einsum('nji,nj->ni', Nl.conj(), wl)
    nu = (l.conj() * r).sum(-1)
    de = (wl.conj() * r).sum(-1)
    with np.errstate(all='ignore'):
        c = np.sqrt(np.abs(nu)) / np.abs(de)
        rho = (wl.conj() * gl).sum(-1).real
        alpha = rho * c * nu.conj() / (2 * np.abs(nu) ** 2)
        beta = -rho * c * de.conj() / np.abs(de) ** 2
        Nr = np.einsum('nij,nj->ni', Nl, r)
        NHl = np.einsum('nji,nj->ni', Nl.conj(), l)
        a, b = alpha[:, None], beta[:, None]
        rw = c[:, None] * gl + a * Nr + a.conj() * NHl + b * r + b.conj() * l
        rN = a.conj()[:, :, None] * (np.einsum('ni,nj->nij', wl, r.conj()) + np.einsum('ni,nj->nij', l, wl.conj())) \
            + b.conj()[:, :, None] * np.einsum('ni,nj->nij', wl, wl.conj())
        zero = np.abs(de) == 0
        rw[zero] = 0
        rN[zero] = 0
        aN, aw, ag = np.abs(N), np.abs(w), np.abs(g)
        rp = np.einsum('nij,nj->ni', aN, aw)
        lp = np.einsum('nji,nj->ni', aN, aw)
        f = lambda v: np.sqrt((np.abs(v).astype(np.float64) ** 2).sum(-1))  # noqa: E731
        e_nu = gamma(2 * D) * (lp * rp).sum(-1) / np.abs(nu).astype(np.float64)
        e_de = gamma(2 * D) * (aw * rp).sum(-1) / np.abs(de).astype(np.float64)
        e_c = e_nu / 2 + e_de
        cf, af_, bf_ = c.astype(np.float64), np.abs(alpha).astype(np.float64), np.abs(beta).astype(np.float64)
        rhop = (aw * ag).sum(-1)
        da = af_ * (e_c + 2 * e_nu) + gamma(D) * rhop * cf / (2 * np.abs(nu).astype(np.float64))
        db = bf_ * (e_c + 2 * e_de) + gamma(D) * rhop * cf / np.abs(de).astype(np.float64)
        nw = f(w)
        bw = C_BAN * (e_c * cf * f(g) + da * (f(Nr) + f(NHl)) + db * (f(r) + f(l))
                      + gamma(2 * D) * (af_ * (f(np.einsum('nij,nj->ni', aN, rp)) + f(np.einsum('nji,nj->ni', aN, lp)))
                                        + bf_ * (f(rp) + f(lp))) + 4 * U * f(gw.numpy()))
        bN = C_BAN * ((da * (f(r) + f(l)) + gamma(D) * af_ * (f(rp) + f(lp))) * nw + db * nw ** 2
                      + 4 * U * np.sqrt((np.abs(gN.numpy()) ** 2).sum((-1, -2))))
    bw = np.where(zero, 0.0, bw)
    bN = np.where(zero, 0.0, bN)
    return rw, rN, bw, bN


def rank_one_grad_ref(a, cov, G):
    """(grad a*, grad C*, bound a, bound C) elementwise: rank_one_grad in long double.  With the device's plain sums
    (t over D, nu over D, G a and G^H a over D, q over D):
      |d grad a_i| <= C_G (gamma(D) (T+ (|Ga_i| + |GHa_i|) + |t| ((|G| |a|)_i + (|G|^T |a|)_i)) / nu
                     + 2 |a_i| (gamma(D) T+ |q| + |t| gamma(2D) q+ + 2 gamma(D) |t| |q|) / nu^2) + 4 u |grad a*_i|,
      |d grad C_dd| <= C_G (gamma(2D) q+ + gamma(D) |q|) / nu,
    T+ = sum_d |C_dd|, q+ = |a|^T |G| |a|; off-diagonal grad C is exactly 0."""
    a = np.asarray(a, dtype=np.complex128)
    C = np.asarray(cov, dtype=np.complex128)
    G = np.asarray(G, dtype=np.complex128)
    D = a.shape[-1]
    al, Cl, Gl = a.astype(CLD), C.astype(CLD), G.astype(CLD)
    tr = np.einsum('nii->n', Cl)[:, None]
    na = (np.abs(al) ** 2).sum(-1)[:, None]
    Ga = np.einsum('nij,nj->ni', Gl, al)
    GHa = np.einsum('nji,nj->ni', Gl.conj(), al)
    q = (al.conj() * Ga).sum(-1)[:, None]
    ga = (tr.conj() * Ga + tr * GHa) / na - 2 * (tr * q.conj()).real / na ** 2 * al
    gC = np.einsum('n,ij->nij', (q / na)[:, 0], np.eye(D))
    aa, aG = np.abs(a), np.abs(G)
    Tp = np.abs(np.einsum('nii->ni', C)).sum(-1)[:, None]
    Gp, GHp = np.einsum('nij,nj->ni', aG, aa), np.einsum('nji,nj->ni', aG, aa)
    qp = (aa * Gp).sum(-1)[:, None]
    nf, tf, qf = na.astype(np.float64), np.abs(tr).astype(np.float64), np.abs(q).astype(np.float64)
    aGa, aGHa = np.abs(Ga).astype(np.float64), np.abs(GHa).astype(np.float64)
    ba = C_G * (gamma(D) * (Tp * (aGa + aGHa) + tf * (Gp + GHp)) / nf
                + 2 * aa * (gamma(D) * Tp * qf + tf * gamma(2 * D) * qp + 2 * gamma(D) * tf * qf) / nf ** 2) \
        + 4 * U * np.abs(ga).astype(np.float64)
    bC = np.einsum('n,ij->nij', (C_G * (gamma(2 * D) * qp + gamma(D) * qf) / nf)[:, 0], np.eye(D))
    return ga, gC, ba, bC


def matvec_grad_ref(M, x, g):
    """(grad M*, grad x*, bound M, bound x) elementwise: g x^H (one complex product: C_G u |g_i| |x_j|) and M^H g
    (C_G gamma(D) sum_k |M_ki| |g_k|), in long double."""
    M = np.asarray(M, dtype=np.complex128)
    x = np.asarray(x, dtype=np.complex128)
    g = np.asarray(g, dtype=np.complex128)
    D = x.shape[-1]
    gM = np.einsum('ni,nj->nij', g.astype(CLD), x.astype(CLD).conj())
    gx = np.einsum('nki,nk->ni', M.astype(CLD).conj(), g.astype(CLD))
    bM = C_G * U * np.einsum('ni,nj->nij', np.abs(g), np.abs(x))
    bx = C_G * gamma(max(D, 2)) * np.einsum('nki,nk->ni', np.abs(M), np.abs(g))
    return gM, gx, bM, bx
