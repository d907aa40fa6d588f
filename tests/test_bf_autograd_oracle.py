"""The closed-form gradients of the get_bf_vector beamformers in oracle/autograd_oracle.py (GEV, PCA, MVDR, BAN, rank-1
estimate, matvec) against torch autograd of their pure-torch restatements, in complex128 at D = 1..8, and the
phase-held eigenvector derivative against mpmath central differences."""
import mpmath
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import bf_autograd_oracle as BO
from oracle import synth


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _t(a, grad=True):
    return torch.tensor(a, dtype=torch.complex128, requires_grad=grad)


def _close(got, ref, rel):
    """max error <= rel times the reference's largest entry, or times 1e-4 where the gradient vanishes analytically
    (the MVDR's noise gradient at D = 1) and both sides are rounding noise of O(1) inputs"""
    got, ref = got.detach(), ref.detach()
    assert torch.isfinite(got).all() and torch.isfinite(ref).all()
    err = (got - ref).abs().max().item()
    assert err <= rel * max(ref.abs().max().item(), 1e-4), (err, ref.abs().max().item())


def _hermitian_with_spectrum(rng, lam):
    """(n, D, D) Q diag(lam) Q^H with a random unitary Q per row of lam (n, D)."""
    n, D = lam.shape
    Q, _ = np.linalg.qr(_cplx(rng, n, D, D))
    return np.einsum('nij,nj,nkj->nik', Q, lam, Q.conj())


def _spectra(kind, n, D, rng):
    if kind == 'separated':
        return np.sort(rng.uniform(0.5, 5.0, (n, D)), -1) + np.arange(D) * 0.5
    if kind == 'rank1':
        lam = np.zeros((n, D))
        lam[:, -1] = rng.uniform(1.0, 3.0, n)
        return lam
    gap = float(kind)  # graded: the top two a relative gap apart, the rest below
    lam = np.sort(rng.uniform(0.1, 0.5, (n, D)), -1)
    lam[:, -1] = 1.0
    if D > 1:
        lam[:, -2] = 1.0 - gap
    return lam


KINDS = ['separated', '1e-1', '1e-4', '1e-8', 'rank1']


def _gap_rel(kind):
    return 1.0 if kind in ('separated', 'rank1') else float(kind)


@pytest.mark.parametrize('D', range(1, 9))
@pytest.mark.parametrize('kind', KINDS)
def test_pca_closed_form_matches_autograd(D, kind):
    rng = np.random.default_rng(100 + D)
    n = 6
    A = _t(_hermitian_with_spectrum(rng, _spectra(kind, n, D, rng)))
    val, w = BO.pca(A)
    g, gl = _t(_cplx(rng, n, D), False), torch.tensor(rng.standard_normal(n), dtype=torch.float64)
    (ref,) = torch.autograd.grad((w, val), A, (g, gl))
    got, _ = BO.eig_grad(A.detach(), None, w.detach(), g, gl)
    _close(got, ref, 1e-10 / _gap_rel(kind))


@pytest.mark.parametrize('D', range(1, 9))
@pytest.mark.parametrize('kind', KINDS)
def test_gev_closed_form_matches_autograd(D, kind):
    rng = np.random.default_rng(200 + D)
    n = 6
    B = _t(synth.pos_def_hermitian(n, D, D, seed=D) + 0.1 * np.eye(D))
    # target T = B^(1/2)-congruent to the chosen spectrum, so the pencil's eigenvalues are the spectrum
    L = np.linalg.cholesky(B.detach().numpy())
    C = _hermitian_with_spectrum(rng, _spectra(kind, n, D, rng))
    A = _t(L @ C @ L.conj().swapaxes(-1, -2))
    w, _ = BO.gev_vector(A, B)
    g = _t(_cplx(rng, n, D), False)
    ref = torch.autograd.grad(w, (A, B), g)
    got = BO.eig_grad(A.detach(), B.detach(), w.detach(), g)
    for a, b in zip(got, ref):
        _close(a, b, 1e-9 / _gap_rel(kind))


def test_rank1_targets_stay_finite():
    rng = np.random.default_rng(7)
    for D in (2, 5, 8):
        a = _cplx(rng, 4, D)
        A = _t(np.einsum('ni,nj->nij', a, a.conj()))
        B = _t(synth.pos_def_hermitian(4, D, D, seed=D) + 0.1 * np.eye(D))
        g = _t(_cplx(rng, 4, D), False)
        w, _ = BO.gev_vector(A, B)
        for x in BO.eig_grad(A.detach(), B.detach(), w.detach(), g):
            assert torch.isfinite(x).all()
        _, v = BO.pca(A)
        assert torch.isfinite(BO.eig_grad(A.detach(), None, v.detach(), g)[0]).all()


@pytest.mark.parametrize('D', range(1, 9))
def test_mvdr_ban_rank_one_matvec_closed_forms(D):
    rng = np.random.default_rng(300 + D)
    n = 5
    a = _t(_cplx(rng, n, D))
    N = _t(synth.pos_def_hermitian(n, D, D, seed=D) + 0.05 * np.eye(D) + 0.01 * _cplx(rng, n, D, D))
    g = _t(_cplx(rng, n, D), False)
    ref = torch.autograd.grad(BO.mvdr_vector(a, N), (a, N), g)
    for x, y in zip(BO.mvdr_grad(a.detach(), N.detach(), g), ref):
        _close(x, y, 1e-10)
    ref = torch.autograd.grad(BO.blind_analytic_normalization(a, N), (a, N), g)
    for x, y in zip(BO.ban_grad(a.detach(), N.detach(), g), ref):
        _close(x, y, 1e-10)
    C = _t(_cplx(rng, n, D, D))
    G = _t(_cplx(rng, n, D, D), False)
    ref = torch.autograd.grad(BO.rank_one_estimate(a, C), (a, C), G)
    for x, y in zip(BO.rank_one_grad(a.detach(), C.detach(), G), ref):
        _close(x, y, 1e-10)
    ref = torch.autograd.grad(BO.matvec(C, a), (C, a), g)
    for x, y in zip(BO.matvec_grad(C.detach(), a.detach(), g), ref):
        _close(x, y, 1e-12)


# ---- the phase-held convention, directly ------------------------------------------------------------------------

def _mp_top(A, B):
    """top eigenvector of the Hermitian pencil (A, B) in mpmath, w^H B w = 1 (B None: the identity)."""
    D = A.rows
    if B is None:
        E, Q = mpmath.eighe(A)
        j = max(range(D), key=lambda i: E[i])
        return Q[:, j]
    L = mpmath.cholesky(B)
    Li = mpmath.inverse(L)
    C = Li * A * Li.transpose_conj()
    C = (C + C.transpose_conj()) / 2
    E, Y = mpmath.eighe(C)
    j = max(range(D), key=lambda i: E[i])
    return Li.transpose_conj() * Y[:, j]


def _mp(M):
    return mpmath.matrix(M.tolist())


@pytest.mark.parametrize('D, pencil', [(2, False), (3, False), (4, False), (2, True), (3, True), (4, True)])
def test_phase_held_derivative_matches_mpmath_central_differences(D, pencil):
    """phi(eps) = w(A + eps E, B + eps F) conj(p) / |p|, p = w0^H B(eps) w(eps), keeps Im(w0^H B phi) = 0; its
    derivative at 0 against the closed form: Re<g, phi'(0)> = Re<grad A, E> + Re<grad B, F>."""
    mpmath.mp.dps = 50
    rng = np.random.default_rng(400 + D + 10 * pencil)
    A = synth.pos_def_hermitian(1, D, D, seed=D)[0]
    B = synth.pos_def_hermitian(1, D, D, seed=D + 50)[0] + 0.2 * np.eye(D) if pencil else None
    E = _cplx(rng, D, D)
    F = _cplx(rng, D, D) if pencil else None
    herm = lambda M: (M + M.conj().T) / 2  # noqa: E731
    eps = mpmath.mpf('1e-20')
    w0 = _mp_top(_mp(herm(A)), None if B is None else _mp(herm(B)))

    def phi(s):
        As = _mp(herm(A)) + s * _mp(herm(E))
        Bs = None if B is None else _mp(herm(B)) + s * _mp(herm(F))
        w = _mp_top(As, Bs)
        p = (w0.transpose_conj() * (w if Bs is None else Bs * w))[0]
        return w * mpmath.conj(p) / abs(p)

    dphi = (phi(eps) - phi(-eps)) / (2 * eps)
    dphi = np.array([complex(dphi[i]) for i in range(D)])
    g = _cplx(rng, D)
    w0n = np.array([complex(w0[i]) for i in range(D)])
    tA = torch.from_numpy(A[None])
    gA, gB = BO.eig_grad(tA, None if B is None else torch.from_numpy(B[None]), torch.from_numpy(w0n[None]),
                         torch.from_numpy(g[None]))
    lhs = np.real(np.vdot(g, dphi))
    rhs = np.real(np.vdot(gA[0].numpy(), E)) + (np.real(np.vdot(gB[0].numpy(), F)) if pencil else 0.0)
    assert abs(lhs - rhs) <= 1e-10 * (abs(lhs) + np.abs(gA[0].numpy()).sum() * np.abs(E).max()), (lhs, rhs)


# ---- the long-double references agree with the closed forms -----------------------------------------------------

def test_long_double_references_match_closed_forms():
    rng = np.random.default_rng(500)
    n, D = 7, 5
    A = synth.pos_def_hermitian(n, D, D, seed=1)
    B = synth.pos_def_hermitian(n, D, D, seed=2) + 0.1 * np.eye(D)
    g = _cplx(rng, n, D)
    w, _ = BO.gev_vector(torch.from_numpy(A), torch.from_numpy(B))
    gA, gB = BO.eig_grad(torch.from_numpy(A), torch.from_numpy(B), w, torch.from_numpy(g))
    rA, rB, bA, bB = BO.eig_grad_ref(A, B, w.numpy(), g)
    assert np.all(BO.normwise_ratio(gA.numpy(), rA, bA) <= 1) and np.all(BO.normwise_ratio(gB.numpy(), rB, bB) <= 1)
    gl = rng.standard_normal(n)
    _, v = BO.pca(torch.from_numpy(A))
    gA, _ = BO.eig_grad(torch.from_numpy(A), None, v, torch.from_numpy(g), torch.from_numpy(gl))
    rA, _, bA, _ = BO.eig_grad_ref(A, None, v.numpy(), g, gl)
    assert np.all(BO.normwise_ratio(gA.numpy(), rA, bA) <= 1)
    a = _cplx(rng, n, D)
    ga, gN = BO.mvdr_grad(torch.from_numpy(a), torch.from_numpy(B), torch.from_numpy(g))
    ra, rN, ba, bN = BO.mvdr_grad_ref(a, B, g)
    assert np.all(BO.normwise_ratio(ga.numpy(), ra, ba) <= 1) and np.all(BO.normwise_ratio(gN.numpy(), rN, bN) <= 1)
    N = B + 0.1 * _cplx(rng, n, D, D)
    gw, gN = BO.ban_grad(torch.from_numpy(a), torch.from_numpy(N), torch.from_numpy(g))
    rw, rN, bw, bN = BO.ban_grad_ref(a, N, g)
    assert np.all(BO.normwise_ratio(gw.numpy(), rw, bw) <= 1) and np.all(BO.normwise_ratio(gN.numpy(), rN, bN) <= 1)
    G = _cplx(rng, n, D, D)
    ga, gC = BO.rank_one_grad(torch.from_numpy(a), torch.from_numpy(N), torch.from_numpy(G))
    ra, rC, ba, bC = BO.rank_one_grad_ref(a, N, G)
    assert np.all(AO._ratio(AO._err(ga.numpy(), ra), ba) <= 1) and np.all(AO._ratio(AO._err(gC.numpy(), rC), bC) <= 1)
    gM, gx = BO.matvec_grad(torch.from_numpy(N), torch.from_numpy(a), torch.from_numpy(g))
    rM, rx, bM, bx = BO.matvec_grad_ref(N, a, g)
    assert np.all(AO._ratio(AO._err(gM.numpy(), rM), bM) <= 1) and np.all(AO._ratio(AO._err(gx.numpy(), rx), bx) <= 1)
