"""The gradients of WPE (pb_bss_b200.wpe: wpe_step, wpe, get_power, get_power_inverse) three ways: a torch
restatement whose own autograd gives the reference gradients, the closed forms of include/pbb.h in NumPy, and those
closed forms in long double (np.clongdouble, with a hand-written LU since NumPy's linalg has no long double).

The contract of wpe_step, for Y (..., D, T) complex and w (..., T) real, every leading index an independent problem
and n = taps D:
  Yt = build_y_tilde(Y, taps, delay) (row k D + d at frame t is Y_{d, t - delay - k}, 0 before frame 0),
  R = sum_S w_t Yt_t Yt_t^H, P = sum_S w_t Yt_t Y_t^H, G = stable_solve(R, P), X = Y - G^H Yt,
with S every frame ('full') or t >= delay + taps - 1 ('valid').  This is the computation of nara_wpe's TensorFlow
wpe_step and ESPnet's wpe_one_iteration given the inverse power w, restated here, not copied; an empty S gives
R = P = 0 for every input and so G = 0, a constant.  wpe (oracle/wpe_oracle.py) is X = Y and `iterations` times
w = 1 / max(lambda_c, 1e-10 max_t lambda_c) per bin, X = wpe_step(Y, w).

Error bounds of the long-double comparison (grad_bound): one stage's gradient goes through one solve with R, whose
relative error is at most about n kappa(R) u (u = 2^-53, kappa the 1-norm condition number of R), and the O(n D T)
sums around it add n T u relative to the magnitudes summed.  Per bin the bound is
    |g_dev - g_ref| <= 64 (n sum_i kappa(R_i) + n T) u S + r sqrt(2) 2^-24 max|g_ref|,
sum_i over the iterations (each stage's solve feeds the next stage's incoming gradient), r the roundings to complex64
/ float32 on the way out (one for a returned gradient, more where autograd sums several in single precision; a
complex rounding moves a value by up to sqrt(2) 2^-24 of its modulus).  S is the larger of max|g_ref| and
the magnitude of the terms the gradient sums: max|xbar| for Y's gradient (ybar = xbar + ...), max|xbar| / min w for
the weights' (c_t carries R^-1 ~ 1 / w).  The terms matter where they cancel: with delay = 0 the current frame is
among the regressors, X is rounding residue and its exact gradient is 0.  For the per-bin max of the weights
only its value and the tie pattern enter, and both are reproduced exactly (the device recomputes lambda_c with the
forward's kernel); the reference takes them from the float64 forward."""
import numpy as np
import torch

EPS_POWER = 1e-10
U = 2.0 ** -53
U32 = 2.0 ** -24


# ---- torch restatement (complex128) -------------------------------------------------------------------------------

def build_y_tilde(Y, taps, delay):
    T = Y.shape[-1]
    rows = []
    for k in range(taps):
        s = min(delay + k, T)
        z = torch.zeros(Y.shape[:-1] + (s,), dtype=Y.dtype, device=Y.device)
        rows.append(torch.cat([z, Y[..., :T - s]], -1))
    return torch.cat(rows, -2)


def _mask(T, taps, delay, statistics_mode, device=None):
    m = torch.ones(T, dtype=torch.float64, device=device)
    if statistics_mode == 'valid':
        m[:delay + taps - 1] = 0
    return m


def wpe_step(Y, w, taps, delay, statistics_mode='full'):
    """(X, G) of one WPE step with weights w (..., T) real."""
    T = Y.shape[-1]
    Yt = build_y_tilde(Y, taps, delay)
    m = _mask(T, taps, delay, statistics_mode, Y.device)
    if not m.any():
        return Y.clone(), torch.zeros(Y.shape[:-2] + (Yt.shape[-2], Y.shape[-2]), dtype=Y.dtype, device=Y.device)
    wm = (w * m).to(Y.dtype)[..., None, :]
    R = (Yt * wm) @ Yt.conj().transpose(-1, -2)
    P = (Yt * wm) @ Y.conj().transpose(-1, -2)
    G = torch.linalg.solve(R, P)
    return Y - G.conj().transpose(-1, -2) @ Yt, G


def window_mean(lam, c):
    """mean over the frames t - c .. t + c that exist (c None: inf)"""
    T = lam.shape[-1]
    if c is None:
        return lam.mean(-1, keepdim=True).expand(lam.shape)
    if c == 0:
        return lam
    cs = torch.cat([torch.zeros(lam.shape[:-1] + (1,), dtype=lam.dtype, device=lam.device), lam.cumsum(-1)], -1)
    t = torch.arange(T, device=lam.device)
    lo, hi = (t - c).clamp(min=0), (t + c).clamp(max=T - 1) + 1
    return (cs[..., hi] - cs[..., lo]) / (hi - lo).to(lam.dtype)


def _c(psd_context):
    return None if np.isposinf(psd_context) else int(psd_context)


def get_power(x, psd_context=0):
    return window_mean((x.abs() ** 2).mean(-2), _c(psd_context))


def get_power_inverse(x, psd_context=0):
    """the max over the whole array"""
    p = get_power(x, psd_context)
    return 1 / torch.maximum(p, EPS_POWER * p.amax())


def power_inverse_per_bin(x, psd_context=0):
    """wpe's weights: the max per bin"""
    p = get_power(x, psd_context)
    return 1 / torch.maximum(p, EPS_POWER * p.amax(-1, keepdim=True))


def wpe(Y, taps=10, delay=3, iterations=3, psd_context=0, statistics_mode='full'):
    X = Y
    for _ in range(iterations):
        X = wpe_step(Y, power_inverse_per_bin(X, psd_context), taps, delay, statistics_mode)[0]
    return X if iterations else Y.clone()


# ---- closed forms (NumPy; complex128 or clongdouble) --------------------------------------------------------------

def lu_solve(A, B):
    """A^-1 B by LU with partial pivoting (first maximum of |re| + |im|), any complex dtype; None on a zero pivot."""
    A, B = A.copy(), B.copy()
    n = A.shape[0]
    for j in range(n):
        mag = np.abs(A[j:, j].real) + np.abs(A[j:, j].imag)
        p = j + int(np.argmax(mag))
        if mag[p - j] == 0:
            return None
        if p != j:
            A[[j, p]] = A[[p, j]]
            B[[j, p]] = B[[p, j]]
        f = A[j + 1:, j] / A[j, j]
        A[j + 1:, j + 1:] -= f[:, None] * A[j, j + 1:][None, :]
        B[j + 1:] -= f[:, None] * B[j][None, :]
    for i in range(n - 1, -1, -1):
        B[i] = (B[i] - A[i, i + 1:] @ B[i + 1:]) / A[i, i]
    return B


def lstsq_solve(R, P):
    """np.linalg.lstsq's minimum-norm R^-1 P for an R whose singular part is exactly zero rows and columns (a dead
    channel of Y zeroes its taps rows of Yt, so those rows and columns of R and those rows of P are 0): the live
    block solved by lu_solve, zeros in the dead rows.  Any dtype, long double included."""
    live = np.flatnonzero(np.any(R != 0, axis=1))
    dead = np.setdiff1d(np.arange(R.shape[0]), live)
    assert not np.any(R[:, dead]) and not np.any(P[dead]), 'the singular part of R is not exactly zero rows'
    G = np.zeros(P.shape, np.result_type(R, P))
    if live.size:
        G[live] = lu_solve(R[np.ix_(live, live)], P[live])
    return G


def live_kappa(R):
    """kappa (1-norm) of the block of R that lstsq_solve solves"""
    live = np.flatnonzero(np.any(R != 0, axis=1))
    return kappa(R[np.ix_(live, live)])


def y_tilde(Y, taps, delay):
    D, T = Y.shape
    out = np.zeros((taps * D, T), dtype=Y.dtype)
    for k in range(taps):
        s = delay + k
        if s < T:
            out[k * D:(k + 1) * D, s:] = Y[:, :T - s]
    return out


def _m(T, taps, delay, statistics_mode):
    m = np.ones(T)
    if statistics_mode == 'valid':
        m[:delay + taps - 1] = 0
    return m


def step_forward(Y, w, taps, delay, statistics_mode='full'):
    """one bin: (X, G, R); G = 0 and R = 0 for an empty S; an exactly zero pivot takes lstsq_solve"""
    D, T = Y.shape
    Yt = y_tilde(Y, taps, delay)
    wm = w * _m(T, taps, delay, statistics_mode).astype(w.dtype)
    R = (Yt * wm) @ Yt.conj().T
    if not wm.any():
        return Y.copy(), np.zeros((taps * D, D), Y.dtype), R
    P = (Yt * wm) @ Y.conj().T
    G = lu_solve(R, P)
    if G is None:
        G = lstsq_solve(R, P)
    return Y - G.conj().T @ Yt, G, R


def step_backward(Y, w, G, R, xbar, taps, delay, statistics_mode='full'):
    """one bin: (ybar, wbar) of X = Y - G^H Yt given the incoming xbar (include/pbb.h):
    Gbar = -sum_t yt_t xbar_t^H, R Pbar = Gbar, c_t = m_t w_t Pbar^H yt_t, u = xbar + c, b_t = m_t w_t x_t,
    Ytbar_t = -G u_t + Pbar b_t, ybar_t = u_t + sum_k Ytbar_{kD+d, t+delay+k}, wbar_t = m_t Re(c'_t^H x_t) with
    c'_t = Pbar^H yt_t."""
    D, T = Y.shape
    m = _m(T, taps, delay, statistics_mode).astype(w.real.dtype)
    if not m.any():
        return xbar.copy(), np.zeros(T, w.dtype)
    Yt = y_tilde(Y, taps, delay)
    X = Y - G.conj().T @ Yt
    Pb = lu_solve(R, -Yt @ xbar.conj().T)
    cp = Pb.conj().T @ Yt
    u = xbar + cp * (m * w)
    b = X * (m * w)
    Ytb = -G @ u + Pb @ b
    ybar = u.copy()
    for k in range(taps):
        s = delay + k
        if s < T:
            ybar[:, :T - s] += Ytb[k * D:(k + 1) * D, s:]
    wbar = m * (cp.conj() * X).sum(0).real
    return ybar, wbar


def window_adjoint(g, c):
    """the adjoint of window_mean: sum over s with |s - t| <= c of g_s / n_s"""
    T = g.shape[-1]
    if c is None:
        return np.full_like(g, g.sum() / T)
    if c == 0:
        return g.copy()
    t = np.arange(T)
    n = np.minimum(t + c, T - 1) - np.maximum(t - c, 0) + 1
    q = g / n
    return np.array([q[max(0, s - c):s + c + 1].sum() for s in range(T)])


def _max_backward(lam_c, zbar, M):
    """(grad of lam_c, grad of M) of max(lam_c, EPS M) (torch.maximum: ties split evenly)"""
    e = EPS_POWER * M
    ga = np.where(lam_c > e, zbar, np.where(lam_c == e, zbar / 2, 0))
    gb = np.where(lam_c < e, zbar, np.where(lam_c == e, zbar / 2, 0))
    return ga, EPS_POWER * gb.sum()


def power_backward(x, gbar, psd_context, mode, lam_c=None):
    """xbar of the power chain for one bin (mode 'plain': gbar is lambda_c's gradient; 'inverse': w's, with the max
    per bin).  lam_c: the forward's lambda_c (default: recomputed in x's precision)."""
    D, T = x.shape
    c = _c(psd_context)
    if lam_c is None:
        lam = (np.abs(x) ** 2).mean(0)
        lam_c = lam if c == 0 else (np.full(T, lam.mean()) if c is None else
                                    np.array([lam[max(0, t - c):t + c + 1].mean() for t in range(T)]))
    if mode == 'inverse':
        M = lam_c.max()
        z = np.maximum(lam_c, EPS_POWER * M)
        ga, Mbar = _max_backward(lam_c, -gbar / z ** 2, M)
        ties = lam_c == M
        gbar = ga + ties * (Mbar / ties.sum())
    lb = window_adjoint(gbar, c)
    return (2.0 / D) * lb * x


def wpe_forward(Y, taps, delay, iterations, psd_context, statistics_mode, lam_cs=None):
    """one bin: (X, [(w_i, G_i, R_i, X_{i-1})])"""
    c = _c(psd_context)
    X, stages = Y, []
    for i in range(iterations):
        lam = (np.abs(X) ** 2).mean(0)
        T = lam.shape[0]
        lc = lam if c == 0 else (np.full(T, lam.mean()) if c is None else
                                 np.array([lam[max(0, t - c):t + c + 1].mean() for t in range(T)]))
        if lam_cs is not None:
            lc = lam_cs[i].astype(lc.dtype)
        w = 1 / np.maximum(lc, EPS_POWER * lc.max())
        Xn, G, R = step_forward(Y, w, taps, delay, statistics_mode)
        stages.append((w, G, R, X, lc))
        X = Xn
    return X, stages


def wpe_backward(Y, stages, xbar, taps, delay, psd_context, statistics_mode):
    """one bin: ybar of wpe, the stages from the last to the first"""
    ybar = np.zeros_like(Y)
    for i in range(len(stages) - 1, -1, -1):
        w, G, R, Xprev, lc = stages[i]
        yb, wb = step_backward(Y, w, G, R, xbar, taps, delay, statistics_mode)
        ybar += yb
        xb = power_backward(Xprev, wb, psd_context, 'inverse', lc)
        if i == 0:
            ybar += xb
        else:
            xbar = xb
    return ybar if stages else xbar.copy()


def kappa(R):
    """1-norm condition number (inf for a singular R; 1 for the R = 0 of an empty S, whose G = 0 is exact)"""
    if not np.any(R):
        return 1.0
    try:
        return np.linalg.cond(np.asarray(R, np.complex128), 1)
    except np.linalg.LinAlgError:
        return np.inf


def grad_bound(ref, kappas, n, T, roundings, terms=0.0):
    """the per-bin bound of the module docstring for a bin's reference gradient; roundings: to single precision on the
    way out; terms: the magnitude of the terms it sums"""
    top = float(np.max(np.abs(ref))) if ref.size else 0.0
    return 64 * (n * sum(kappas) + n * T) * U * max(top, float(terms)) + roundings * np.sqrt(2) * U32 * top
