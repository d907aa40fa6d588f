"""References and inputs for the EM kernels at the edges of their shape and number domains.

Builds on oracle/pb_bss_oracle.py (the float64 restatement of the reference) and adds:
- input generators whose fitted covariances land where the kernels switch code paths: ``graded_stft`` (every class
  of a bin shares a direction of relative power ~1/cond, so every class's scatter matrix has condition ~cond,
  whatever the affiliations) and ``extreme_stft`` (frames on one class's floor eigenvector and another's principal
  one, class weights down to 1e-12: a user model at the limits the product-form softmax is proved for) and
  ``separated_stft`` (classes in their own subspaces: fitted models that approach those limits);
- error scales from which the tests derive their tolerances instead of a flat rtol (``q_error_scale``,
  ``posterior_bound``);
- mpmath references (``mp_quadratic_form``, ``mp_log_det``, ``mp_cw_log_norm``, ``mp_cacg_m_step``) for the inputs
  where float64 cannot judge a kernel: ill-conditioned models, and the Watson normaliser, which the device
  computes by its own series / closed form.
"""
import math

import numpy as np

from . import linalg_oracle as _L
from . import pb_bss_oracle as _O

EPS = np.finfo(np.float64).eps
DPS = 40


# ---- inputs ----------------------------------------------------------------------------------------------------------
def graded_stft(F, T, D, K, cond, seed=0, rank=None, zero_frames=0):
    """Per bin a K-class complex Gaussian mixture (F, T, D) whose class covariances Q_k diag(lam) Q_k^H share one
    unitary's last D - r columns (r = D - 1, or ``rank``): those directions carry relative power 2^k/cond in class k (0 for
    ``rank``: the observations then span only r dimensions).  The first r eigenvalues of a class run over one
    decade in a class-specific rotation, so classes differ but every class scatter matrix -- for any affiliation --
    has lambda_min / lambda_max ~ 1/cond.  ``zero_frames``: that many all-zero frames at the start of every bin.
    Returns (y, labels)."""
    rng = np.random.default_rng(seed)
    r = D - 1 if rank is None else rank
    y = np.zeros((F, T, D), dtype=np.complex128)
    labels = rng.integers(0, K, size=(F, T))
    for f in range(F):
        Q = _L.unitary(D, rng)
        for k in range(K):
            U = Q[:, :r] @ _L.unitary(r, rng)
            n = int(np.sum(labels[f] == k))
            top = np.logspace(0, -1, r) if r > 1 else np.ones(r)
            x = (rng.standard_normal((n, r)) + 1j * rng.standard_normal((n, r))) * np.sqrt(top / 2)
            v = x @ U.T
            if rank is None:
                # class k: power 2^k / cond, so that flooring it or not changes the classes' q differently
                low = (rng.standard_normal((n, D - r)) + 1j * rng.standard_normal((n, D - r))) * np.sqrt(
                    2.0 ** k / (2 * cond))
                v = v + low @ Q[:, r:].T
            y[f, labels[f] == k] = v
        y[f] *= rng.uniform(0.5, 2.0, size=(T, 1))
    y[:, :zero_frames] = 0
    return y, labels


def extreme_model(F, D, K, floor, seed=0, min_weight=1e-12):
    """A cACGMM (dict of weight (F, K, 1), eigenvectors (F, K, D, D), eigenvalues (F, K, D)) at the limits of the
    product-form softmax: class 0 has eigenvalues floor..1 (log det = (D-1) log10 floor decades), class 1's
    principal eigenvector is class 0's floor eigenvector, the other classes are random; weights fall geometrically
    to ``min_weight``."""
    rng = np.random.default_rng(seed)
    V = np.empty((F, K, D, D), dtype=np.complex128)
    lam = np.empty((F, K, D))
    for f in range(F):
        Q = _L.unitary(D, rng)
        for k in range(K):
            if k == 0:
                V[f, k], lam[f, k] = Q, np.r_[floor, np.full(D - 2, floor), 1.0] if D > 2 else [floor, 1.0]
            elif k == 1:
                # principal eigenvector (last column) = class 0's floor eigenvector (first column)
                V[f, k], lam[f, k] = np.concatenate([Q[:, 1:], Q[:, :1]], axis=1), np.r_[np.full(D - 1, 0.1), 1.0]
            else:
                V[f, k], lam[f, k] = _L.unitary(D, rng), np.sort(rng.uniform(floor ** (1 / 3), 1.0, D))
                lam[f, k, -1] = 1.0
    w = np.logspace(0, np.log10(min_weight), K)
    w = np.broadcast_to(w / w.sum(), (F, K))[..., None].copy()
    return dict(weight=w, eigenvectors=V, eigenvalues=lam)


def extreme_stft(F, T, D, K, floor, seed=0, min_weight=1e-12):
    """Observations (F, T, D) for ``extreme_model(F, D, K, floor, seed, min_weight)``: a third of the frames on class
    0's floor eigenvector (q_0 = 1/floor), a third on its principal one, the rest complex Gaussian; tiny
    perturbations keep every frame off an exact eigenvector.  Returns (y, model)."""
    model = extreme_model(F, D, K, floor, seed, min_weight)
    rng = np.random.default_rng(seed + 1)
    y = (rng.standard_normal((F, T, D)) + 1j * rng.standard_normal((F, T, D))) / np.sqrt(2)
    a, b = T // 3, 2 * T // 3
    Q = model['eigenvectors'][:, 0]
    y[:, :a] = Q[:, None, :, 0] + 1e-3 * y[:, :a]
    y[:, a:b] = Q[:, None, :, -1] + 1e-3 * y[:, a:b]
    y *= rng.uniform(0.5, 2.0, size=(F, T, 1))
    return y, model


def separated_stft(F, T, D, K, seed=0):
    """Observations (F, T, D) whose classes each lie in their own random (D-1)-dimensional subspace (complex
    Gaussian inside it): as EM separates the classes, every fitted covariance gets an eigenvalue far below the others
    (down to the floor) and the frames of the other classes have a component along it, so q ratios and log-det spans
    grow towards the limits the product-form softmax is proved for (1e6 to 1e34 after five iterations from a 70 %
    correct start at D = 4..8).  Returns (y, labels)."""
    rng = np.random.default_rng(seed)
    y = np.empty((F, T, D), dtype=np.complex128)
    labels = rng.integers(0, K, size=(F, T))
    for f in range(F):
        for k in range(K):
            U = _L.unitary(D, rng)[:, :D - 1]
            n = int(np.sum(labels[f] == k))
            x = (rng.standard_normal((n, D - 1)) + 1j * rng.standard_normal((n, D - 1))) / np.sqrt(2)
            y[f, labels[f] == k] = x @ U.T
        y[f] *= rng.uniform(0.5, 2.0, size=(T, 1))
    return y, labels


# ---- error scales ----------------------------------------------------------------------------------------------------
def q_error_scale(y, model):
    """(F, K, T): z^H |B^-1| z with |.| taken element by element, B^-1 = V diag(1/lam) V^H, z the normalised frame.
    In the kernels' slot form this is sum_s |coef_s| |psi_s|: the scale of the rounding error of the quadratic form
    (each slot product is exact to eps, the sum is not), at least q itself and far above it where the terms cancel
    (ill-conditioned B)."""
    z = _O.normalize_observation_cacg(y)  # (F, D, T)
    Binv = np.einsum('fkde,fke,fkge->fkdg', model['eigenvectors'], 1 / model['eigenvalues'],
                     model['eigenvectors'].conj())
    az = np.abs(z)
    return np.einsum('fdt,fkdg,fgt->fkt', az, np.abs(Binv), az)


def posterior_bound(aff, q, dq, dld=0.0):
    """Bound on |d gamma| (F, K, T) from bounds dq on |d q| (F, K, T) and dld on |d log det| ((F, K) or scalar):
    |d lp_k| <= D |dq_k| / q_k + |d ld_k| (D absorbed into the caller's dq), |d gamma_k| <= 2 gamma_k (1 - gamma_k)
    max_j |d lp_j|."""
    dlp = dq / np.maximum(q, _O.TINY64) + np.broadcast_to(np.asarray(dld, dtype=float), q.shape[:2])[..., None]
    return 2 * aff * (1 - aff) * np.max(dlp, axis=-2, keepdims=True)


# ---- mpmath references -----------------------------------------------------------------------------------------------
def _mp():
    import mpmath
    return mpmath


def mp_quadratic_form(z, V, lam, dps=DPS):
    """z^H V diag(1/lam) V^H z for one class, z (D, N) normalised frames: (N,) at dps digits, rounded."""
    mp = _mp()
    with mp.workdps(dps):
        Vm = _L._to_mp(V)
        out = np.empty(z.shape[1])
        for t in range(z.shape[1]):
            zt = _L._to_mp(z[:, [t]])
            s = mp.mpf(0)
            for e in range(len(lam)):
                p = mp.fsum(mp.conj(Vm[d, e]) * zt[d] for d in range(len(lam)))
                s += (mp.re(p) ** 2 + mp.im(p) ** 2) / mp.mpf(float(lam[e]))
            out[t] = float(s)
    return out


def mp_log_det(lam, dps=DPS):
    """sum log lam at dps digits."""
    mp = _mp()
    with mp.workdps(dps):
        return float(mp.fsum(mp.log(mp.mpf(float(x))) for x in np.ravel(lam)))


def mp_cw_log_norm(kappa, D, dps=DPS):
    """log(1F1(1; D; kappa) 2 pi^D / (D-1)!), the complex Watson normaliser (complex_watson.py:157-168), for an array
    of kappa."""
    mp = _mp()
    kappa = np.asarray(kappa, dtype=float)
    out = np.empty(kappa.shape)
    with mp.workdps(dps):
        for i, k in np.ndenumerate(kappa):
            out[i] = float(mp.log(mp.hyp1f1(1, D, mp.mpf(float(k))) * 2 * mp.pi ** D / mp.factorial(D - 1)))
    return out


def cw_log_norm(kappa, D):
    """The oracle's normaliser: scipy (the reference's ``hyp1f1``) where its value is finite, mpmath elsewhere.
    Over D = 2..34 and kappa in [0, 500] scipy's log agrees with mpmath to 1e-13 (pinned in tests/test_em_oracle.py);
    beyond that range 1F1 overflows float64 first."""
    kappa = np.asarray(kappa, dtype=float)
    ref = np.array(_O.cw_log_norm(kappa, D), dtype=float)
    bad = ~np.isfinite(ref)
    if np.any(bad):
        ref = np.where(bad, 0.0, ref)
        ref[bad] = mp_cw_log_norm(kappa[bad], D)
    return ref


def mp_cacg_m_step(z, quadratic_form, affiliation, eigenvalue_floor=1e-10, dps=DPS):
    """One cACG M-step (cacg.py:253-342, covariance_norm='eigenvalue') of one bin at dps digits:
    z (D, N) normalised frames, quadratic_form / affiliation (K, N) -> floored eigenvalues (K, D), ascending, and
    the unfloored ones relative to lambda_max (K, D), both rounded to float64."""
    mp = _mp()
    D, N = z.shape
    K = affiliation.shape[0]
    lam_f = np.empty((K, D))
    lam_raw = np.empty((K, D))
    with mp.workdps(dps):
        zm = _L._to_mp(z)
        for k in range(K):
            S = mp.matrix(D, D)
            for t in range(N):
                c = mp.mpf(float(affiliation[k, t])) / mp.mpf(float(max(quadratic_form[k, t], 10 * _O.TINY64)))
                for d in range(D):
                    for e in range(D):
                        S[d, e] += c * zm[d, t] * mp.conj(zm[e, t])
            w, _ = mp.eighe(S)
            w = sorted(mp.re(x) for x in w)
            lam_raw[k] = [float(x / w[-1]) for x in w]
            lam_f[k] = np.maximum(lam_raw[k], eigenvalue_floor)
    return lam_f, lam_raw


# ---- the product-form softmax switches (api_cacgmm.cu) ---------------------------------------------------------------
def softmax_fast_ok(D, floor):
    """The per-iteration integer-power softmax: 2 D log10(1/floor) < 280 (eigenvalue norm, 0 < floor <= 1)."""
    return 0 < floor <= 1 and 2 * D * math.log10(1 / floor) < 280


def lean_ok(D, K, floor):
    """The persistent kernel's lean variant: softmax_fast_ok and (K - 1) D (log10(1/floor) + 1) < 290."""
    return softmax_fast_ok(D, floor) and (K - 1) * D * (math.log10(1 / floor) + 1) < 290


def lean_threshold(D, K):
    """The floor at which lean_ok switches: log10(1/floor) = 290 / ((K - 1) D) - 1 (capped by softmax_fast_ok)."""
    return 10.0 ** -min(290 / ((K - 1) * D) - 1, 140 / D)


def fast_threshold(D):
    """The floor at which softmax_fast_ok switches: log10(1/floor) = 140 / D."""
    return 10.0 ** -(140 / D)
