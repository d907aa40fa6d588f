"""References for the beamforming linear algebra (heig, GEV, solve and what is built on them).

Two levels:
- float64, matrix by matrix: LAPACK through NumPy / SciPy.  The beamformer references already live in
  oracle/pb_bss_oracle.py and oracle/extraction_oracle.py and are re-exported here under one roof.
- high precision: mpmath at ``DPS`` decimal digits (``mp.eighe``, ``mp.lu_solve``), for the inputs where a float64
  reference, accurate to eps |A| only, cannot judge a kernel: the smallest eigenvalues of graded matrices.  mpmath's
  own error is about 10^-dps |A|; steeply graded matrices need more than the default digits.

The matrix generators build Q diag(lambda) Q^H with a Haar-random unitary Q, so the spectrum is known up to the
rounding of the product; graded() builds S H S with S = logspace(0, -decades, D) and H well conditioned, where
Jacobi with the relative stopping rule |a_pq|^2 > eps^2 |a_pp a_qq| is accurate to a few ulps in EVERY eigenvalue,
and an absolute rule is not once the grading is steep (12 decades).
"""
import numpy as np
import scipy.linalg

from . import extraction_oracle as _E
from . import pb_bss_oracle as _O

DPS = 40

# float64 beamformer references (one copy each, in the modules they were written for)
power_spectral_density = _O.power_spectral_density
mvdr_vector = _O.mvdr_vector
gev_vector = _O.gev_vector
mvdr_vector_souden = _O.mvdr_vector_souden
blind_analytic_normalization = _O.blind_analytic_normalization
apply_beamforming_vector = _O.apply_beamforming_vector
stable_solve = _E.stable_solve


def hermitian_part(a):
    return 0.5 * (a + np.conj(np.swapaxes(a, -1, -2)))


def eigh(a):
    """np.linalg.eigh of the Hermitian part, (w ascending, V columns), per matrix."""
    return np.linalg.eigh(hermitian_part(np.asarray(a, dtype=np.complex128)))


def gev(a, b):
    """All generalised eigenpairs of one pair through scipy.linalg.eigh(a, b) (LAPACK zhegvd, ITYPE = 1):
    ascending eigenvalues and eigenvectors normalised to w^H b w = 1."""
    return scipy.linalg.eigh(hermitian_part(a), hermitian_part(b))


def rank_one_estimate(vector, covariance):
    """a a^H trace(cov) / trace(a a^H) (beamformer_wrapper.py:11-69)."""
    tr = np.einsum('...dd->...', covariance)
    outer = vector[..., :, None] * vector[..., None, :].conj()
    return outer * (tr / np.einsum('...d,...d->...', vector, vector.conj()).real)[..., None, None]


# ---- high precision ------------------------------------------------------------------------------------------------
def _mp():
    import mpmath
    return mpmath


def _to_mp(a):
    mp = _mp()
    a = np.asarray(a)
    return mp.matrix([[mp.mpc(complex(a[i, j])) for j in range(a.shape[1])] for i in range(a.shape[0])])


def mp_eigvalsh(a, dps=DPS):
    """Eigenvalues (ascending, as float64) of the Hermitian part of one matrix, at dps digits."""
    mp = _mp()
    with mp.workdps(dps):
        w, _ = mp.eighe(_to_mp(hermitian_part(np.asarray(a, dtype=np.complex128))))
        return np.sort(np.array([float(mp.re(x)) for x in w]))


def mp_eigh(a, dps=DPS):
    """(w ascending, V columns) of the Hermitian part of one matrix at dps digits, rounded to float64."""
    mp = _mp()
    with mp.workdps(dps):
        w, v = mp.eighe(_to_mp(hermitian_part(np.asarray(a, dtype=np.complex128))))
        w = np.array([float(mp.re(x)) for x in w])
        V = np.array([[complex(v[i, j]) for j in range(v.cols)] for i in range(v.rows)])
    order = np.argsort(w, kind='stable')
    return w[order], V[:, order]


def mp_solve(a, b, dps=DPS):
    """A^-1 B of one regular system at dps digits, rounded to complex128."""
    mp = _mp()
    b = np.asarray(b).reshape(a.shape[0], -1)
    with mp.workdps(dps):
        A = _to_mp(a)
        cols = [mp.lu_solve(A, _to_mp(b[:, [c]])) for c in range(b.shape[1])]
        return np.array([[complex(cols[c][i]) for c in range(b.shape[1])] for i in range(a.shape[0])])


# ---- matrices with known spectra -------------------------------------------------------------------------------------
def unitary(D, rng):
    """Haar-random unitary (QR of a complex Gaussian with the phases of R's diagonal divided out)."""
    z = (rng.standard_normal((D, D)) + 1j * rng.standard_normal((D, D))) / np.sqrt(2)
    q, r = np.linalg.qr(z)
    d = np.diagonal(r)
    return q * (d / np.abs(d))[None, :]


def from_spectrum(lam, rng):
    """Q diag(lam) Q^H, exactly Hermitian (the rounding of the product is symmetrised away)."""
    lam = np.asarray(lam, dtype=np.float64)
    Q = unitary(lam.size, rng)
    return hermitian_part((Q * lam[None, :]) @ Q.conj().T)


def graded(D, rng, decades=7.0, cond_h=10.0):
    """S H S, S = logspace(0, -decades, D), H Hermitian positive definite with condition cond_h."""
    s = np.logspace(0, -decades, D)
    H = from_spectrum(np.logspace(0, -np.log10(cond_h), D), rng)
    return hermitian_part(s[:, None] * H * s[None, :])


SPECTRA = ('pd', 'indefinite', 'rank1', 'rank_half', 'zero', 'identity', 'unsorted_diagonal', 'cluster',
           'cond1e14', 'cond1e16', 'graded')


def spectrum_matrix(kind, D, rng):
    """One D x D Hermitian test matrix of the named kind (SPECTRA)."""
    if kind == 'pd':
        return from_spectrum(rng.uniform(0.1, 1.0, D), rng)
    if kind == 'indefinite':
        return from_spectrum(rng.uniform(-1.0, 1.0, D), rng)
    if kind == 'rank1':
        return from_spectrum(np.r_[1.0, np.zeros(D - 1)], rng)
    if kind == 'rank_half':
        r = max(D // 2, 1)
        return from_spectrum(np.r_[rng.uniform(0.5, 1.0, r), np.zeros(D - r)], rng)
    if kind == 'zero':
        return np.zeros((D, D), dtype=np.complex128)
    if kind == 'identity':
        return np.eye(D, dtype=np.complex128)
    if kind == 'unsorted_diagonal':
        return np.diag(rng.permutation(np.linspace(-1.0, 2.0, D))).astype(np.complex128)
    if kind == 'cluster':
        return from_spectrum(1.0 + 1e-12 * rng.standard_normal(D), rng)
    if kind == 'cond1e14':
        return from_spectrum(np.logspace(0, -14, D), rng)
    if kind == 'cond1e16':
        return from_spectrum(np.logspace(0, -16, D), rng)
    if kind == 'graded':
        return graded(D, rng)
    raise ValueError(kind)


def conditioned(D, cond, rng, hermitian=False):
    """U diag(logspace(0, -log10 cond, D)) V^H (V = U for hermitian=True: positive definite)."""
    s = np.logspace(0, -np.log10(cond), D) if D > 1 else np.ones(1)
    U = unitary(D, rng)
    if hermitian:
        return hermitian_part((U * s[None, :]) @ U.conj().T)
    return (U * s[None, :]) @ unitary(D, rng).conj().T
