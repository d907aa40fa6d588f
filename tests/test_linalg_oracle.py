"""The float64 references of oracle/linalg_oracle.py pinned to the mpmath ones on well-conditioned inputs, and the
matrix generators checked against the spectra they promise."""
import numpy as np
import pytest

from oracle import linalg_oracle as L

EPS = np.finfo(np.float64).eps


@pytest.mark.parametrize('D', [1, 3, 8])
def test_eigh_matches_mpmath(D):
    pytest.importorskip('mpmath')
    rng = np.random.default_rng(D)
    a = L.spectrum_matrix('pd', D, rng)
    w, V = L.eigh(a)
    wm, Vm = L.mp_eigh(a)
    np.testing.assert_allclose(w, wm, rtol=0, atol=10 * D * EPS)
    # separated eigenvalues: the eigenvectors agree up to phase
    for i in range(D):
        assert abs(abs(np.vdot(V[:, i], Vm[:, i])) - 1) < 1e-12


def test_mp_eigvalsh_resolves_the_smallest_eigenvalues_of_steeply_graded_matrices():
    """With S = logspace(0, -12, D) the smallest eigenvalue is ~1e-25 of the largest.  mpmath's error is about
    10^-dps |A|, so 60 digits give it to full float64 precision (80 digits change nothing) and the kernel can be
    judged RELATIVE to it; a float64 reference only promises eps |A|."""
    pytest.importorskip('mpmath')
    rng = np.random.default_rng(5)
    a = L.graded(8, rng, decades=12.0)
    w = L.mp_eigvalsh(a, dps=60)
    assert np.all(w > 0) and w[0] < 1e-22 * w[-1]
    np.testing.assert_array_equal(L.mp_eigvalsh(a, dps=80), w)
    np.testing.assert_allclose(np.linalg.eigvalsh(a), w, rtol=0, atol=10 * 8 * EPS * w[-1])


@pytest.mark.parametrize('D', [1, 4, 9])
def test_solve_matches_mpmath(D):
    pytest.importorskip('mpmath')
    rng = np.random.default_rng(10 + D)
    a = L.conditioned(D, 10.0, rng)
    b = rng.standard_normal((D, 2)) + 1j * rng.standard_normal((D, 2))
    np.testing.assert_allclose(L.stable_solve(a, b), L.mp_solve(a, b), rtol=0, atol=100 * D * EPS * np.abs(b).max())


def test_gev_is_normalised_and_solves_the_pencil():
    rng = np.random.default_rng(2)
    D = 6
    a = L.spectrum_matrix('pd', D, rng)
    b = L.conditioned(D, 1e3, rng, hermitian=True)
    lam, W = L.gev(a, b)
    np.testing.assert_allclose(W.conj().T @ b @ W, np.eye(D), atol=1e-12)
    np.testing.assert_allclose(a @ W, b @ W * lam[None, :], atol=1e-12)
    w = L.gev_vector(a[None], b[None])[0]
    assert abs(abs(np.vdot(w, W[:, -1])) / (np.linalg.norm(w) * np.linalg.norm(W[:, -1])) - 1) < 1e-12


def test_stable_solve_falls_back_to_the_minimum_norm_solution():
    rng = np.random.default_rng(3)
    D = 5
    a = np.zeros((D, D), dtype=np.complex128)
    a[:3, :3] = L.spectrum_matrix('pd', 3, rng)
    b = rng.standard_normal((D, 1)) + 1j * rng.standard_normal((D, 1))
    x = L.stable_solve(a, b)
    np.testing.assert_allclose(x, np.linalg.pinv(a) @ b, atol=1e-12)
    assert np.all(x[3:] == 0)


@pytest.mark.parametrize('kind', L.SPECTRA)
@pytest.mark.parametrize('D', [1, 2, 7, 16])
def test_generators_have_the_promised_spectra(kind, D):
    rng = np.random.default_rng(D)
    a = L.spectrum_matrix(kind, D, rng)
    assert a.shape == (D, D) and a.dtype == np.complex128
    np.testing.assert_array_equal(a, a.conj().T)  # exactly Hermitian
    w = np.linalg.eigvalsh(a)
    scale = max(np.abs(w).max(), 1.0)
    tol = 10 * D * EPS * scale
    if kind == 'zero':
        assert np.all(a == 0)
    elif kind == 'identity':
        np.testing.assert_array_equal(a, np.eye(D))
    elif kind == 'rank1':
        np.testing.assert_allclose(w, np.r_[np.zeros(D - 1), 1.0], atol=tol)
    elif kind == 'rank_half':
        assert np.sum(np.abs(w) > 1e-3) == max(D // 2, 1)
    elif kind == 'pd':
        assert w[0] > 0.05
    elif kind == 'cluster':
        np.testing.assert_allclose(w, 1.0, atol=1e-10)
    elif kind == 'cond1e14':
        np.testing.assert_allclose(w, np.sort(np.logspace(0, -14, D)), atol=tol)
    elif kind == 'unsorted_diagonal':
        np.testing.assert_array_equal(np.sort(np.diag(a).real), np.linspace(-1.0, 2.0, D))
    elif kind == 'graded':
        assert w[0] > 0


def test_rank_one_estimate():
    rng = np.random.default_rng(4)
    v = rng.standard_normal((3, 4)) + 1j * rng.standard_normal((3, 4))
    cov = np.stack([L.spectrum_matrix('pd', 4, rng) for _ in range(3)])
    r = L.rank_one_estimate(v, cov)
    np.testing.assert_allclose(np.einsum('fdd->f', r), np.einsum('fdd->f', cov), rtol=1e-13)
    np.testing.assert_allclose(r @ v[..., None], v[..., None] * np.einsum('fdd->f', cov)[:, None, None], rtol=1e-12)
