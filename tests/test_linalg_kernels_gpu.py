"""The beamforming linear-algebra kernels against float64 and mpmath references (oracle/linalg_oracle.py): heig, GEV,
solve / stable_solve, the beamformers and post-processing built on them, the PSD and apply_beamforming_vector.

Eigen- and solve results are judged through norms scaled by D * eps (residual, orthonormality, backward error), not
entry by entry; eigenvectors through their projectors, where the eigenvalues are separated.  The sizes reach past the
paths of the kernels: the templated Jacobi (D <= 8) and the generic one, more than 32 lanes' worth of rows, both sides
of the minimum-norm fallback (D <= 40), the frame chunks of the PSD kernels and more than 65535 bins."""
import numpy as np
import pytest

from conftest import cos_similarity
from oracle import extraction_oracle as EO
from oracle import linalg_oracle as L

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
C = 20  # constant of the D * eps bounds


def _fro(a):
    return np.linalg.norm(a, axis=(-2, -1))


def _spec(a):
    return np.linalg.norm(a, ord=2, axis=(-2, -1))


def _batch(kinds, D, seed):
    rng = np.random.default_rng(seed)
    return np.stack([L.spectrum_matrix(k, D, rng) for k in kinds])


def _projector_distance(u, v):
    """|u u^H - v v^H|_F of unit vectors (..., D)."""
    return _fro(u[..., :, None] * u[..., None, :].conj() - v[..., :, None] * v[..., None, :].conj())


def _check_eigenpairs(A, w, V):
    n, D, _ = A.shape
    H = L.hermitian_part(A)
    nrm = _spec(H)
    assert np.all(np.diff(w, axis=-1) >= 0), 'eigenvalues not ascending'
    res = _fro(H @ V - V * w[:, None, :])
    assert np.all(res <= C * D * EPS * nrm), (res / np.maximum(nrm, 1e-300)).max()
    orth = _fro(V.conj().swapaxes(-1, -2) @ V - np.eye(D))
    assert np.all(orth <= C * D * EPS), orth.max()
    wr, Vr = np.linalg.eigh(H)
    assert np.all(np.abs(w - wr) <= C * D * EPS * nrm[:, None]), np.abs(w - wr).max()
    for i in range(D):
        others = np.delete(wr, i, axis=-1)
        gap = np.abs(others - wr[:, i:i + 1]).min(-1) if D > 1 else np.full(n, np.inf)
        bound = C * D * EPS * nrm / np.maximum(gap, 1e-300)
        sel = (bound < 1e-2) & (gap > 0)
        dist = _projector_distance(V[:, :, i], Vr[:, :, i])
        assert np.all(dist[sel] <= bound[sel] + 4 * D * EPS), (i, dist[sel].max())


# ---- heig ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', range(1, 65))
def test_heig_every_size_and_spectrum(D):
    from pb_bss_b200.extraction.linalg import eigh
    full = _batch([L.SPECTRA[i % len(L.SPECTRA)] for i in range(257)], D, seed=D)
    for n in (1, 3, 5, 257):
        A = full[-n:] if n < 257 else full
        w, V = eigh(A)
        assert w.shape == (n, D) and V.shape == (n, D, D)
        _check_eigenpairs(A, w, V)
    # an unsorted diagonal is already diagonal: its sorted diagonal comes back exactly, V is a permutation
    diag = _batch(['unsorted_diagonal'], D, seed=D)
    w, V = eigh(diag)
    np.testing.assert_array_equal(w[0], np.sort(np.diag(diag[0]).real))
    np.testing.assert_array_equal(np.sort(np.abs(V[0]), axis=0), np.r_[np.zeros((D - 1, D)), np.ones((1, D))])


@pytest.mark.parametrize('D', [1, 2, 5, 8, 9, 33, 64])
def test_heig_non_hermitian_input_is_its_hermitian_part(D):
    """(A + A^H) / 2 is what LAPACK's one-triangle read amounts to; the device result is bit for bit that of the
    Hermitian part."""
    from pb_bss_b200.extraction.linalg import eigh
    rng = np.random.default_rng(D)
    A = _batch(['pd', 'indefinite', 'rank_half'], D, seed=D)
    A = A + (rng.standard_normal(A.shape) + 1j * rng.standard_normal(A.shape))
    w, V = eigh(A)
    wh, Vh = eigh(L.hermitian_part(A))
    np.testing.assert_array_equal(w, wh)
    np.testing.assert_array_equal(V, Vh)
    _check_eigenpairs(A, w, V)


@pytest.mark.parametrize('D', [4, 8, 16, 32])
def test_heig_graded_matrices_to_high_relative_accuracy(D):
    """S H S with S = logspace(0, -12, D), H well conditioned: every eigenvalue, the smallest (~1e-25 of the largest)
    included, within 10 D eps RELATIVE of the 60-digit one -- what the relative Jacobi stopping rule
    |a_pq|^2 > eps^2 |a_pp a_qq| promises and what the E-step's 1 / lambda needs.  The grading is steep enough that
    an absolute rule (eps^2 max(a_pp^2, a_qq^2)) leaves off-diagonals behind that move the small eigenvalues by far
    more than that from D = 8 on; with 7 decades both rules would pass."""
    pytest.importorskip('mpmath')
    from pb_bss_b200.extraction.linalg import eigh
    rng = np.random.default_rng(100 + D)
    A = np.stack([L.graded(D, rng, decades=12.0) for _ in range(3 if D < 32 else 2)])
    w, _ = eigh(A)
    for i in range(A.shape[0]):
        ref = L.mp_eigvalsh(A[i], dps=60)
        rel = np.abs(w[i] - ref) / np.abs(ref)
        assert np.all(rel <= 10 * D * EPS), (i, rel.max() / (D * EPS), rel.argmax())


SCALES = [200, -200, 480, -480, 500, -500, 600, -600]


@pytest.mark.parametrize('D', [3, 8, 13, 40])
def test_heig_is_exact_under_power_of_two_scaling(D):
    """w(sA) = s w(A) and V(sA) = V(A) bit for bit for s = 2^k: at |s| ~ 1e154 the squares of the rotation test
    overflow, at ~1e-150 they underflow, unless the kernel scales the matrix itself."""
    from pb_bss_b200.extraction.linalg import eigh
    A = _batch([k for k in L.SPECTRA if k != 'graded'], D, seed=7 + D)
    w, V = eigh(A)
    for k in SCALES:
        ws, Vs = eigh(A * 2.0 ** k)
        np.testing.assert_array_equal(ws, w * 2.0 ** k, err_msg=f'k = {k}')
        np.testing.assert_array_equal(Vs, V, err_msg=f'k = {k}')


def test_heig_reports_the_first_bad_matrix():
    from pb_bss_b200.extraction.linalg import eigh
    for D in (4, 40):
        A = _batch(['pd'] * 10, D, seed=1)
        A[3, 0, 1] = np.nan
        A[7, 1, 1] = np.inf
        with pytest.raises(np.linalg.LinAlgError, match=r'matrix 3$'):
            eigh(A)


# ---- gev -------------------------------------------------------------------------------------------------------------
CONDS = [1.0, 1e4, 1e8, 1e12]


@pytest.mark.parametrize('D', range(1, 65))
def test_gev_every_size_and_noise_conditioning(D):
    from pb_bss_b200.extraction import get_gev_vector
    rng = np.random.default_rng(D)
    n = 3
    for cond in CONDS:
        A = np.stack([L.spectrum_matrix('pd', D, rng) for _ in range(n)])
        B = np.stack([L.conditioned(D, cond, rng, hermitian=True) for _ in range(n)])
        kappa = np.linalg.cond(B)
        w = get_gev_vector(A, B)
        assert w.shape == (n, D)
        bwb = np.einsum('fa,fab,fb->f', w.conj(), B, w)
        tol = C * D * EPS * kappa
        assert np.all(np.abs(bwb - 1) <= tol), (cond, np.abs(bwb - 1).max())
        lam = np.einsum('fa,fab,fb->f', w.conj(), A, w).real / bwb.real
        res = np.linalg.norm(np.einsum('fab,fb->fa', A, w) - lam[:, None] * np.einsum('fab,fb->fa', B, w), axis=-1)
        scale = (_spec(A) + np.abs(lam) * _spec(B)) * np.linalg.norm(w, axis=-1)
        assert np.all(res <= tol * scale), (cond, (res / scale).max())
        if cond > 1e8:
            continue  # there the eps * kappa(B) bounds of the Cholesky reduction (which LAPACK shares) say little
        for f in range(n):
            lr, Wr = L.gev(A[f], B[f])
            ref = Wr[:, -1]
            relgap = (lr[-1] - lr[-2]) / abs(lr[-1]) if D > 1 else np.inf
            dist = _projector_distance(w[f] / np.linalg.norm(w[f]), ref / np.linalg.norm(ref))
            assert dist <= 100 * D * EPS * kappa[f] / relgap + 1e-13, (cond, f, dist)


@pytest.mark.parametrize('D', [3, 8, 13, 40])
def test_gev_is_exact_under_power_of_two_scaling(D):
    """Target scaled by 2^k, noise by 2^j (j even): the same direction, normalised to w^H B w = 1, so the vector is
    exactly 2^(-j/2) times the unscaled one."""
    from pb_bss_b200.extraction import get_gev_vector
    rng = np.random.default_rng(D)
    A = np.stack([L.spectrum_matrix('pd', D, rng) for _ in range(3)])
    B = np.stack([L.conditioned(D, 1e3, rng, hermitian=True) for _ in range(3)])
    w = get_gev_vector(A, B)
    for k, j in [(600, 0), (0, 600), (-600, 0), (0, -600), (-600, -600), (500, -500), (-480, 480), (200, -200)]:
        ws = get_gev_vector(A * 2.0 ** k, B * 2.0 ** j)
        np.testing.assert_array_equal(ws, w * 2.0 ** (-j // 2), err_msg=f'k = {k}, j = {j}')


def test_gev_rejects_non_pd_noise_and_names_the_first_bad_bin():
    """The reference loops over the bins and raises at the first one whose noise matrix is not positive definite
    (beamformer.py:395-409)."""
    from pb_bss_b200.extraction import get_gev_vector
    for D in (4, 40):
        A = _batch(['pd'] * 10, D, seed=2)
        B = _batch(['pd'] * 10, D, seed=3)
        B[3] = -B[3]
        with pytest.raises(ValueError, match=r'frequency 3:'):
            get_gev_vector(A, B)
        B[7] = L.spectrum_matrix('indefinite', D, np.random.default_rng(0))
        with pytest.raises(ValueError, match=r'frequency 3:'):
            get_gev_vector(A, B)


# ---- solve / stable_solve --------------------------------------------------------------------------------------------
SOLVE_D = [1, 2, 8, 9, 31, 32, 33, 40, 41, 64]


@pytest.mark.parametrize('D', SOLVE_D)
@pytest.mark.parametrize('R', ['1', 'D', '64'])
def test_solve_backward_error(D, R):
    from pb_bss_b200.extraction.linalg import stable_solve
    R = {'1': 1, 'D': D, '64': 64}[R]
    rng = np.random.default_rng(D * 100 + R)
    for cond in CONDS:
        A = np.stack([L.conditioned(D, cond, rng) for _ in range(3)])
        B = rng.standard_normal((3, D, R)) + 1j * rng.standard_normal((3, D, R))
        X = stable_solve(A, B)
        back = _fro(A @ X - B) / (_fro(A) * _fro(X))
        assert np.all(back <= C * D * EPS), (cond, back.max())
        ref = np.linalg.solve(A, B)
        fwd = _fro(X - ref) / _fro(ref)
        assert np.all(fwd <= C * D * EPS * cond), (cond, fwd.max())


def _singular_hermitian(D, rng):
    """Hermitian PSD with exactly zero rows and columns (rank D / 2, symmetrically permuted): elimination meets an
    exactly zero pivot."""
    r = max(D // 2, 1)
    A = np.zeros((D, D), dtype=np.complex128)
    A[:r, :r] = L.spectrum_matrix('pd', r, rng)
    p = rng.permutation(D)
    return A[np.ix_(p, p)]


@pytest.mark.parametrize('D', [2, 9, 33, 40])
def test_stable_solve_singular_gives_the_minimum_norm_solution(D):
    from pb_bss_b200.extraction.linalg import stable_solve
    rng = np.random.default_rng(D)
    A = np.stack([_singular_hermitian(D, rng) for _ in range(3)] + [np.zeros((D, D), dtype=np.complex128)])
    B = rng.standard_normal((4, D, 2)) + 1j * rng.standard_normal((4, D, 2))
    X = stable_solve(A, B)
    for i in range(4):
        ref = np.linalg.lstsq(A[i], B[i], rcond=None)[0]
        np.testing.assert_allclose(X[i], ref, rtol=0, atol=1e-10 * max(np.abs(ref).max(), 1e-300), err_msg=f'{i}')


def test_stable_solve_singular_past_the_fallback_raises():
    from pb_bss_b200.extraction.linalg import stable_solve
    rng = np.random.default_rng(41)
    A = np.stack([L.conditioned(41, 10.0, rng), _singular_hermitian(41, rng)])
    B = rng.standard_normal((2, 41, 1)) + 0j
    with pytest.raises(np.linalg.LinAlgError, match='singular matrix 1'):
        stable_solve(A, B)


@pytest.mark.parametrize('D', [6, 9, 40])
def test_stable_solve_is_exact_under_power_of_two_scaling(D):
    """X(2^k A, B) = 2^-k X(A, B) bit for bit, for singular Hermitian systems (minimum-norm branch) and regular ones
    (elimination: cdiv squares the pivot)."""
    from pb_bss_b200.extraction.linalg import stable_solve
    rng = np.random.default_rng(D)
    A = np.stack([_singular_hermitian(D, rng), _singular_hermitian(D, rng), L.conditioned(D, 1e3, rng)])
    B = rng.standard_normal((3, D, 2)) + 1j * rng.standard_normal((3, D, 2))
    X = stable_solve(A, B)
    for k in SCALES:
        np.testing.assert_array_equal(stable_solve(A * 2.0 ** k, B), X * 2.0 ** -k, err_msg=f'k = {k}')


@pytest.mark.parametrize('D', [2, 9, 40, 41])
def test_solve_nan_in_nan_out(D):
    from pb_bss_b200.extraction.linalg import stable_solve
    rng = np.random.default_rng(D)
    A = np.stack([L.conditioned(D, 10.0, rng) for _ in range(3)])
    A[1, D - 1, 0] = np.nan
    B = rng.standard_normal((3, D, 1)) + 0j
    X = stable_solve(A, B)
    assert np.all(np.isnan(X[1]))
    np.testing.assert_allclose(X[[0, 2]], np.linalg.solve(A[[0, 2]], B[[0, 2]]), rtol=1e-10)


# ---- beamformers and post-processing ---------------------------------------------------------------------------------
BF_D = [1, 2, 9, 16, 33, 64]


def _close(got, ref, tol=1e-11):
    err = np.linalg.norm(np.asarray(got) - ref) / max(np.linalg.norm(ref), 1e-300)
    assert err <= tol, err


def _psds(D, F, seed):
    rng = np.random.default_rng(seed)
    target = np.stack([L.spectrum_matrix('pd', D, rng) for _ in range(F)])
    noise = np.stack([L.spectrum_matrix('pd', D, rng) for _ in range(F)])
    return target, noise, rng


@pytest.mark.parametrize('D', BF_D)
def test_mvdr_souden_ban_rank_one_match_the_oracle(D):
    from pb_bss_b200 import extraction as E
    from pb_bss_b200.extraction import beamformer_wrapper as W
    F = 7
    target, noise, rng = _psds(D, F, D)
    atf = rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D))
    w = E.get_mvdr_vector(atf, noise)
    _close(w, L.mvdr_vector(atf, noise))
    np.testing.assert_allclose(np.einsum('fd,fd->f', w.conj(), atf), 1, atol=1e-12)  # distortionless
    s, ch = E.get_mvdr_vector_souden(target, noise, return_ref_channel=True)
    s_ref, ch_ref = L.mvdr_vector_souden(target, noise)
    assert ch == ch_ref
    _close(s, s_ref)
    _close(E.blind_analytic_normalization(atf, noise), L.blind_analytic_normalization(atf, noise))
    _close(W._rank_one(atf, target), L.rank_one_estimate(atf, target))
    _close(W._matvec(noise, atf), np.einsum('fab,fb->fa', noise, atf))
    _close(W.get_pca_rank_one_estimate(target), L.rank_one_estimate(L.eigh(target)[1][..., -1], target), 1e-8)
    gev = L.gev_vector(target, noise)
    _close(W.get_gev_rank_one_estimate(target, noise),
           L.rank_one_estimate(np.einsum('fab,fb->fa', noise, gev), target), 1e-8)


@pytest.mark.parametrize('D', BF_D)
def test_lcmv_wmwf_merl_match_the_oracle(D):
    from pb_bss_b200 import extraction as E
    F = 7
    target, noise, rng = _psds(D, F, 50 + D)
    K = min(2, D)
    atf = rng.standard_normal((K, F, D)) + 1j * rng.standard_normal((K, F, D))
    response = np.r_[1.0, np.zeros(K - 1)]
    w = E.get_lcmv_vector(atf, response, noise)
    _close(w, EO.lcmv_vector(atf, response, noise))
    np.testing.assert_allclose(np.einsum('kfd,fd->kf', atf.conj(), w), np.broadcast_to(response[:, None], (K, F)),
                               atol=1e-10)
    for mu in (1.0, 0.0, 'frequency_dependent'):
        _close(E.get_wmwf_vector(target, noise, distortion_weight=mu), EO.wmwf_vector(target, noise,
                                                                                      distortion_weight=mu))
    merl = E.get_mvdr_vector_merl(target, noise)
    _close(merl, EO.mvdr_vector_merl(target, noise))
    np.testing.assert_allclose(merl, E.get_wmwf_vector(target, noise, reference_channel=0, distortion_weight=0.0),
                               rtol=1e-13, atol=1e-15)
    filt = EO.wmwf_filter(target, noise)
    assert E.get_optimal_reference_channel(filt, target, noise) == EO.optimal_reference_channel(filt, target, noise)


@pytest.mark.parametrize('D', BF_D)
def test_post_processing_matches_the_oracle(D):
    from pb_bss_b200 import extraction as E
    F = 7
    target, noise, rng = _psds(D, F, 90 + D)
    v = rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D))
    atf = rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D))
    _close(E.condition_covariance(target, 0.3), EO.condition_covariance(target, 0.3))
    _close(E.distortionless_normalization(v, atf, noise), EO.distortionless_normalization(v, atf, noise))
    _close(E.mvdr_snr_postfilter(v, target, noise), EO.mvdr_snr_postfilter(v, target, noise))
    _close(E.zero_degree_normalization(v, D - 1), EO.zero_degree_normalization(v, D - 1))
    _close(E.phase_correction(v), EO.phase_correction(v))


# ---- PSD -------------------------------------------------------------------------------------------------------------
PSD_T = [1, 31, 32, 33, 127, 128, 129]
PSD_K = [1, 2, 3, 4, 5, 19]


def _check_psd(got, ref):
    got = np.asarray(got)
    assert got.shape == ref.shape
    err = _fro(got - ref)
    assert np.all(err <= 1e-12 * _fro(ref)), (err / np.maximum(_fro(ref), 1e-300)).max()


def _obs(F, D, T, rng):
    return rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T))


@pytest.mark.parametrize('D', range(1, 35))
def test_psd_every_size_and_chunk_edge(D):
    """Every D < 35 with K up to 19 and T at the frame-chunk edges of the fast (32-frame) and generic (128-frame)
    kernels; mask None, normalize=False, a mask row summing to zero, complex64, permuted dims."""
    from pb_bss_b200.extraction import get_power_spectral_density_matrix as psd
    rng = np.random.default_rng(D)
    F = 2
    for T in PSD_T:
        Y = _obs(F, D, T, rng)
        for K in PSD_K:
            mask = rng.uniform(size=(F, K, T))
            _check_psd(psd(Y, mask), L.power_spectral_density(Y, mask))
        _check_psd(psd(Y), L.power_spectral_density(Y))
        mask = rng.uniform(size=(F, 3, T))
        mask[1, 2] = 0
        got = psd(Y, mask)
        _check_psd(got, L.power_spectral_density(Y, mask))
        assert np.all(got[1, 2] == 0)
        _check_psd(psd(Y, mask, normalize=False), L.power_spectral_density(Y, mask, normalize=False))
        _check_psd(psd(Y, mask[:, 0]), L.power_spectral_density(Y, mask[:, 0]))
        Y64 = Y.astype(np.complex64)
        _check_psd(psd(Y64, mask), L.power_spectral_density(Y64.astype(np.complex128), mask))
        # (F, T, D) observation with sensor_dim=-1, time_dim=-2; (F, T, K) mask with source_dim=-1, time_dim=-2
        got = psd(np.ascontiguousarray(Y.swapaxes(-1, -2)), np.ascontiguousarray(mask.swapaxes(-1, -2)),
                  sensor_dim=-1, source_dim=-1, time_dim=-2)
        _check_psd(got, L.power_spectral_density(Y, mask))


@pytest.mark.parametrize('D,K', [(1, 1), (4, 3), (6, 2), (8, 4), (13, 19), (34, 3)])
def test_psd_long_utterance(D, K):
    from pb_bss_b200.extraction import get_power_spectral_density_matrix as psd
    rng = np.random.default_rng(D)
    Y = _obs(2, D, 20000, rng)
    mask = rng.uniform(size=(2, K, 20000))
    _check_psd(psd(Y, mask), L.power_spectral_density(Y, mask))
    _check_psd(psd(Y), L.power_spectral_density(Y))


# ---- apply_beamforming_vector ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', range(1, 30))
def test_apply_beamforming_vector_every_size(D):
    from pb_bss_b200.extraction import apply_beamforming_vector as apply
    rng = np.random.default_rng(D)
    F = 3
    for T in (1, 255, 256, 257):
        mix = _obs(F, D, T, rng)
        v = rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D))
        _close(apply(v, mix), L.apply_beamforming_vector(v, mix), 1e-13)
        vk = rng.standard_normal((2, F, D)) + 1j * rng.standard_normal((2, F, D))  # shared mix, broadcast over 2
        _close(apply(vk, mix), L.apply_beamforming_vector(vk, mix), 1e-13)
        m64 = mix.astype(np.complex64)
        _close(apply(vk, m64), L.apply_beamforming_vector(vk, m64.astype(np.complex128)), 1e-13)


# ---- more than 65535 bins --------------------------------------------------------------------------------------------
def test_chain_past_65535_bins():
    """128 utterances x 513 bins = 65664 bins, D = 2, T = 8: PSD -> GEV -> BAN -> apply, every bin against the
    oracle (each stage fed the device result of the one before, so the GEV phase does not matter)."""
    from pb_bss_b200 import extraction as E
    rng = np.random.default_rng(0)
    shape = (128, 513, 2, 8)
    Y = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    mask = rng.uniform(size=(128, 513, 2, 8))
    psd = E.get_power_spectral_density_matrix(Y, mask)
    _check_psd(psd, L.power_spectral_density(Y, mask))
    _check_psd(E.get_power_spectral_density_matrix(Y), L.power_spectral_density(Y))
    target, noise = psd[..., 0, :, :], psd[..., 1, :, :]
    w = E.get_gev_vector(target, noise)
    ref = L.gev_vector(target, noise)
    assert np.all(cos_similarity(w, ref) >= 1 - 1e-10)
    np.testing.assert_allclose(np.einsum('...a,...ab,...b->...', w.conj(), noise, w).real, 1, rtol=1e-10)
    ban = E.blind_analytic_normalization(w, noise)
    np.testing.assert_allclose(ban, L.blind_analytic_normalization(w, noise), rtol=1e-12, atol=1e-14)
    out = E.apply_beamforming_vector(ban, Y)
    np.testing.assert_allclose(out, L.apply_beamforming_vector(ban, Y), rtol=1e-12, atol=1e-13)
    # two beamformers sharing the one mix (the shared path, 2 x 65664 bins)
    vk = np.stack([ban, w])
    out = E.apply_beamforming_vector(vk, Y)
    np.testing.assert_allclose(out, L.apply_beamforming_vector(vk, Y), rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize('D,K', [(4, 2), (8, 3)])
def test_psd_fast_kernel_past_65535_bins(D, K):
    """The templated M-step kernel (D in {4, 6, 8}, K in 2..4) over 128 x 513 = 65664 bins."""
    from pb_bss_b200.extraction import get_power_spectral_density_matrix as psd
    rng = np.random.default_rng(D)
    for T in (8, 40):
        Y = rng.standard_normal((128, 513, D, T)) + 1j * rng.standard_normal((128, 513, D, T))
        mask = rng.uniform(size=(128, 513, K, T))
        _check_psd(psd(Y, mask), L.power_spectral_density(Y, mask))


def test_heig_gev_solve_past_65535_matrices():
    from pb_bss_b200.extraction import get_gev_vector
    from pb_bss_b200.extraction.linalg import eigh, stable_solve
    rng = np.random.default_rng(1)
    n, D = 70000, 2
    z = rng.standard_normal((n, D, 4)) + 1j * rng.standard_normal((n, D, 4))
    A = z @ z.conj().swapaxes(-1, -2)
    z = rng.standard_normal((n, D, 4)) + 1j * rng.standard_normal((n, D, 4))
    B = z @ z.conj().swapaxes(-1, -2)
    w, V = eigh(A)
    _check_eigenpairs(A, w, V)
    g = get_gev_vector(A, B)
    ref = L.gev_vector(A, B)
    assert np.all(cos_similarity(g, ref) >= 1 - 1e-9)
    rhs = rng.standard_normal((n, D, 1)) + 0j
    X = stable_solve(B, rhs)
    assert np.all(_fro(B @ X - rhs) <= C * D * EPS * _fro(B) * _fro(X))
