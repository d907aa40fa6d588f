"""Multi-source beamformers (LCMV, WMWF, MERL MVDR), vector post-processing and time-varying beamforming on the
device against the fixture of the unmodified reference (oracle/make_golden_extraction.py), against the NumPy
restatement (oracle/extraction_oracle.py) and against invariants that do not depend on either."""
import numpy as np
import pytest
import torch

from conftest import cos_similarity, load_golden
from oracle import extraction_oracle as X
from oracle import pb_bss_oracle as O
from oracle import synth
from pb_bss_b200 import extraction as E

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-9, 1e-12


@pytest.fixture(scope='module')
def g():
    return load_golden('extraction')


def close(a, b, rtol=RTOL, atol=ATOL):
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def cplx(rng, *shape):
    return rng.randn(*shape) + 1j * rng.randn(*shape)


# ---- parity with the reference's fixture -----------------------------------------------------------------------

def test_lcmv_matches_reference(g):
    atf, noise = g['atf'], g['noise']
    close(E.get_lcmv_vector(atf, [1, 0, 0], noise), g['lcmv_onehot'])
    close(E.get_lcmv_vector(atf, [1, 1e-3, 1e-3], noise), g['lcmv_clipped'])
    close(E.get_lcmv_vector(atf, [0, 1, 0], g['noise_sing']), g['lcmv_sing'])   # zero bin: lstsq, complex64 y
    close(E.get_lcmv_vector(g['atf_kd'], [0, 0, 1, 0], noise), g['lcmv_kd'])


def test_wmwf_matches_reference(g):
    t, n = g['target'], g['noise']
    close(E.get_wmwf_vector(t, n, reference_channel=1), g['wmwf_ref1'])
    close(E.get_wmwf_vector(t, n), g['wmwf_auto'])
    close(E.get_wmwf_vector(t, n, reference_channel=2, distortion_weight=0.), g['wmwf_mu0'])
    close(E.get_wmwf_vector(t, n, distortion_weight=3.5), g['wmwf_mu3'])
    close(E.get_wmwf_vector(t, n, reference_channel=0, distortion_weight='frequency_dependent'), g['wmwf_fd'])
    close(E.get_wmwf_vector(t, n, distortion_weight='frequency_dependent'), g['wmwf_fd_auto'])
    close(E.get_wmwf_vector(t, n, channel_selection_vector=g['csv']), g['wmwf_csv'])


def test_merl_matches_reference(g):
    close(E.get_mvdr_vector_merl(g['target'], g['noise']), g['merl'])


def test_reference_channel_and_pca_match_reference(g):
    ch = E.get_optimal_reference_channel(g['w_mat'], g['target'], g['noise'])
    assert isinstance(ch, int) and ch == int(g['ref_channel'])
    vec, val = E.get_pca(g['target'])
    close(val, g['pca_val'])
    close(cos_similarity(vec, g['pca_vec']), 1, atol=1e-10)
    close(np.linalg.norm(vec, axis=-1), 1)
    vecs, vals = E.get_pca(g['target'], return_all_vecs=True)
    assert vecs.shape == g['pca_all_vecs'].shape and vals.shape == g['pca_all_vals'].shape
    close(vals, g['pca_all_vals'])
    close(cos_similarity(np.swapaxes(vecs, -1, -2), np.swapaxes(g['pca_all_vecs'], -1, -2)), 1, atol=1e-10)


def test_post_processing_matches_reference(g):
    vec, t, n = g['vec'], g['target'], g['noise']
    close(E.distortionless_normalization(vec, g['atf'][0], n), g['distortionless'])
    post = E.mvdr_snr_postfilter(vec, t, n)
    assert post.shape == (vec.shape[0], 1)
    close(post, g['snr_postfilter'])
    close(E.zero_degree_normalization(vec, 2), g['zero_degree_ref2'])
    close(E.condition_covariance(g['cc_x'], float(g['cc_gamma'])), g['condition_covariance'])


def test_phase_correction_matches_reference(g):
    """(F, D): the cumulative product runs over the bins.  (K, F, D): it runs over K (the reference's axis 0)."""
    vec = g['vec'].copy()
    close(E.phase_correction(vec), g['phase_fd'])
    np.testing.assert_array_equal(vec, g['vec'])             # the input is not modified
    close(E.phase_correction(g['vec_kfd']), g['phase_kfd'])
    close(E.phase_correction(list(g['vec'])), g['phase_fd'])  # array-likes, as np.array(vector) accepts them
    w = np.array([[1, 1], [-1, -1]], dtype=np.complex128)     # the reference's doctest
    close(E.phase_correction(w), [[1, 1], [1, 1]])
    close(E.phase_correction([w])[0], [[1, 1], [1, 1]])


def test_online_application_matches_reference(g):
    v, mix = g['online_vector'], g['online_mix']
    out = E.apply_online_beamforming_vector(v, mix)
    assert out.shape == g['online_c128'].shape
    close(out, g['online_c128'])
    close(E.apply_online_beamforming_vector(v, g['online_mix64']), g['online_c64'], rtol=1e-5, atol=1e-6)


def test_online_application_broadcast_and_sizes():
    """A mix broadcast over a leading dim (stride 0) is read in place; D beyond the register cache; both dtypes."""
    rng = np.random.RandomState(5)
    for T, F, D in ((500, 513, 8), (37, 5, 11), (3, 2, 1)):
        v = cplx(rng, T, F, D)
        mix = cplx(rng, F, D, T)
        ref = X.apply_online_beamforming_vector(v, mix)
        close(E.apply_online_beamforming_vector(v, mix), ref)
        m64 = mix.astype(np.complex64)
        close(E.apply_online_beamforming_vector(v, m64), X.apply_online_beamforming_vector(v, m64), rtol=1e-5,
              atol=1e-5)
        md = torch.from_numpy(m64).cuda().expand(3, F, D, T)
        assert md.stride(0) == 0
        out = E.apply_online_beamforming_vector(torch.from_numpy(v).cuda(), md)
        assert out.shape == (3, F, T)
        close(out.cpu().numpy(), np.broadcast_to(X.apply_online_beamforming_vector(v, m64), (3, F, T)), rtol=1e-5,
              atol=1e-5)
    # one vector bin broadcast over the bins of the mix, as the reference's einsum allows
    v = cplx(rng, 7, 1, 4)
    mix = cplx(rng, 2, 6, 4, 7)
    close(E.apply_online_beamforming_vector(v, mix), X.apply_online_beamforming_vector(v, mix))


# ---- invariants --------------------------------------------------------------------------------------------------

def test_invariants_at_full_size():
    F, D, K = 513, 8, 3
    rng = np.random.RandomState(11)
    noise = synth.pos_def_hermitian(F, D, D, seed=12)
    atf = cplx(rng, K, F, D)
    r = np.array([1, 1e-3, 1e-3])
    w = E.get_lcmv_vector(atf, r, noise)
    r32 = r.astype(np.complex64).astype(np.complex128)
    assert np.abs(np.einsum('kfd,fd->fk', atf.conj(), w) - r32).max() <= 1e-9 * np.linalg.norm(r)
    close(w, X.lcmv_vector(atf, r, noise), rtol=1e-8, atol=1e-12)
    vec = cplx(rng, F, D)
    # distortionless_normalization lies in the span of N w
    out = E.distortionless_normalization(vec, atf[0], noise)
    u = np.einsum('fab,fb->fa', noise, vec)
    proj = u * (np.einsum('fa,fa->f', u.conj(), out) / np.einsum('fa,fa->f', u.conj(), u))[:, None]
    close(out, proj, rtol=1e-10, atol=1e-12)
    # zero_degree_normalization: channel ref real and non-negative, moduli unchanged
    z = E.zero_degree_normalization(vec, 5)
    assert np.all(z[:, 5].real >= 0) and np.abs(z[:, 5].imag).max() <= 1e-15 * np.abs(z[:, 5]).max()
    close(np.abs(z), np.abs(vec), rtol=1e-13)
    # phase_correction keeps the moduli
    for v in (vec, cplx(rng, K, F, D)):
        np.testing.assert_allclose(np.abs(E.phase_correction(v)), np.abs(v), rtol=1e-12)
        close(E.phase_correction(v), X.phase_correction(v), rtol=1e-10)
    # MERL = WMWF with mu = 0 at channel 0; WMWF against the restatement
    t = synth.pos_def_hermitian(F, D, D, seed=13)
    close(E.get_mvdr_vector_merl(t, noise), E.get_wmwf_vector(t, noise, reference_channel=0, distortion_weight=0.),
          rtol=1e-12)
    close(E.get_wmwf_vector(t, noise), X.wmwf_vector(t, noise), rtol=1e-9)
    close(E.condition_covariance(t, 0.5), X.condition_covariance(t, 0.5), rtol=1e-13)


# ---- the reference's shape tests (tests/test_extraction/test_beamformer.py:25-118) -------------------------------

SHAPES = [pytest.param((3, 6, 6), id='TestBeamformerWrapper'),
          pytest.param((1, 6, 6), id='TestBeamformerWrapperWithoutIndependent'),
          pytest.param((2, 3, 6, 6), id='TestBeamformerWrapperWithSpeakers')]


@pytest.mark.parametrize('shape_psd', SHAPES)
def test_reference_shape_tests(shape_psd):
    K, F, D = 2, 3, 6
    shape_vector = shape_psd[:-1]
    rng = np.random.RandomState(0)
    pdh = lambda seed: synth.pos_def_hermitian(*shape_psd, seed=seed)  # noqa: E731
    assert E.get_gev_vector(pdh(1), pdh(2)).shape == shape_vector
    assert E.blind_analytic_normalization(E.get_gev_vector(pdh(1), pdh(2)), pdh(3)).shape == shape_vector
    if len(shape_psd) == 4:
        with pytest.raises(ValueError):
            E.get_mvdr_vector_souden(pdh(1), pdh(2))
    else:
        assert E.get_mvdr_vector_souden(pdh(1), pdh(2)).shape == shape_vector
    assert E.get_mvdr_vector_souden(pdh(1), pdh(2), ref_channel=1).shape == shape_vector
    assert E.get_wmwf_vector(pdh(1), pdh(2), reference_channel=1).shape == shape_vector
    assert E.get_wmwf_vector(pdh(1), pdh(2), reference_channel=1,
                             distortion_weight='frequency_dependent').shape == shape_vector
    u = cplx(rng, *shape_psd)
    assert E.get_pca_vector(u).shape == shape_vector
    assert E.get_pca_vector(u, 'trace').shape == shape_vector
    assert E.get_pca_vector(u, 'eigenvalue').shape == shape_vector
    assert E.get_mvdr_vector(cplx(rng, *shape_vector), u).shape == shape_vector
    assert E.get_lcmv_vector(cplx(rng, K, F, D), [1, 0], cplx(rng, F, D, D)).shape == (F, D)
    h = cplx(rng, 6, 6)
    h = h + h.conj().T
    close(cos_similarity(E.get_gev_vector(h, np.eye(6)), E.get_pca_vector(h)), 1.0, atol=1e-6)


# ---- a multi-source pipeline ---------------------------------------------------------------------------------------

def test_cacgmm_psd_pca_lcmv_pipeline():
    """cACGMM fit -> masked PSDs -> PCA ATFs of two sources -> LCMV per source with the third class as noise,
    against the NumPy pipeline.  PCA vectors have an arbitrary phase per bin; with a one-hot response it multiplies
    the LCMV vector, so that comparison is phase-free."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, D, K, I = 16, 300, 6, 3, 10
    y, _ = synth.structured_stft(F, T, D, K, seed=21)
    init = synth.init_affiliation(F, K, T, seed=22)
    Y = np.ascontiguousarray(y.transpose(0, 2, 1))
    aff = CACGMMTrainer().fit(y, initialization=init, iterations=I).predict(y)
    ref = O.cacgmm_fit(y, init, I)
    aff_ref = O.cacgmm_predict(y, ref)
    close(aff, aff_ref, rtol=1e-6, atol=1e-8)
    psd = E.get_power_spectral_density_matrix(Y, aff)
    psd_ref = O.power_spectral_density(Y, aff_ref)
    close(psd, psd_ref, rtol=1e-5, atol=1e-8)
    atf = np.stack([E.get_pca_vector(psd[:, k]) for k in range(2)])
    atf_ref = np.stack([np.linalg.eigh(psd_ref[:, k])[1][..., -1] for k in range(2)])
    for k in range(2):
        resp = np.eye(2)[k]
        w = E.get_lcmv_vector(atf, resp, psd[:, 2])
        w_ref = X.lcmv_vector(atf_ref, resp, psd_ref[:, 2])
        close(cos_similarity(w, w_ref), 1, atol=1e-6)
        close(np.linalg.norm(w, axis=-1), np.linalg.norm(w_ref, axis=-1), rtol=1e-5)
        close(np.einsum('kfd,fd->fk', atf.conj(), w), np.broadcast_to(resp, (F, 2)), atol=1e-9)


# ---- error types ---------------------------------------------------------------------------------------------------

def test_error_types():
    rng = np.random.RandomState(3)
    F, D = 4, 3
    t, n = synth.pos_def_hermitian(F, D, D, seed=1), synth.pos_def_hermitian(F, D, D, seed=2)
    with pytest.raises(ValueError):
        E.get_lcmv_vector(cplx(rng, F, D), [1], n)                   # atf not 3-D
    with pytest.raises(AssertionError):
        E.get_lcmv_vector(cplx(rng, 2, F, D), [1, 0], n[:, :2, :2])  # noise not (F, D, D)
    sing = n.copy()
    sing[1] = 0
    with pytest.raises(np.linalg.LinAlgError):
        E.get_mvdr_vector_merl(t, sing)
    with pytest.raises(ValueError):
        E.get_mvdr_vector_merl(t[None], n[None])
    with pytest.raises(ValueError):
        E.get_optimal_reference_channel(cplx(rng, 2, F, D, D), t, n)
    with pytest.raises(AssertionError):
        E.get_optimal_reference_channel(cplx(rng, F, D, D), t * np.inf, n)
    with pytest.raises(NotImplementedError, match='not yet thoroughly tested'):
        E.get_lcmv_vector_souden(t, t, n)
    with pytest.raises(TypeError):
        E.phase_correction(rng.randn(F, D))
    with pytest.raises(TypeError):
        E.phase_correction(torch.ones(F, D, dtype=torch.float64, device='cuda'))
    with pytest.raises(ValueError):
        E.apply_online_beamforming_vector(cplx(rng, 5, D), cplx(rng, F, D, 5))


# ---- CUDA tensors in give CUDA tensors out --------------------------------------------------------------------------

def test_cuda_tensors_in_cuda_tensors_out(g):
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    t, n, atf, vec = c(g['target']), c(g['noise']), c(g['atf']), c(g['vec'])
    outs = {
        'get_lcmv_vector': E.get_lcmv_vector(atf, c(np.array([1., 0, 0])), n),
        'get_wmwf_vector': E.get_wmwf_vector(t, n, reference_channel=1),
        'get_wmwf_vector auto': E.get_wmwf_vector(t, n),
        'get_wmwf_vector csv': E.get_wmwf_vector(t, n, channel_selection_vector=c(g['csv'])),
        'get_mvdr_vector_merl': E.get_mvdr_vector_merl(t, n),
        'get_pca': E.get_pca(t)[0],
        'get_pca values': E.get_pca(t)[1],
        'get_pca all': E.get_pca(t, return_all_vecs=True)[0],
        'condition_covariance': E.condition_covariance(c(g['cc_x']), 0.3),
        'distortionless_normalization': E.distortionless_normalization(vec, atf[0], n),
        'mvdr_snr_postfilter': E.mvdr_snr_postfilter(vec, t, n),
        'zero_degree_normalization': E.zero_degree_normalization(vec, 2),
        'phase_correction': E.phase_correction(c(g['vec_kfd'])),
        'apply_online_beamforming_vector': E.apply_online_beamforming_vector(c(g['online_vector']),
                                                                             c(g['online_mix64'])),
    }
    for name, o in outs.items():
        assert isinstance(o, torch.Tensor) and o.is_cuda, name
    close(outs['get_lcmv_vector'].cpu().numpy(), g['lcmv_onehot'])
    close(outs['phase_correction'].cpu().numpy(), g['phase_kfd'])
    assert E.get_optimal_reference_channel(c(g['w_mat']), t, n) == int(g['ref_channel'])
    # complex64 w_mat: eps is float32's tiny, as np.finfo(np.complex64).tiny
    assert E.get_optimal_reference_channel(c(g['w_mat'].astype(np.complex64)), t, n) == int(g['ref_channel'])
