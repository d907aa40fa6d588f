"""The NumPy restatement of the multi-source beamformers and vector post-processing (oracle/extraction_oracle.py)
against the fixture the unmodified reference wrote (oracle/make_golden_extraction.py).  CPU only."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import extraction_oracle as X


@pytest.fixture(scope='module')
def g():
    return load_golden('extraction')


def close(a, b):
    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-12)


def test_lcmv(g):
    atf, noise = g['atf'], g['noise']
    close(X.lcmv_vector(atf, [1, 0, 0], noise), g['lcmv_onehot'])
    close(X.lcmv_vector(atf, [1, 1e-3, 1e-3], noise), g['lcmv_clipped'])
    close(X.lcmv_vector(atf, [0, 1, 0], g['noise_sing']), g['lcmv_sing'])
    close(X.lcmv_vector(g['atf_kd'], [0, 0, 1, 0], noise), g['lcmv_kd'])
    # the response is met as complex64, the reference's cast (beamformer.py:444)
    resp = np.einsum('kfd,fd->fk', atf.conj(), g['lcmv_clipped'])
    np.testing.assert_allclose(resp[:, 1], np.float32(1e-3), rtol=0, atol=1e-12)
    assert np.all(np.abs(resp[:, 1] - 1e-3) > 1e-11)


def test_wmwf(g):
    t, n = g['target'], g['noise']
    close(X.wmwf_vector(t, n, reference_channel=1), g['wmwf_ref1'])
    close(X.wmwf_vector(t, n), g['wmwf_auto'])
    close(X.wmwf_vector(t, n, reference_channel=2, distortion_weight=0.), g['wmwf_mu0'])
    close(X.wmwf_vector(t, n, distortion_weight=3.5), g['wmwf_mu3'])
    close(X.wmwf_vector(t, n, reference_channel=0, distortion_weight='frequency_dependent'), g['wmwf_fd'])
    close(X.wmwf_vector(t, n, distortion_weight='frequency_dependent'), g['wmwf_fd_auto'])
    close(X.wmwf_vector(t, n, channel_selection_vector=g['csv']), g['wmwf_csv'])


def test_merl_is_wmwf_with_mu_zero_at_channel_zero(g):
    t, n = g['target'], g['noise']
    close(X.mvdr_vector_merl(t, n), g['merl'])
    close(X.wmwf_vector(t, n, reference_channel=0, distortion_weight=0.), g['merl'])


def test_reference_channel_and_pca(g):
    assert X.optimal_reference_channel(g['w_mat'], g['target'], g['noise']) == int(g['ref_channel'])
    w, v = np.linalg.eigh(g['target'])
    close(w, g['pca_all_vals'])
    close(np.abs(np.einsum('fdk,fdk->fk', v.conj(), g['pca_all_vecs'])), 1)


def test_post_processing(g):
    vec, t, n = g['vec'], g['target'], g['noise']
    close(X.distortionless_normalization(vec, g['atf'][0], n), g['distortionless'])
    close(X.mvdr_snr_postfilter(vec, t, n), g['snr_postfilter'])
    close(X.zero_degree_normalization(vec, 2), g['zero_degree_ref2'])
    close(X.condition_covariance(g['cc_x'], float(g['cc_gamma'])), g['condition_covariance'])


def test_phase_correction_runs_along_axis_zero(g):
    close(X.phase_correction(g['vec']), g['phase_fd'])
    close(X.phase_correction(g['vec_kfd']), g['phase_kfd'])
    # for (K, F, D) the product is over K: vector k = 0 is scaled by one factor per bin only
    v = g['vec_kfd']
    e = np.exp(1j * np.angle(np.sum(v[0, 1:].conj() * v[0, :-1], axis=-1)))
    close(g['phase_kfd'][0, 1:], v[0, 1:] * e[:, None])


def test_online_application(g):
    close(X.apply_online_beamforming_vector(g['online_vector'], g['online_mix']), g['online_c128'])
    np.testing.assert_allclose(X.apply_online_beamforming_vector(g['online_vector'], g['online_mix64']),
                               g['online_c64'], rtol=1e-5, atol=1e-6)
