"""Generate tests/golden/extraction.npz from the UNMODIFIED reference (oracle/ref_shim.py): the multi-source
beamformers and vector post-processing of pb_bss/extraction/beamformer.py.

Run where a reference checkout or oracle/_ref is present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_extraction [OUT_DIR]

Inputs are stored next to the reference's outputs, so the tests need neither the reference nor this script.
"""
import os
import sys

import numpy as np

from . import ref_shim, synth

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def _cplx(rng, *shape):
    return rng.randn(*shape) + 1j * rng.randn(*shape)


def make_extraction(out_dir=OUT):
    RB = ref_shim.load().beamformer
    rng = np.random.RandomState(61)
    F, D, K = 9, 4, 3
    out = {}
    target = synth.pos_def_hermitian(F, D, D, seed=62)
    noise = synth.pos_def_hermitian(F, D, D, seed=63)
    atf = _cplx(rng, K, F, D)
    out.update(target=target, noise=noise, atf=atf)

    # LCMV: one-hot and epsilon-clipped responses, a zero noise matrix in one bin (lstsq path), K = D
    out['lcmv_onehot'] = RB.get_lcmv_vector(atf, [1, 0, 0], noise)
    out['lcmv_clipped'] = RB.get_lcmv_vector(atf, [1, 1e-3, 1e-3], noise)
    noise_sing = noise.copy()
    noise_sing[4] = 0
    out['noise_sing'] = noise_sing
    out['lcmv_sing'] = RB.get_lcmv_vector(atf, [0, 1, 0], noise_sing)
    atf_kd = _cplx(rng, D, F, D)
    out['atf_kd'] = atf_kd
    out['lcmv_kd'] = RB.get_lcmv_vector(atf_kd, [0, 0, 1, 0], noise)

    # WMWF: every distortion_weight form, explicit and automatic reference channel, channel selection
    out['wmwf_ref1'] = RB.get_wmwf_vector(target, noise, reference_channel=1)
    out['wmwf_auto'] = RB.get_wmwf_vector(target, noise)
    out['wmwf_mu0'] = RB.get_wmwf_vector(target, noise, reference_channel=2, distortion_weight=0.)
    out['wmwf_mu3'] = RB.get_wmwf_vector(target, noise, distortion_weight=3.5)
    out['wmwf_fd'] = RB.get_wmwf_vector(target, noise, reference_channel=0, distortion_weight='frequency_dependent')
    out['wmwf_fd_auto'] = RB.get_wmwf_vector(target, noise, distortion_weight='frequency_dependent')
    csv = rng.uniform(size=(F, D))
    out['csv'] = csv
    out['wmwf_csv'] = RB.get_wmwf_vector(target, noise, channel_selection_vector=csv)

    # MERL MVDR
    out['merl'] = RB.get_mvdr_vector_merl(target, noise)

    # reference channel, PCA
    w_mat = _cplx(rng, F, D, D)
    out['w_mat'] = w_mat
    out['ref_channel'] = np.int64(RB.get_optimal_reference_channel(w_mat, target, noise))
    vecs, vals = RB.get_pca(target)
    out.update(pca_vec=vecs, pca_val=vals)
    vecs, vals = RB.get_pca(target, return_all_vecs=True)
    out.update(pca_all_vecs=vecs, pca_all_vals=vals)

    # post-processing
    vec = _cplx(rng, F, D)
    out['vec'] = vec
    out['distortionless'] = RB.distortionless_normalization(vec, atf[0], noise)
    out['snr_postfilter'] = RB.mvdr_snr_postfilter(vec, target, noise)
    out['zero_degree_ref2'] = RB.zero_degree_normalization(vec, 2)
    out['phase_fd'] = RB.phase_correction(vec)
    vec_kfd = _cplx(rng, K, F, D)
    out['vec_kfd'] = vec_kfd
    out['phase_kfd'] = RB.phase_correction(vec_kfd)      # the product runs over K (axis 0), not over F
    x = synth.pos_def_hermitian(2, F, D, D, seed=64) + 0.1j * _cplx(rng, 2, F, D, D)
    out['cc_x'] = x
    out['cc_gamma'] = np.float64(0.3)
    out['condition_covariance'] = RB.condition_covariance(x, 0.3)

    # time-varying application: complex128 and complex64 mixes, a leading dim on the mix
    T = 12
    v_on = _cplx(rng, T, F, D)
    mix = _cplx(rng, 2, F, D, T)
    out.update(online_vector=v_on, online_mix=mix)
    out['online_c128'] = RB.apply_online_beamforming_vector(v_on, mix)
    mix64 = mix[0].astype(np.complex64)
    out['online_mix64'] = mix64
    out['online_c64'] = RB.apply_online_beamforming_vector(v_on, mix64)
    np.savez_compressed(os.path.join(out_dir, 'extraction.npz'), **out)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    os.makedirs(out, exist_ok=True)
    ref_shim.load()
    make_extraction(out)


if __name__ == '__main__':
    main()
