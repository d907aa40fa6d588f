"""Generate tests/golden/mask.npz from the UNMODIFIED reference (oracle/ref_shim.py): the oracle masks of
pb_bss/extraction/mask_module.py and the array geometry of pb_bss/extraction/beamform_utils.py, plus one oracle-mask
beamforming pipeline and one superdirective MVDR.

Run where a reference checkout or oracle/_ref is present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_mask [OUT_DIR]

Inputs are stored next to the reference's outputs, so the tests need neither the reference nor this script.
"""
import importlib
import os
import sys

import numpy as np

from . import ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')

SOURCE_MASKS = ['ideal_binary_mask', 'wiener_like_mask', 'ideal_ratio_mask', 'ideal_amplitude_mask',
                'phase_sensitive_mask', 'ideal_complex_mask']


def make_mask(out_dir=OUT):
    ns = ref_shim.load()
    M = importlib.import_module('pb_bss.extraction.mask_module')
    BU = importlib.import_module('pb_bss.extraction.beamform_utils')
    RB = ns.beamformer
    rng = np.random.RandomState(71)
    K, D, F, T = 2, 3, 9, 12
    sig = rng.randn(K, D, F, T) + 1j * rng.randn(K, D, F, T)
    ties = rng.randint(-2, 3, size=(K, F, T)).astype(np.float32)  # integer powers: exact ties between sources
    out = {'sig': sig, 'ties': ties}

    for name in SOURCE_MASKS:
        fn = getattr(M, name)
        out[name] = fn(sig)
        out[name + '_src1'] = fn(np.moveaxis(sig, 0, 1), source_axis=1)
        out[name + '_c64'] = fn(sig.astype(np.complex64))
        out[name + '_f32'] = fn(ties)
    for name in ('ideal_binary_mask', 'wiener_like_mask'):
        fn = getattr(M, name)
        out[name + '_sens'] = fn(sig, sensor_axis=1)
        out[name + '_sens_keep'] = fn(sig, sensor_axis=1, keepdims=True)
        out[name + '_sens_c64'] = fn(sig.astype(np.complex64), sensor_axis=1)

    # Lorenz: pooled and per channel, several fractions and weights, one axis, float32 / complex64, arange ties
    out['lorenz'] = M.lorenz_mask(sig)
    out['lorenz_sens'] = M.lorenz_mask(sig, sensor_axis=1)
    out['lorenz_sens_keep'] = M.lorenz_mask(sig, sensor_axis=1, keepdims=True)
    for frac, w in ((0.1, 0.5), (0.4, 0.999), (0.8, 0), (0.89, 1)):
        out[f'lorenz_f{frac}_w{w}'] = M.lorenz_mask(sig, sensor_axis=0, lorenz_fraction=frac, weight=w)
    out['lorenz_axis_t'] = M.lorenz_mask(sig, axis=-1, lorenz_fraction=0.7)
    out['lorenz_axis_f'] = M.lorenz_mask(sig, axis=-2, lorenz_fraction=0.7)
    out['lorenz_c64'] = M.lorenz_mask(sig.astype(np.complex64), sensor_axis=1)
    out['lorenz_ties'] = M.lorenz_mask(ties, lorenz_fraction=0.6)
    out['arange33'] = np.arange(9).reshape(3, 3).astype(np.float32)
    out['lorenz_arange33'] = M.lorenz_mask(out['arange33'], weight=1)
    out['arange233'] = np.arange(18).reshape(2, 3, 3).astype(np.float32)
    out['lorenz_arange233'] = M.lorenz_mask(out['arange233'], weight=1)

    # quantile: the default tuple along F, both axes, single quantiles, float32 ties and complex64
    out['quantile'] = M.quantile_mask(sig)
    out['quantile_ft'] = M.quantile_mask(sig, axis=(-2, -1))
    out['quantile_t_03'] = M.quantile_mask(sig, 0.3, axis=-1, weight=0.5)
    out['quantile_neg'] = M.quantile_mask(sig, -0.25)
    out['quantile_c64'] = M.quantile_mask(sig.astype(np.complex64))
    out['quantile_f32'] = M.quantile_mask(ties, (0.5, -0.5, 0.0, 1.0))

    # biased binary mask: F > high_cut (only the last axis is cut above high_cut) and F < high_cut
    big = rng.randn(2, 3, 520) + 1j * rng.randn(2, 3, 520)
    out['bbm_big'] = big
    out['bbm_big_out'] = M.biased_binary_mask(big)
    small = (rng.randn(2, 5, 40) + 1j * rng.randn(2, 5, 40)).astype(np.complex64)   # F = 40 < high_cut
    out['bbm_small'] = small
    out['bbm_small_out'] = M.biased_binary_mask(small)
    out['bbm_small_cut_out'] = M.biased_binary_mask(small, low_cut=3, high_cut=30)
    out['vu_513_v'], out['vu_513_u'] = M.voiced_unvoiced_split_characteristic(513)

    # geometry
    sensors = rng.uniform(-0.1, 0.1, size=(3, 4))
    sources = rng.uniform(-2, 2, size=(3, 2))
    angles = np.stack([rng.uniform(-np.pi, np.pi, 3), rng.uniform(-np.pi / 2, np.pi / 2, 3)])
    tdoa = rng.uniform(-3e-4, 3e-4, size=(2, 4))
    dist = np.linalg.norm(sensors[:, :, None] - sensors[:, None, :], axis=0)
    out.update(sensors=sensors, sources=sources, angles=angles, tdoa=tdoa, dist=dist)
    out['steer'] = BU.get_steering_vector(tdoa, stft_size=64)
    out['steer_norm'] = BU.get_steering_vector(tdoa, stft_size=64, normalize=True)
    out['diffuse'] = BU.get_diffuse_noise_psd(dist, fft_size=64)
    out['tof'] = BU.get_nearfield_time_of_flight(sources, sensors)
    out['tdoa_ff'] = BU.get_farfield_time_difference_of_arrival(angles, sensors)
    out['tdoa_ff_ref0'] = BU.get_farfield_time_difference_of_arrival(angles, sensors, reference_channel=0)

    # oracle-mask pipeline: IBM pooled over sensors -> PSD -> Souden MVDR -> apply
    obs = sig.sum(0)                                              # (D, F, T)
    ibm = M.ideal_binary_mask(sig, sensor_axis=1)                 # (K, F, T)
    Y = obs.transpose(1, 0, 2)                                    # (F, D, T)
    psd = RB.get_power_spectral_density_matrix(Y, ibm.transpose(1, 0, 2))   # (F, K, D, D)
    w = RB.get_mvdr_vector_souden(psd[:, 0], psd[:, 1])
    out['pipe_out'] = RB.apply_beamforming_vector(w, Y)
    # superdirective MVDR: steering vector of one direction against the diffuse-noise coherence (F = 33 bins)
    sv = BU.get_steering_vector(tdoa[0], stft_size=64).T          # (F, D)
    out['superdirective'] = RB.get_mvdr_vector(sv, out['diffuse'] + 1e-3 * np.eye(4))

    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'mask.npz')
    np.savez_compressed(path, **out)
    return path


if __name__ == '__main__':
    print(make_mask(*sys.argv[1:]))
