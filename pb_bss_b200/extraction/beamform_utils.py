"""Array geometry on the device, signatures of pb_bss/extraction/beamform_utils.py: analytic steering vectors, the
diffuse-noise coherence matrix and near- / far-field propagation delays.  With get_mvdr_vector they give
delay-and-sum and superdirective beamformers.  numpy in -> numpy out, CUDA tensors in -> CUDA tensors out.
"""
import numpy as np
import torch
from numpy.exceptions import AxisError

from .. import _device


def get_stft_center_frequencies(size=1024, sample_rate=16000):
    """Center frequency of every STFT bin, size // 2 + 1 of them (pb_bss/utils.py:172-182); host NumPy."""
    return np.arange(0, size / 2 + 1) * sample_rate / size


def _f64(x):
    like_numpy = not _device.is_tensor(x)
    return _device.to_device(np.asarray(x, dtype=np.float64) if like_numpy else x, torch.float64), like_numpy


def get_steering_vector(
        time_difference_of_arrival,
        stft_size=1024,
        sample_rate=16000,
        normalize=False
):
    """exp(-2j pi f tdoa) for the STFT center frequencies f, shape tdoa.shape + (F,), complex128
    (beamform_utils.py:36-63).  normalize=True divides by the 2-norm over axis -2, whatever that axis is."""
    tdoa, like_numpy = _f64(time_difference_of_arrival)
    if normalize and tdoa.dim() < 1:
        raise AxisError(-2, 1)
    freq = _device.to_device(get_stft_center_frequencies(stft_size, sample_rate))
    F = freq.shape[0]
    M = tdoa.shape[-1] if normalize else 1
    A = tdoa.numel() // M if M else 0
    out = _device.empty((*tdoa.shape, F), torch.complex128)
    if out.numel():
        _device.call('pbb_steering_vector', tdoa, A, M, freq, F, int(bool(normalize)), out)
    return _device.to_host(out, like_numpy)


def get_diffuse_noise_psd(
        sensor_distances,
        fft_size=1024,
        sample_rate=16000,
        sound_velocity=343
):
    """Spatial coherence of a spherically isotropic sound field, np.sinc(2 f d / c), shape (F, D, D), float64
    (beamform_utils.py:66-97; Bitzer and Simmer, "Superdirective microphone arrays", 2001, eq. 2.17)."""
    dist, like_numpy = _f64(sensor_distances)
    assert dist.dim() == 2 and dist.shape[0] == dist.shape[1], 'sensor_distances: (num_channels, num_channels)'
    freq = _device.to_device(get_stft_center_frequencies(size=fft_size, sample_rate=sample_rate))
    F, D = freq.shape[0], dist.shape[0]
    out = _device.empty((F, D, D), torch.float64)
    if out.numel():
        _device.call('pbb_diffuse_noise_coherence', dist, D, freq, F, float(sound_velocity), out)
    return _device.to_host(out, like_numpy)


def get_nearfield_time_of_flight(source_positions, sensor_positions,
                                 sound_velocity=343):
    """Exact time of flight |source - sensor| / c in seconds, shape (sources, sensors) (beamform_utils.py:100-116).
    Positions are 3-D column vectors: source_positions (3, S), sensor_positions (3, M)."""
    src, like_numpy = _f64(source_positions)
    sen, _ = _f64(sensor_positions)
    assert src.shape[0] == 3
    assert sen.shape[0] == 3
    src, sen = src.reshape(3, -1), sen.reshape(3, -1)
    S, M = src.shape[1], sen.shape[1]
    out = _device.empty((S, M), torch.float64)
    if out.numel():
        _device.call('pbb_array_geometry', 0, src, S, sen, M, 0, float(sound_velocity), out)
    return _device.to_host(out, like_numpy)


def get_farfield_time_difference_of_arrival(
        source_angles,
        sensor_positions,
        reference_channel=1,
        sound_velocity=343.,
):
    """Far-field TDOA of plane waves from the (azimuth, elevation) angles (2, K) at the sensors (3, M), relative to
    sensor reference_channel, shape (M, K) (beamform_utils.py:119-159)."""
    ang, like_numpy = _f64(source_angles)
    sen, _ = _f64(sensor_positions)
    M, K = sen.shape[1], ang.shape[1]
    if not -M <= reference_channel < M:
        raise IndexError(f'index {reference_channel} is out of bounds for axis 1 with size {M}')
    out = _device.empty((M, K), torch.float64)
    if out.numel():
        _device.call('pbb_array_geometry', 1, ang, K, sen, M, reference_channel % M, float(sound_velocity), out)
    return _device.to_host(out, like_numpy)
