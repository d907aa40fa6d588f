"""Oracle masks and array geometry on the device against the fixture of the unmodified reference
(oracle/make_golden_mask.py), against the NumPy restatement of the selections (oracle/mask_oracle.py) and against the
properties the masks promise independently of either."""
import numpy as np
import pytest
import torch
from numpy.exceptions import AxisError

from conftest import load_golden
from oracle import mask_oracle as MO
from pb_bss_b200 import _lib, extraction as E
from pb_bss_b200.extraction import beamform_utils as BU

pytestmark = pytest.mark.gpu

SOURCE_MASKS = ['ideal_binary_mask', 'wiener_like_mask', 'ideal_ratio_mask', 'ideal_amplitude_mask',
                'phase_sensitive_mask', 'ideal_complex_mask']


@pytest.fixture(scope='module')
def g():
    return load_golden('mask')


def cplx(rng, *shape):
    return rng.randn(*shape) + 1j * rng.randn(*shape)


def close(a, b, rtol=1e-12, atol=1e-15):
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


# ---- parity with the reference's fixture -----------------------------------------------------------------------

@pytest.mark.parametrize('name', SOURCE_MASKS)
def test_source_masks_match_reference(g, name):
    fn = getattr(E, name)
    sig = g['sig']
    exact = name == 'ideal_binary_mask'
    check = (lambda a, b: np.testing.assert_array_equal(a, b)) if exact else close
    check(fn(sig), g[name])
    check(fn(np.moveaxis(sig, 0, 1), source_axis=1), g[name + '_src1'])
    # the reference computes the complex64 masks in float32, the device in fp64 from the stored values
    got = fn(sig.astype(np.complex64))
    assert got.dtype == g[name + '_c64'].dtype
    if exact:
        np.testing.assert_array_equal(got, g[name + '_c64'])
    else:
        np.testing.assert_allclose(got, g[name + '_c64'], rtol=1e-6, atol=1e-6)
    with np.errstate(divide='ignore', invalid='ignore'):
        got = fn(g['ties'])
    # exact ties between the sources (integer powers) and, for the complex mask, zero observations (inf / nan)
    np.testing.assert_array_equal(got, g[name + '_f32']) if exact else \
        np.testing.assert_allclose(got, g[name + '_f32'], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize('name', ['ideal_binary_mask', 'wiener_like_mask'])
def test_sensor_pooling_matches_reference(g, name):
    fn = getattr(E, name)
    sig = g['sig']
    check = np.testing.assert_array_equal if name == 'ideal_binary_mask' else close
    check(fn(sig, sensor_axis=1), g[name + '_sens'])
    check(fn(sig, sensor_axis=1, keepdims=True), g[name + '_sens_keep'])
    got = fn(sig.astype(np.complex64), sensor_axis=1)
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, g[name + '_sens_c64'], rtol=1e-6, atol=1e-7)


def test_lorenz_matches_reference(g):
    sig = g['sig']
    np.testing.assert_array_equal(E.lorenz_mask(sig), g['lorenz'])
    np.testing.assert_array_equal(E.lorenz_mask(sig, sensor_axis=1), g['lorenz_sens'])
    np.testing.assert_array_equal(E.lorenz_mask(sig, sensor_axis=1, keepdims=True), g['lorenz_sens_keep'])
    for frac, w in ((0.1, 0.5), (0.4, 0.999), (0.8, 0), (0.89, 1)):
        np.testing.assert_array_equal(E.lorenz_mask(sig, sensor_axis=0, lorenz_fraction=frac, weight=w),
                                      g[f'lorenz_f{frac}_w{w}'])
    np.testing.assert_array_equal(E.lorenz_mask(sig, axis=-1, lorenz_fraction=0.7), g['lorenz_axis_t'])
    np.testing.assert_array_equal(E.lorenz_mask(sig, axis=-2, lorenz_fraction=0.7), g['lorenz_axis_f'])
    np.testing.assert_array_equal(E.lorenz_mask(g['ties'], lorenz_fraction=0.6), g['lorenz_ties'])
    np.testing.assert_array_equal(E.lorenz_mask(g['arange33'], weight=1), g['lorenz_arange33'])
    np.testing.assert_array_equal(E.lorenz_mask(g['arange233'], weight=1), g['lorenz_arange233'])


def test_lorenz_complex64_against_float32_reference(g):
    """fp64 from the stored complex64 values: exact against the fp64 oracle; against the reference's float32
    result the two masks differ only at elements whose power lies between the two thresholds."""
    s64 = g['sig'].astype(np.complex64)
    got = E.lorenz_mask(s64, sensor_axis=1)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, MO.lorenz_mask(s64, sensor_axis=1))
    ref = g['lorenz_c64']
    diff = got != ref
    print('lorenz complex64: %d of %d elements differ from the float32 reference' % (diff.sum(), diff.size))
    assert diff.sum() <= 2


def test_quantile_matches_reference(g):
    sig = g['sig']
    np.testing.assert_array_equal(E.quantile_mask(sig), g['quantile'])
    np.testing.assert_array_equal(E.quantile_mask(sig, axis=(-2, -1)), g['quantile_ft'])
    np.testing.assert_array_equal(E.quantile_mask(sig, 0.3, axis=-1, weight=0.5), g['quantile_t_03'])
    np.testing.assert_array_equal(E.quantile_mask(sig, -0.25), g['quantile_neg'])
    np.testing.assert_array_equal(E.quantile_mask(sig.astype(np.complex64)), g['quantile_c64'])
    got = E.quantile_mask(g['ties'], (0.5, -0.5, 0.0, 1.0))
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, g['quantile_f32'])


def test_biased_binary_mask_matches_reference(g):
    got = E.biased_binary_mask(g['bbm_big'])
    assert got.dtype == np.bool_
    np.testing.assert_array_equal(got, g['bbm_big_out'])
    np.testing.assert_array_equal(E.biased_binary_mask(g['bbm_small']), g['bbm_small_out'])
    np.testing.assert_array_equal(E.biased_binary_mask(g['bbm_small'], low_cut=3, high_cut=30),
                                  g['bbm_small_cut_out'])
    v, u = E.voiced_unvoiced_split_characteristic(513)
    np.testing.assert_array_equal(v, g['vu_513_v'])
    np.testing.assert_array_equal(u, g['vu_513_u'])


def test_geometry_matches_reference(g):
    close(BU.get_steering_vector(g['tdoa'], stft_size=64), g['steer'])
    close(BU.get_steering_vector(g['tdoa'], stft_size=64, normalize=True), g['steer_norm'])
    close(BU.get_diffuse_noise_psd(g['dist'], fft_size=64), g['diffuse'])
    assert (np.diagonal(BU.get_diffuse_noise_psd(g['dist'], fft_size=64), axis1=1, axis2=2) == 1).all()
    close(BU.get_nearfield_time_of_flight(g['sources'], g['sensors']), g['tof'])
    close(BU.get_farfield_time_difference_of_arrival(g['angles'], g['sensors']), g['tdoa_ff'], atol=1e-18)
    close(BU.get_farfield_time_difference_of_arrival(g['angles'], g['sensors'], reference_channel=0),
          g['tdoa_ff_ref0'], atol=1e-18)


def test_oracle_mask_pipeline_and_superdirective_mvdr(g):
    sig = g['sig']
    Y = sig.sum(0).transpose(1, 0, 2)
    ibm = E.ideal_binary_mask(sig, sensor_axis=1)
    psd = E.get_power_spectral_density_matrix(Y, ibm.transpose(1, 0, 2))
    w = E.get_mvdr_vector_souden(psd[:, 0], psd[:, 1])
    np.testing.assert_allclose(E.apply_beamforming_vector(w, Y), g['pipe_out'], rtol=1e-9, atol=1e-12)
    sv = BU.get_steering_vector(g['tdoa'][0], stft_size=64).T
    w_sd = E.get_mvdr_vector(sv, BU.get_diffuse_noise_psd(g['dist'], fft_size=64) + 1e-3 * np.eye(4))
    np.testing.assert_allclose(w_sd, g['superdirective'], rtol=1e-9, atol=1e-12)


# ---- properties (written for this port) --------------------------------------------------------------------------

@pytest.mark.parametrize('shape,sensor_axis', [((2, 3), None), ((2, 3, 5), None), ((2, 3, 5), 1),
                                               ((3, 4, 6, 7), 1), ((2, 4, 6, 7), 2)])
def test_binary_and_wiener_shapes_binary_sum_to_one(shape, sensor_axis):
    rng = np.random.RandomState(1)
    sig = cplx(rng, *shape)
    expect = tuple(n for i, n in enumerate(shape) if i != sensor_axis)
    ibm = E.ideal_binary_mask(sig, sensor_axis=sensor_axis)
    assert ibm.shape == expect and set(np.unique(ibm)) <= {0.0, 1.0}
    np.testing.assert_array_equal(ibm.sum(0), 1.0)
    wlm = E.wiener_like_mask(sig, sensor_axis=sensor_axis)
    assert wlm.shape == expect and (wlm >= 0).all() and (wlm <= 1).all()
    np.testing.assert_allclose(wlm.sum(0), 1.0, rtol=1e-12)
    for name in ('ideal_ratio_mask', 'ideal_amplitude_mask', 'phase_sensitive_mask', 'ideal_complex_mask'):
        assert getattr(E, name)(sig).shape == shape
    np.testing.assert_allclose(E.ideal_ratio_mask(sig).sum(0), 1.0, rtol=1e-12)
    np.testing.assert_allclose(E.ideal_complex_mask(sig).sum(0), 1.0, rtol=1e-12, atol=1e-12)


def test_equal_power_ties_and_eps():
    np.testing.assert_array_equal(E.ideal_binary_mask(np.array([1 + 1j, 1 - 1j])), [1.0, 0.0])
    np.testing.assert_array_equal(E.wiener_like_mask(np.asarray([0.5 + 0.5j, 0.5 + 0.5j])), [0.5, 0.5])
    np.testing.assert_array_equal(E.wiener_like_mask(np.zeros((2, 3))), np.zeros((2, 3)))


@pytest.mark.parametrize('sensor_axis', [None, 0, 1])
@pytest.mark.parametrize('frac', [0.1, 0.4, 0.8, 0.89])
def test_lorenz_weight_zero_and_bounds(sensor_axis, frac):
    rng = np.random.RandomState(2)
    sig = cplx(rng, 2, 3, 17, 19)
    m0 = E.lorenz_mask(sig, sensor_axis=sensor_axis, lorenz_fraction=frac, weight=0)
    assert m0.shape == tuple(n for i, n in enumerate(sig.shape) if i != sensor_axis)
    np.testing.assert_array_equal(m0, 0.5)
    for w in (0.5, 0.999):
        m = E.lorenz_mask(sig, sensor_axis=sensor_axis, lorenz_fraction=frac, weight=w)
        assert (m >= 0.5 * (1 - w)).all() and (m <= 0.5 * (1 + w)).all()


def test_lorenz_list_input_and_arange():
    rng = np.random.RandomState(3)
    s = cplx(rng, 7, 9)
    m1, m2 = E.lorenz_mask(s), E.lorenz_mask([s, s])
    np.testing.assert_array_equal(m2[0], m1)
    np.testing.assert_array_equal(m2[1], m1)
    a = np.arange(9).reshape(3, 3).astype(np.float32)
    np.testing.assert_array_equal(E.lorenz_mask(a, weight=1), np.array([0, 0, 0, 0, 1, 1, 1, 1, 1],
                                                                        np.float32).reshape(3, 3))
    a = np.arange(18).reshape(2, 3, 3).astype(np.float32)
    np.testing.assert_array_equal(E.lorenz_mask(a, weight=1), np.array(
        [[[0, 0, 0], [0, 1, 1], [1, 1, 1]], [[0, 0, 1], [1, 1, 1], [1, 1, 1]]], np.float32))


def _lorenz_rows_close(got, sig, **kw):
    """Equal to the fp64 oracle except where the Lorenz value of the threshold lies within 1e-12 of the fraction
    (the sums are formed in another order)."""
    ref = MO.lorenz_mask(sig, **kw)
    diff = got != ref
    if diff.any():
        frac = kw.get('lorenz_fraction', 0.98)
        power = np.abs(sig) ** 2
        if kw.get('sensor_axis') is not None:
            power = power.sum(kw['sensor_axis'])
        assert diff.sum() < 4, diff.sum()
        p = np.sort(power.ravel())[::-1]
        lv = np.cumsum(p) / p.sum()
        assert np.min(np.abs(lv - frac)) < 1e-12


@pytest.mark.parametrize('T', [300, 4096, 4097, 9000])
def test_lorenz_both_sides_of_the_row_length_threshold(T):
    rng = np.random.RandomState(T)
    sig = cplx(rng, 3, 2, T)
    for axis in (-1, (-2, -1)):
        got = E.lorenz_mask(sig, axis=axis, lorenz_fraction=0.9)
        _lorenz_rows_close(got, sig, axis=axis, lorenz_fraction=0.9)


@pytest.mark.parametrize('F,axis', [(513, -2), (4096, -2), (4097, -2), (40, (-2, -1)), (513, (-2, -1))])
def test_quantile_both_sides_of_the_row_length_threshold(F, axis):
    rng = np.random.RandomState(F)
    sig = cplx(rng, 2, 3, F, 64)
    np.testing.assert_array_equal(E.quantile_mask(sig, axis=axis), MO.quantile_mask(sig, axis=axis))
    s32 = np.abs(sig).astype(np.float32)
    np.testing.assert_array_equal(E.quantile_mask(s32, (0.3, -0.7), axis=axis),
                                  MO.quantile_mask(s32, (0.3, -0.7), axis=axis))


def test_realistic_size_against_oracle():
    """(K, D, F, T) = (2, 6, 513, 500) complex128: Lorenz pooled over sensors (two rows of 256500), Lorenz along
    time (6156 rows of 500) and the default quantile mask along frequency (strided rows of 513)."""
    rng = np.random.RandomState(2024)
    sig = cplx(rng, 2, 6, 513, 500)
    x = torch.from_numpy(sig).cuda()
    got = E.lorenz_mask(x, sensor_axis=1)
    assert isinstance(got, torch.Tensor) and got.is_cuda and got.shape == (2, 513, 500)
    _lorenz_rows_close(got.cpu().numpy(), sig, sensor_axis=1)
    got = E.lorenz_mask(sig, axis=-1, lorenz_fraction=0.9)
    ref = MO.lorenz_mask(sig, axis=-1, lorenz_fraction=0.9)
    assert (got != ref).sum() < 4
    np.testing.assert_array_equal(E.quantile_mask(x).cpu().numpy(), MO.quantile_mask(sig))
    np.testing.assert_array_equal(E.ideal_binary_mask(x, sensor_axis=1).cpu().numpy(),
                                  np.expand_dims(np.argmax((np.abs(sig) ** 2).sum(1), 0), 0) ==
                                  np.arange(2)[:, None, None])


def test_tensor_in_tensor_out_and_strided_views():
    rng = np.random.RandomState(5)
    sig = cplx(rng, 4, 2, 3, 11)                                  # (F, K, D, T): source axis 1
    x = torch.from_numpy(sig).cuda()
    for name in ('ideal_binary_mask', 'wiener_like_mask'):
        got = getattr(E, name)(x, source_axis=1, sensor_axis=2)
        assert isinstance(got, torch.Tensor) and got.is_cuda and got.dtype == torch.float64
        np.testing.assert_allclose(got.cpu().numpy(), getattr(E, name)(sig, source_axis=1, sensor_axis=2), rtol=0)
    xt = x.transpose(0, 3)                                        # a non-contiguous view: read in place
    got = E.ideal_complex_mask(xt, source_axis=1)
    assert got.dtype == torch.complex128
    np.testing.assert_allclose(got.cpu().numpy(), E.ideal_complex_mask(np.ascontiguousarray(sig.transpose(3, 1, 2, 0)),
                                                                       source_axis=1), rtol=0)
    q = E.quantile_mask(xt[:, :, 0], axis=-1)
    assert isinstance(q, torch.Tensor) and q.shape == (2, 11, 2, 4)
    tv = BU.get_steering_vector(torch.zeros(3, dtype=torch.float64, device='cuda'), stft_size=16)
    assert isinstance(tv, torch.Tensor) and tv.shape == (3, 9)


def test_errors():
    rng = np.random.RandomState(6)
    sig = cplx(rng, 2, 3, 5)
    for name in ('ideal_ratio_mask', 'ideal_amplitude_mask', 'phase_sensitive_mask', 'ideal_complex_mask'):
        with pytest.raises(AssertionError):
            getattr(E, name)(sig, sensor_axis=1)
    with pytest.raises(AssertionError):
        E.quantile_mask(sig, sensor_axis=1)
    with pytest.raises(AssertionError):
        E.biased_binary_mask(cplx(rng, 3, 4, 20))
    with pytest.raises(NotImplementedError):
        E.biased_binary_mask(cplx(rng, 2, 4, 20), sensor_axis=1)
    with pytest.raises(AxisError):
        E.lorenz_mask(np.ones(5))
    # the largest value holds more than lorenz_fraction of a row: np.min of an empty selection in the reference
    peaked = np.ones((2, 4, 6))
    peaked[1, 2, 3] = 1e6
    with pytest.raises(ValueError, match='row 1'):
        E.lorenz_mask(peaked)
    with pytest.raises(ValueError):
        E.lorenz_mask(np.zeros((3, 4)))
    long_zero = np.zeros((2, 5000))
    long_zero[0] = 1.0
    with pytest.raises(ValueError, match='row 1'):
        E.lorenz_mask(long_zero, axis=-1)
    with pytest.raises(AssertionError):
        BU.get_nearfield_time_of_flight(np.zeros((2, 3)), np.zeros((3, 3)))
    lib = _lib.load()
    assert lib.pbb_source_mask(None, 1, 0, 2, 1, 1, 0, 1, None, 0.0, None, None) == -1
