"""pb_bss_b200.wpe on the device against the NumPy oracle (oracle/wpe_oracle.py): shapes, parameters, statistics
modes, dtypes, layouts, the lstsq and NaN branches, reproducibility and the errors."""
import math

import numpy as np
import pytest
import torch

from oracle import wpe_oracle as W

pytestmark = pytest.mark.gpu


def _y(shape, seed=0, dtype=np.complex128):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)


def _oracle(Y, **kw):
    """The oracle's X and, per bin, n eps kappa(R) of its last R: the forward-error bound of a backward-stable solve,
    kappa over the eigenvalues above lstsq's cut-off (an exactly singular R is solved on its range)."""
    Y = np.asarray(Y)
    flat = Y.reshape((-1,) + Y.shape[-2:])
    X, bound = [], []
    for y in flat:
        with np.errstate(invalid='ignore'):
            x, last, _ = W.wpe_bin(y, details=True, **kw)
        X.append(x)
        if last is None:
            bound.append(0.0)
            continue
        lam = np.abs(np.linalg.eigvalsh(last[1]))
        lam = lam[lam > lam.max() * lam.size * np.finfo(np.float64).eps] if lam.max() > 0 else lam[:0]
        bound.append(lam.size * np.finfo(np.float64).eps * lam.max() / lam.min() if lam.size else 0.0)
    return np.stack(X).reshape(Y.shape).astype(Y.dtype), np.array(bound)


def _close(got, want, Y, bound=None):
    """per-bin max error at most 1e-10 max|Y_f|, or that bin's n eps kappa(R) max|Y_f| where R is worse conditioned;
    complex64 adds one float32 rounding of the output."""
    got, want, Y = (np.asarray(a).reshape((-1,) + a.shape[-2:]) for a in (got, want, Y))
    assert got.shape == want.shape and got.dtype == want.dtype
    rtol = np.full(got.shape[0], 1e-10) if bound is None else np.maximum(1e-10, bound)
    if got.dtype == np.complex64:
        rtol = np.maximum(rtol, 4 * np.finfo(np.float32).eps)
    err = np.abs(got.astype(np.complex128) - want.astype(np.complex128)).max(axis=(-2, -1))
    scale = np.abs(Y).max(axis=(-2, -1))
    assert (err <= rtol * scale).all(), (err / scale / rtol).max()


def _check(got, Y, **kw):
    want, bound = _oracle(Y, **kw)
    _close(got, want, Y, bound)


def _run(Y, **kw):
    from pb_bss_b200 import wpe
    return wpe.wpe(Y, **kw)


@pytest.mark.parametrize('D', [1, 2, 4, 6, 8])
@pytest.mark.parametrize('taps', [1, 5, 10, 12])
@pytest.mark.parametrize('delay', [0, 1, 3])
def test_shapes_against_oracle(D, taps, delay):
    # with delay 0 the current frame is part of Yt: one iteration leaves X = Y - Y at rounding level, and weights
    # 1 / lambda of that residue would depend on the rounding, not on the data
    Y = _y((3, D, 200), seed=D * 100 + taps * 10 + delay)
    kw = dict(taps=taps, delay=delay, iterations=1 if delay == 0 else 3)
    _check(_run(Y, **kw), Y, **kw)


@pytest.mark.parametrize('iterations', [0, 1, 3])
@pytest.mark.parametrize('psd_context', [0, 1, 3, math.inf])
@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_parameters_against_oracle(iterations, psd_context, mode):
    Y = _y((4, 4, 300), seed=iterations + 7)
    kw = dict(taps=5, delay=2, iterations=iterations, psd_context=psd_context, statistics_mode=mode)
    _check(_run(Y, **kw), Y, **kw)


@pytest.mark.parametrize('mode', ['full', 'valid'])
@pytest.mark.parametrize('T,F', [(1, 4), ('edge', 4), (500, 513), (20000, 1)])
def test_frame_counts_against_oracle(T, F, mode):
    taps, delay, D = (10, 3, 8) if T == 500 else (5, 3, 2)
    T = taps + delay - 1 if T == 'edge' else T
    Y = _y((F, D, T), seed=T)
    kw = dict(taps=taps, delay=delay, statistics_mode=mode)
    _check(_run(Y, **kw), Y, **kw)


@pytest.mark.parametrize('dtype', [np.complex64, np.complex128])
def test_dtypes_leading_dims_views_and_inplace(dtype):
    from pb_bss_b200 import transform
    Y = _y((2, 5, 3, 150), seed=3, dtype=dtype)          # (B, F, D, T)
    want, bound = _oracle(Y, taps=4, delay=2)
    _close(_run(Y, taps=4, delay=2), want, Y, bound)
    # a CUDA tensor in gives a CUDA tensor out, in the input's layout
    t = torch.from_numpy(Y).cuda()
    out = _run(t, taps=4, delay=2)
    assert out.is_cuda and out.dtype == t.dtype and out.stride() == t.stride()
    _close(out.cpu().numpy(), want, Y, bound)
    # transposed views: (D, T, F) -> (F, D, T), as stft(y).transpose(...) gives
    v = torch.from_numpy(np.ascontiguousarray(Y[0].transpose(1, 2, 0))).cuda().permute(2, 0, 1)
    assert not v.is_contiguous()
    out = _run(v, taps=4, delay=2)
    assert out.stride() == v.stride()
    _close(out.cpu().numpy(), want[0], Y[0], bound[:5])
    # leading dims that do not collapse to one stride take one copy
    u = torch.from_numpy(np.ascontiguousarray(Y.transpose(1, 0, 2, 3))).cuda().transpose(0, 1)
    _close(_run(u, taps=4, delay=2).cpu().numpy(), want, Y, bound)
    # in place: NumPy and CUDA
    Yc = Y.copy()
    assert _run(Yc, taps=4, delay=2, inplace=True) is Yc
    _close(Yc, want, Y, bound)
    tc = torch.from_numpy(Y).cuda()
    assert _run(tc, taps=4, delay=2, inplace=True) is tc
    _close(tc.cpu().numpy(), want, Y, bound)
    vc = torch.from_numpy(np.ascontiguousarray(Y[0].transpose(1, 2, 0))).cuda().permute(2, 0, 1)
    assert _run(vc, taps=4, delay=2, inplace=True) is vc
    _close(vc.cpu().numpy(), want[0], Y[0], bound[:5])
    # the STFT front end
    x = np.random.default_rng(9).standard_normal((2, 4000))
    S = transform.stft(torch.from_numpy(x).cuda(), size=256, shift=64)      # (D, T, F)
    Sv = S.permute(2, 0, 1)
    Sn = np.ascontiguousarray(Sv.cpu().numpy())
    # overlapping frames make R ill-conditioned: the bound is that of kappa(R)
    _check(_run(Sv, taps=5, delay=3).cpu().numpy(), Sn, taps=5, delay=3)


def test_helpers_against_oracle():
    from pb_bss_b200 import wpe
    for dtype in (np.complex64, np.complex128):
        Y = _y((3, 4, 2, 60), seed=5, dtype=dtype)
        for c in (0, 1, 3, 100, math.inf):
            np.testing.assert_allclose(wpe.get_power(Y, c), W.get_power(Y.astype(np.complex128), c), rtol=1e-13)
            np.testing.assert_allclose(wpe.get_power_inverse(Y, c), W.get_power_inverse(Y.astype(np.complex128), c),
                                       rtol=1e-13)
        for taps, delay in ((1, 0), (3, 2), (4, 70)):
            got = wpe.build_y_tilde(Y, taps, delay)
            assert got.dtype == Y.dtype
            np.testing.assert_array_equal(got, W.build_y_tilde(Y, taps, delay))
    t = torch.from_numpy(Y).cuda().transpose(-1, -2).contiguous().transpose(-1, -2)
    out = wpe.get_power(t, 1)
    assert out.is_cuda
    np.testing.assert_allclose(out.cpu().numpy(), W.get_power(Y.astype(np.complex128), 1), rtol=1e-13)


def test_dead_channel_takes_lstsq_and_zero_bin_is_nan():
    from pb_bss_b200 import wpe
    Y = _y((5, 4, 250), seed=11)
    Y[:, 2] = 0                                      # a dead channel in every bin
    Y[3] = 0                                         # and one all-zero bin
    X, status = wpe._run(torch.from_numpy(Y).cuda(), 5, 2, 3, 0, 'full', False)
    assert status == wpe.LSTSQ | wpe.NONFINITE
    X = X.cpu().numpy()
    assert np.isnan(X[3]).all() and np.isfinite(X[[0, 1, 2, 4]]).all()
    keep = [0, 1, 2, 4]
    want, bound = _oracle(Y[keep], taps=5, delay=2)
    _close(X[keep], want, Y[keep], bound)
    _, status = wpe._run(torch.from_numpy(_y((2, 4, 250))).cuda(), 5, 2, 3, 0, 'full', False)
    assert status == 0


@pytest.mark.parametrize('D,taps', [(8, 10), (8, 12), (4, 24)])
def test_dead_channel_lstsq_at_large_n(D, taps):
    """n = taps D of 80 and 96: the minimum-norm fallback's eigensolver runs more than 32 rotation pairs per round."""
    from pb_bss_b200 import wpe
    Y = _y((3, D, 400), seed=D + taps)
    Y[:, 1] = 0
    X, status = wpe._run(torch.from_numpy(Y).cuda(), taps, 3, 3, 0, 'full', False)
    assert status == wpe.LSTSQ
    want, bound = _oracle(Y, taps=taps, delay=3)
    _close(X.cpu().numpy(), want, Y, bound)


@pytest.mark.parametrize('D,taps', [(12, 8), (16, 6), (22, 4), (24, 4), (30, 3), (30, 1)])
def test_many_channels_against_oracle(D, taps):
    """n + D > 104: more lower-triangle tiles than one pass of wpe_corr_kernel holds (and, from D = 23 on, more than
    48 KB of its shared memory)."""
    Y = _y((2, D, 300), seed=D * taps)
    kw = dict(taps=taps, delay=2)
    _check(_run(Y, **kw), Y, **kw)


def test_power_of_many_bins():
    from pb_bss_b200 import wpe
    Y = _y((70000, 2, 3), seed=2)
    np.testing.assert_allclose(wpe.get_power(Y), W.get_power(Y), rtol=1e-13)
    np.testing.assert_allclose(wpe.get_power_inverse(Y, 1), W.get_power_inverse(Y, 1), rtol=1e-13)


def test_repeated_calls_are_bitwise_equal():
    t = torch.from_numpy(_y((9, 6, 3000), seed=4)).cuda()
    a = _run(t, taps=10, delay=3, psd_context=2)
    b = _run(t, taps=10, delay=3, psd_context=2)
    assert torch.equal(a.view(torch.float64), b.view(torch.float64))


def _reverberant(F, D, T, delay, tail, seed):
    """STFT-domain reverberation: a source with a varying envelope, per-channel direct paths and exponentially
    decaying late responses from frame `delay` on."""
    rng = np.random.default_rng(seed)
    env = np.exp(2 * np.sin(np.arange(T) / 17.0)) * (1 + rng.random(T))
    s = env * (rng.standard_normal((F, T)) + 1j * rng.standard_normal((F, T)))
    h0 = np.exp(2j * np.pi * rng.random((F, D)))
    direct = h0[..., None] * s[:, None, :]
    Y = direct.copy()
    for l in range(delay, delay + tail):
        h = 0.6 * np.exp(-(l - delay) / 4.0) * (rng.standard_normal((F, D)) + 1j * rng.standard_normal((F, D)))
        Y[..., l:] += h[..., None] * s[:, None, :T - l]
    return Y, direct


def test_reverberant_orthogonality_and_direct_path():
    from pb_bss_b200 import wpe
    taps, delay = 10, 3
    Y, direct = _reverberant(8, 4, 800, delay, 12, seed=1)
    X = wpe.wpe(Y, taps=taps, delay=delay, iterations=1)
    # the last solve's normal equations: sum_t w_t Yt_t X_t^H = 0 with w from Y (one iteration)
    for f in range(Y.shape[0]):
        w = wpe.get_power_inverse(Y[f])
        Yt = wpe.build_y_tilde(Y[f], taps, delay)
        resid = (Yt * w) @ X[f].conj().T
        scale = np.abs(Yt * w) @ np.abs(X[f]).T
        assert np.abs(resid).max() < 1e-11 * scale.max()
    X3 = wpe.wpe(Y, taps=taps, delay=delay)
    e_in = np.sum(np.abs(Y - direct) ** 2)
    e_out = np.sum(np.abs(X3 - direct) ** 2)
    assert e_out < 0.5 * e_in, (e_out, e_in)


def test_errors():
    from pb_bss_b200 import wpe
    Y = _y((2, 4, 50))
    with pytest.raises(TypeError):
        wpe.wpe(Y.real)
    with pytest.raises(TypeError):
        wpe.get_power(torch.from_numpy(Y.real).cuda())
    with pytest.raises(NotImplementedError, match='96'):
        wpe.wpe(_y((2, 8, 50)), taps=13)
    with pytest.raises(NotImplementedError, match='30'):
        wpe.wpe(_y((2, 31, 50)), taps=1)
    with pytest.raises(NotImplementedError, match='30'):
        wpe.get_power(_y((2, 31, 50)))
    with pytest.raises(ValueError):
        wpe.wpe(Y, taps=0)
    with pytest.raises(ValueError):
        wpe.wpe(Y, delay=-1)
    with pytest.raises(ValueError):
        wpe.wpe(Y, statistics_mode='cropped')
    with pytest.raises(ValueError):
        wpe.wpe(Y, psd_context=-1)
    with pytest.raises(ValueError):
        wpe.get_power_inverse(Y, -2)
    with pytest.raises(ValueError):
        wpe.build_y_tilde(Y, 0, 1)
