"""The FFT kernels against the long-double oracle of oracle/fft_oracle.py, at every size and every tiling the host can
choose: stft_kernel (plain, Griffin-Lim, MISI), istft_frames_kernel + overlap_add_kernel (csrc/fft.cuh) and the
four-step FFT of csrc/fft_large.cuh through SRMR's Hilbert envelopes.

Shapes are found with pbb_stft_frames_per_cta for this GPU's SM count, so every frames-per-CTA value (fpc) from 1 to
4096 / size runs, with the last tile full and partial.  Test signals span about 120 dB from frame to frame and carry
runs of exact zeros longer than a window: the bounds are per frame (forward) and per sample (inverse), so a quiet
frame is held to its own size, and a zero frame must come out exactly zero.  The bounds and constants are in
oracle/fft_oracle.py; the module prints the fpc values reached per size and the worst error/bound ratio per group."""
import functools

import numpy as np
import pytest

from oracle import fft_oracle as FO
from oracle import transform_oracle as TO

pytestmark = pytest.mark.gpu

SIZES = [64, 128, 256, 512, 1024, 2048, 4096]
TILINGS = [(size, fpc) for size in SIZES for fpc in (1 << i for i in range(13)) if fpc <= 4096 // size]
REACHED = {}
WORST = {}


class BoundExceeded(AssertionError):
    pass


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for size in sorted(REACHED):
        print(f'size {size}: fpc reached {sorted(REACHED[size])}')
    for group in sorted(WORST):
        print(f'{group}: worst error/bound {WORST[group]:.3f}')


def _note(group, ratio):
    r = np.asarray(ratio, dtype=np.float64)
    if r.size:
        WORST[group] = max(WORST.get(group, 0.0), float(r.max()))
    if not (r <= 1).all():
        raise BoundExceeded(f'{group}: error/bound {r.max():.3g}')


@functools.lru_cache(maxsize=None)
def _sms():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _fpc(size, rows, T):
    from pb_bss_b200 import _lib
    f = _lib.load().pbb_stft_frames_per_cta(size, rows, T, _sms())
    assert f > 0
    return f


def _rows_for(size, T, fpc):
    """The fewest rows at which T frames per row run at fpc frames per CTA (None if no row count does)."""
    for rows in range(1, 2 * _sms() + 1):
        f = _fpc(size, rows, T)
        if f == fpc:
            return rows
        if f > fpc:
            return None
    return None


def _length(T, size, shift, wl, fading, pad):
    """A signal length that gives T frames (None if none does)."""
    guess = (T - 1) * shift + wl - (2 * (wl - shift) if fading else 0)
    for n in range(max(guess - 2 * shift, 0), max(guess + 2 * shift, 0) + 1):
        if TO.num_frames(n, size, shift, wl, fading, pad) == T:
            return n
    return None


def _reach(size, rows, T):
    f = _fpc(size, rows, T)
    REACHED.setdefault(size, set()).add(f)
    return f


def _check_stft(x, size, shift, wl, fading, pad, group):
    from pb_bss_b200.transform import stft
    out = stft(x, size=size, shift=shift, window_length=wl, fading=fading, pad=pad)
    ref = FO.stft(x, size, shift, wl, fading, pad)
    assert out.shape == ref.shape and out.dtype == np.complex128
    _note(group, FO.forward_ratio(out, ref, size)[0])


# ---- STFT ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('size,fpc', TILINGS)
def test_stft_at_every_tiling(size, fpc):
    """Full last tile, one frame in it and fpc - 1 frames in it; float64 and float32; all fading / pad options."""
    shift, wl = size // 4, size
    for last in sorted({0, 1 % fpc, (fpc - 1) % fpc}):
        T = 4 * fpc + last
        rows = _rows_for(size, T, fpc)
        assert rows is not None, (size, T, fpc)
        assert _reach(size, rows, T) == fpc
        for fading in (True, False):
            for pad in (True, False):
                n = _length(T, size, shift, wl, fading, pad)
                assert n is not None
                x = FO.spread_signal((rows, n), wl, size * fpc + last)
                for dtype in (np.float64, np.float32):
                    _check_stft(x.astype(dtype), size, shift, wl, fading, pad, 'stft')


@pytest.mark.parametrize('size', SIZES)
def test_stft_odd_window_lengths_and_extreme_shifts(size):
    """wl = 1 (the j + 1 < wl packing edge), 63 and size - 1, with shift = 1 (a sample in up to wl frames) and
    shift = wl."""
    for wl in (1, 63, size - 1):
        for shift in sorted({1, wl}):
            n = wl + (100 if shift == 1 else 6 * size)
            for fading in ((True, False) if shift > 1 or wl <= 64 else (False,)):
                for pad in (True, False):
                    x = FO.spread_signal((3, n), wl, size + wl + shift)
                    _reach(size, 3, TO.num_frames(n, size, shift, wl, fading, pad) or 1)
                    _check_stft(x, size, shift, wl, fading, pad, 'stft, odd wl')


# ---- iSTFT -----------------------------------------------------------------------------------------------------------
def _spectra(rows, T, size, seed):
    """Random spectra spanning 120 dB from frame to frame, with every fifth frame exactly zero."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((rows, T, size // 2 + 1)) + 1j * rng.standard_normal((rows, T, size // 2 + 1))
    X *= 10.0 ** (-6 * rng.random((rows, T, 1)))
    X[:, 2::5] = 0
    return X


def _check_istft(X, size, shift, wl, fading, group):
    from pb_bss_b200.transform import istft
    out = istft(X, size=size, shift=shift, window_length=wl, fading=fading)
    ref, scale = FO.istft_parts(X, size, shift, wl, fading)
    assert out.shape == ref.shape
    _note(group, FO.inverse_ratio(out, ref, scale, size))


@pytest.mark.parametrize('size,fpc', TILINGS)
def test_istft_at_every_tiling(size, fpc):
    """T in {1, fpc - 1, fpc + 1, 2 fpc - 1} wherever some row count runs it at fpc; shift in {1, 3, size / 4, wl}."""
    ran = 0
    for T in sorted({t for t in (1, fpc - 1, fpc + 1, 2 * fpc - 1) if t >= 1}):
        rows = _rows_for(size, T, fpc)
        if rows is None:
            continue
        assert _reach(size, rows, T) == fpc
        X = _spectra(rows, T, size, size * fpc + T)
        for shift in (1, 3, size // 4, size):
            for fading in (True, False):
                _check_istft(X, size, shift, size, fading, 'istft')
        ran += 1
    assert ran >= 1


@pytest.mark.parametrize('size', SIZES)
def test_istft_odd_window_lengths(size):
    for wl in (1, 63, size - 1):
        X = _spectra(3, 40, size, size + wl)
        for shift in sorted({1, min(3, wl), wl}):
            for fading in (True, False):
                _check_istft(X, size, shift, wl, fading, 'istft, odd wl')


# ---- bitwise invariance under the tiling -----------------------------------------------------------------------------
@pytest.mark.parametrize('size', SIZES)
def test_a_row_does_not_depend_on_the_tiling(size):
    """A row alone and the same row inside a batch that runs at the largest fpc: bitwise equal (stft, istft and the
    Griffin-Lim step; MISI couples the rows)."""
    import torch
    from pb_bss_b200.transform import istft, stft
    from pb_bss_b200.transform.fourier import griffin_lim_stft
    shift, n, R = size // 4, 8 * size + 5, 2 * _sms()
    batch = FO.spread_signal((R, n), size, size)
    T = TO.num_frames(n, size, shift, size, True, True)
    assert _fpc(size, R, T) == 4096 // size and _fpc(size, 1, T) < 4096 // size or size == 4096
    xb = torch.from_numpy(batch).cuda()
    Xb = stft(xb, size=size, shift=shift)
    X1 = stft(xb[5:6].clone(), size=size, shift=shift)
    assert torch.equal(X1[0], Xb[5])
    assert torch.equal(istft(X1, size=size, shift=shift)[0], istft(Xb, size=size, shift=shift)[5])
    target = torch.from_numpy(_spectra(R, T, size, size)).cuda()
    ddb, db = griffin_lim_stft(xb, target, None, size, shift, True)
    dd1, d1 = griffin_lim_stft(xb[5:6].clone(), target[5:6].clone(), None, size, shift, True)
    assert torch.equal(dd1[0], ddb[5]) and torch.equal(d1[0], db[5])


# ---- Griffin-Lim / MISI ----------------------------------------------------------------------------------------------
def _assert_magnitude(d, X):
    """exp(i angle 0) = 1: X_dash = |X| + 0j where X_dash_dash is zero.  The imaginary part is exactly zero; the real
    part is CUDA's hypot, documented within 2 ulp of the exact |X| (it differs from NumPy's by an ulp or two at about
    1 % of the bins), so it is compared with |X| in long double."""
    ref = np.abs(np.asarray(X).astype(np.clongdouble))
    assert (d.imag == 0).all()
    ulps = (np.abs(d.real.astype(FO.LD) - ref) / np.spacing(ref.astype(np.float64))).astype(np.float64)
    assert ulps.max(initial=0.0) <= 2, f'{ulps.max()} ulp'


def _check_step(x_hat, X, y, size, shift, fading, group):
    import torch
    from pb_bss_b200.transform.fourier import griffin_lim_stft
    dd, d = griffin_lim_stft(torch.from_numpy(x_hat).cuda(), torch.from_numpy(X).cuda(),
                             None if y is None else torch.from_numpy(y).cuda(), size, shift, fading)
    dd, d = dd.cpu().numpy(), d.cpu().numpy()
    dd_ref, _ = FO.griffin_lim_step(x_hat, X, y, size, shift, fading)
    _note(group + ' X_dash_dash', FO.forward_ratio(dd, dd_ref, size)[0])
    _note(group + ' X_dash', FO.dash_ratio(d, X, dd_ref, size))
    zero = np.all(dd_ref == 0, axis=-1)
    assert zero.any()
    _assert_magnitude(d[zero], X[zero])


@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('K,misi', [(3, False), (1, True), (2, True), (3, True), (9, True), (17, True)])
def test_griffin_lim_and_misi_step(size, K, misi):
    shift, largest = size // 4, 4096 // size
    for target in sorted({1, largest}):
        # 24 frames: long enough for a zero run of 2 size + 8 samples, short enough for fpc = 1 at K = 17
        T = 24 if target == 1 else largest * -(-2 * _sms() // K)
        for fading in (True, False):
            n = _length(T, size, shift, size, fading, True)
            assert _reach(size, K, T) == target
            x_hat = FO.spread_signal((K, n), size, size + K + T)
            y = FO.spread_signal((1, n), size, size * K)[0] if misi else None
            X = _spectra(K, T, size, size + K)
            _check_step(x_hat, X, y, size, shift, fading, 'misi' if misi else 'griffin-lim')


# ---- four-step FFT: SRMR's Hilbert envelopes -------------------------------------------------------------------------
def _log2_fft(N):
    from pb_bss_b200 import _lib
    return _lib.load().pbb_srmr_fft_log2(N)


def _check_envelopes(x, nr=None):
    import torch
    from pb_bss_b200.evaluation import module_srmr as M
    rows, N = x.shape
    nr = np.full(rows, N) if nr is None else np.asarray(nr)
    y = torch.from_numpy(x[None].copy()).cuda()
    M._hilbert_envelopes(y, torch.from_numpy(nr.astype(np.int64)).cuda())
    out = y.cpu().numpy()[0]
    m = 1 << _log2_fft(N)
    for r in range(rows):
        _note('envelope', FO.envelope_ratio(out[r, :nr[r]], FO.analytic(x[r, :nr[r]]), m))


@pytest.mark.parametrize('logP', range(23))
def test_envelope_at_every_four_step_split(logP):
    """One N per log2 P (P = M / 2 points of the complex FFT): every P1 x P2 split and column width runs."""
    N = 1 if logP == 0 else 2 if logP == 1 else 3 * (1 << logP) // 4 + 1
    assert _log2_fft(N) - 1 == logP
    rows = 2 if logP < 20 else 1
    _check_envelopes(FO.spread_signal((rows, N), 64, logP, zero_runs=N > 1000))


@pytest.mark.parametrize('logP', [9, 16, 21])
def test_envelopes_of_a_group_with_different_lengths(logP):
    N = 3 * (1 << logP) // 4 + 1
    assert _log2_fft(N) - 1 == logP
    _check_envelopes(FO.spread_signal((4, N), 64, logP), nr=[N, N - 7, N // 3, 1])


# ---- zero-length signals ---------------------------------------------------------------------------------------------
def test_stft_of_a_zero_length_signal():
    import torch
    from pb_bss_b200.transform import stft
    for fading in (True, False):
        for pad in (True, False):
            ref = TO.stft(np.zeros((2, 0)), size=256, shift=64, fading=fading, pad=pad)
            for x in (np.zeros((2, 0)), torch.zeros((2, 0), dtype=torch.float64, device='cuda'),
                      np.zeros((2, 0), np.float32)):
                out = stft(x, size=256, shift=64, fading=fading, pad=pad)
                out = out if isinstance(out, np.ndarray) else out.cpu().numpy()
                assert out.shape == ref.shape and (out == 0).all()
    assert TO.stft(np.zeros((2, 0)), size=256, shift=64, fading=False).shape == (2, 1, 129)


@pytest.mark.parametrize('misi', [False, True])
def test_griffin_lim_step_of_a_zero_length_signal(misi):
    import torch
    from pb_bss_b200.transform import MISI, GriffinLim
    from pb_bss_b200.transform.fourier import griffin_lim_stft
    K, size, shift = 3, 256, 64
    for fading in (True, False):
        T = TO.num_frames(0, size, shift, size, fading, True)
        X = torch.from_numpy(_spectra(K, T, size, 7)).cuda()
        x_hat = torch.zeros((K, 0), dtype=torch.float64, device='cuda')
        y = torch.zeros(0, dtype=torch.float64, device='cuda') if misi else None
        dd, d = griffin_lim_stft(x_hat, X, y, size, shift, fading)
        assert torch.equal(dd, torch.zeros_like(dd))
        _assert_magnitude(d.cpu().numpy(), X.cpu().numpy())
    # the public class: first guess y / K of an empty mixture, then a step (istft of T = 3 frames is empty with
    # fading)
    m = (MISI if misi else GriffinLim)(_spectra(K, 3, size, 8), np.zeros(0), first_guess='y', size=size, shift=shift,
                                       fading=True)
    m.step()
    assert m.x_hat.shape == (K, 0) and (m.X_dash_dash == 0).all()


# ---- the bounds can fail ---------------------------------------------------------------------------------------------
@pytest.mark.xfail(strict=True, raises=BoundExceeded,
                   reason='a twiddle table off by 1e-13 in its sines must break the forward bound')
def test_forward_bound_sees_a_perturbed_twiddle_table(monkeypatch):
    """sin (1 + 1e-13) in the cached table: test_stft_matches_oracle's per-row 1e-12 tolerance still passes, the
    per-frame bound must not."""
    from pb_bss_b200 import _device
    from pb_bss_b200.transform import fourier, stft
    size, shift = 1024, 256
    bad = fourier._twiddle(size).clone()
    bad[:, 1] *= 1 + 1e-13
    monkeypatch.setitem(fourier._twiddles, (size, _device.device()), bad)
    x = np.random.default_rng(1).standard_normal((3, 6 * size + 17))
    out = stft(x, size=size, shift=shift)
    ref = TO.stft(x, size=size, shift=shift)
    scale = np.abs(ref).reshape(3, -1).max(axis=-1)[:, None, None]
    assert (np.abs(out - ref) <= 1e-12 * scale).all()
    ratio, _ = FO.forward_ratio(out, FO.stft(x, size, shift), size)
    if not (ratio <= 1).all():
        raise BoundExceeded(f'error/bound {ratio.max():.3g}')
