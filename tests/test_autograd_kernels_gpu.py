"""The backward kernels of the mask-based beamforming chain against the long-double and mpmath references of
oracle/autograd_oracle.py, over the shapes where the kernels branch: every FFT size and frames-per-CTA value (fpc)
for stft / istft, D = 1..34 and K up to 19 for the PSD, D = 1..64 and every solve_kernel warp count for Souden MVDR,
T around the warp width and F past the grid's y limit for apply_beamforming_vector, n around the 8192-sample chunks
and every broadcast pattern for SI-SDR.  Everything runs through the public differentiable functions and
torch.autograd.grad, except the singular D > 40 Souden bin, whose forward raises.

Inputs span about 120 dB with runs of exact zeros where the bound is per frame or per sample, so a quiet frame is
held to its own size and an all-zero gradient frame must give exactly zero.  The module prints the values reached
(fpc per size, D / K / warps per kernel) and the worst error/bound ratio per group."""
import functools

import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import fft_oracle as FO
from oracle import linalg_oracle as LO
from oracle import synth
from oracle import transform_oracle as TO

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200 import _device, _lib
    from pb_bss_b200.evaluation import si_sdr
    from pb_bss_b200.extraction import beamformer as B
    from pb_bss_b200.transform import istft, stft

DEV = 'cuda'
SIZES = [64, 128, 256, 512, 1024, 2048, 4096]
TILINGS = [(size, fpc) for size in SIZES for fpc in (1 << i for i in range(13)) if fpc <= 4096 // size]
REACHED = {}
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for key in sorted(REACHED):
        print(f'{key}: reached {sorted(REACHED[key])}')
    for group in sorted(WORST):
        print(f'{group}: worst error/bound {WORST[group]:.3g}')


def _reach(key, value):
    REACHED.setdefault(key, set()).add(value)


def _note(group, ratio):
    r = np.asarray(ratio, dtype=np.float64)
    if r.size:
        WORST[group] = max(WORST.get(group, 0.0), float(r.max()))
    assert (r <= 1).all(), f'{group}: error/bound {r.max():.3g}'


def _t(a, grad=True, dtype=None):
    return torch.tensor(a, device=DEV, dtype=dtype, requires_grad=grad)


def _np(x):
    return x.detach().cpu().numpy()


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


@functools.lru_cache(maxsize=None)
def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _fpc(size, rows, T):
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
    guess = (T - 1) * shift + wl - (2 * (wl - shift) if fading else 0)
    for n in range(max(guess - 2 * shift, 0), max(guess + 2 * shift, 0) + 1):
        if TO.num_frames(n, size, shift, wl, fading, pad) == T:
            return n
    return None


def _spectra(rows, T, size, seed):
    """Random gradient spectra spanning 120 dB from frame to frame, every fifth frame exactly zero."""
    rng = np.random.default_rng(seed)
    X = _cplx(rng, rows, T, size // 2 + 1)
    X *= 10.0 ** (-6 * rng.random((rows, T, 1)))
    X[:, 2::5] = 0
    return X


# ---- stft backward: the inverse body on G^ (stft_backward_kernel) and the overlap-add --------------------------------
def _check_stft_backward(rows, n, size, shift, wl, fading, pad, seed, group):
    """grad x of stft (float64 against the long-double transpose, per sample) and of float32 input (the float64
    gradient rounded once: the backward does not read x)."""
    x = FO.spread_signal((rows, n), wl, seed)
    T = TO.num_frames(n, size, shift, wl, fading, pad)
    G = _spectra(rows, T, size, seed + 1)
    Gd = torch.from_numpy(G).to(DEV)
    grads = []
    for dtype in (torch.float64, torch.float32):
        xd = _t(x, dtype=dtype)
        (gx,) = torch.autograd.grad(stft(xd, size=size, shift=shift, window_length=wl, fading=fading, pad=pad), xd, Gd)
        assert gx.dtype == dtype
        grads.append(gx)
    assert torch.equal(grads[1], grads[0].to(torch.float32))
    ref, scale = AO.stft_grad_parts(G, n, size, shift, wl, fading)
    _note(group, FO.inverse_ratio(_np(grads[0]), ref, scale, size))
    return grads[0]


@pytest.mark.parametrize('size,fpc', TILINGS)
def test_stft_backward_at_every_tiling(size, fpc):
    """Last tile full, holding one frame and holding fpc - 1 frames; fading and pad both ways."""
    shift, wl = size // 4, size
    for last in sorted({0, 1 % fpc, (fpc - 1) % fpc}):
        T = 4 * fpc + last
        rows = _rows_for(size, T, fpc)
        assert rows is not None, (size, T, fpc)
        assert _fpc(size, rows, T) == fpc
        _reach(f'stft backward size {size:4d} fpc', fpc)
        for fading in (True, False):
            for pad in (True, False):
                n = _length(T, size, shift, wl, fading, pad)
                assert n is not None
                _check_stft_backward(rows, n, size, shift, wl, fading, pad, size * fpc + last, 'stft backward')


@pytest.mark.parametrize('size', SIZES)
def test_stft_backward_odd_window_lengths_and_extreme_shifts(size):
    """wl = 1 (the j + 1 < wl packing edge), 63 and size - 1 with shift = 1 and shift = wl."""
    for wl in (1, 63, size - 1):
        for shift in sorted({1, wl}):
            n = wl + (100 if shift == 1 else 6 * size)
            for fading in (True, False):
                _check_stft_backward(3, n, size, shift, wl, fading, True, size + wl + shift, 'stft backward, odd wl')


def test_stft_backward_tail_without_pad_is_exactly_zero():
    """pad=False drops the samples past the last full frame: their gradient is exactly 0 (with fading, only a shift
    above wl - shift leaves samples uncovered)."""
    size, shift = 256, 192
    for fading in (True, False):
        n = 20 * shift + 37
        T = TO.num_frames(n, size, shift, size, fading, False)
        covered = (T - 1) * shift + size - (size - shift if fading else 0)
        assert covered < n
        gx = _check_stft_backward(2, n, size, shift, size, fading, False, 7, 'stft backward')
        assert (gx[:, covered:] == 0).all()
        assert (gx[:, :covered] != 0).any()


def test_stft_backward_past_the_overlap_add_grid_cap():
    """rows n above 4 * 32 * SMs * 256: the overlap-add kernel strides."""
    size = shift = 1024
    rows = 2
    n = (4 * 32 * _sms() * 256) // rows + 3 * size + 5
    _check_stft_backward(rows, n, size, shift, size, False, True, 11, 'stft backward, grid cap')


# ---- istft backward: the forward body on the synthesis-windowed gradient (istft_backward_kernel) ---------------------
def _check_istft_backward(rows, T, size, shift, wl, fading, seed, group):
    X = _t(_spectra(rows, T, size, seed))
    out = istft(X, size=size, shift=shift, window_length=wl, fading=fading)
    g = FO.spread_signal(tuple(out.shape), wl, seed + 1)
    (gX,) = torch.autograd.grad(out, X, torch.from_numpy(g).to(DEV))
    assert gX.dtype == torch.complex128
    _note(group, FO.forward_ratio(_np(gX), AO.istft_grad(g, T, size, shift, wl, fading), size)[0])
    return gX


@pytest.mark.parametrize('size,fpc', TILINGS)
def test_istft_backward_at_every_tiling(size, fpc):
    for last in sorted({0, 1 % fpc, (fpc - 1) % fpc}):
        T = 4 * fpc + last
        rows = _rows_for(size, T, fpc)
        assert rows is not None, (size, T, fpc)
        _reach(f'istft backward size {size:4d} fpc', _fpc(size, rows, T))
        for shift in (size // 4, size):
            for fading in (True, False):
                _check_istft_backward(rows, T, size, shift, size, fading, size * fpc + last + shift, 'istft backward')


@pytest.mark.parametrize('size', SIZES)
def test_istft_backward_odd_window_lengths_and_extreme_shifts(size):
    for wl in (1, 63, size - 1):
        for shift in sorted({1, wl}):
            for fading in (True, False):
                _check_istft_backward(3, 40, size, shift, wl, fading, size + wl, 'istft backward, odd wl')


def test_istft_backward_of_an_empty_output():
    """fading, T = 1 and shift < wl / 2: no output sample, so the gradient is exactly zero."""
    size, shift = 256, 64
    X = _t(_spectra(3, 1, size, 3))
    out = istft(X, size=size, shift=shift, fading=True)
    assert out.shape == (3, 0)
    (gX,) = torch.autograd.grad(out.sum(), X)
    assert gX.shape == X.shape and (gX == 0).all()


# ---- the FFT backward kernels: invariants ----------------------------------------------------------------------------
@pytest.mark.parametrize('size', SIZES)
def test_fft_backward_row_does_not_depend_on_the_tiling(size):
    """A row's gradient alone (smallest fpc) and inside 2 SMs rows (largest fpc): bitwise equal."""
    shift, n, R = size // 4, 8 * size + 5, 2 * _sms()
    T = TO.num_frames(n, size, shift, size, True, True)
    assert _fpc(size, R, T) == 4096 // size and (_fpc(size, 1, T) < 4096 // size or size == 4096)
    x = _t(FO.spread_signal((R, n), size, size))
    G = torch.from_numpy(_spectra(R, T, size, size)).to(DEV)
    (gb,) = torch.autograd.grad(stft(x, size=size, shift=shift), x, G)
    x1 = _t(_np(x[5:6]))
    (g1,) = torch.autograd.grad(stft(x1, size=size, shift=shift), x1, G[5:6].clone())
    assert torch.equal(g1[0], gb[5])
    X = _t(_spectra(R, T, size, size + 1))
    out = istft(X, size=size, shift=shift)
    go = torch.from_numpy(FO.spread_signal(tuple(out.shape), size, 3)).to(DEV)
    (gXb,) = torch.autograd.grad(out, X, go)
    X1 = _t(_np(X[5:6]))
    (gX1,) = torch.autograd.grad(istft(X1, size=size, shift=shift), X1, go[5:6].clone())
    assert torch.equal(gX1[0], gXb[5])


@pytest.mark.parametrize('dtype', [torch.float64, torch.float32])
def test_fft_backward_layout(dtype):
    """stft over axis 0 of a (n, rows) signal, and a transposed view, against contiguous (rows, n) copies: bitwise,
    in the input's dtype; istft of a permuted spectrum view against its contiguous copy."""
    size, shift = 256, 64
    x = _t(FO.spread_signal((3, 4000), size, 5).T.copy(), dtype=dtype)      # (n, rows)
    X0 = stft(x, size=size, shift=shift, axis=0)                            # (T, F, rows)
    G = torch.from_numpy(_spectra(3, X0.shape[0], size, 6)).to(DEV)        # (rows, T, F)
    (g0,) = torch.autograd.grad(X0, x, G.permute(1, 2, 0))
    xc = _t(_np(x).T.copy(), dtype=dtype)
    (gc,) = torch.autograd.grad(stft(xc, size=size, shift=shift), xc, G)
    assert g0.dtype == dtype and torch.equal(g0.T, gc)
    xv = _t(_np(x), dtype=dtype)
    (gv,) = torch.autograd.grad(stft(xv.T, size=size, shift=shift), xv, G)  # non-contiguous (rows, n) view
    assert torch.equal(gv.T, gc)
    Xs = _t(_spectra(2, 30, size, 8).transpose(1, 0, 2).copy())            # (T, rows, F)
    out = istft(Xs.transpose(0, 1), size=size, shift=shift)
    go = torch.from_numpy(FO.spread_signal(tuple(out.shape), size, 9)).to(DEV)
    (gs,) = torch.autograd.grad(out, Xs, go)
    Xc = _t(_np(Xs).transpose(1, 0, 2).copy())
    (gcs,) = torch.autograd.grad(istft(Xc, size=size, shift=shift), Xc, go)
    assert torch.equal(gs.transpose(0, 1), gcs)


# ---- PSD (psd_backward_kernel) ---------------------------------------------------------------------------------------
PSD_K = (1, 2, 3, 18, 19)
PSD_T = (1, 63, 64, 65, 129, 1000)


def _psd_smem(D, K):
    return (D * D + 2 * D * 64) * 16 + 24 * K


def _check_psd(y, m, normalize, seed, group):
    """y (F, D, T) complex64 / complex128, m (F, K, T) or None through the public function."""
    F, D, T = y.shape
    K = 1 if m is None else m.shape[1]
    yd = _t(y)
    md = None if m is None else _t(m)
    phi = B.get_power_spectral_density_matrix(yd, md, normalize=normalize)
    G = _cplx(np.random.default_rng(seed), *phi.shape)
    inputs = (yd,) if md is None else (yd, md)
    grads = torch.autograd.grad(phi, inputs, torch.from_numpy(G).to(DEV))
    gy_ref, gm_ref, by, bm = AO.psd_grad_ld(y, m, G.reshape(F, K, D, D), normalize)
    assert grads[0].dtype == yd.dtype
    _note(group + ' grad y', AO._ratio(AO._err(_np(grads[0]), gy_ref), AO._rounded(by, gy_ref, y.dtype)))
    if md is not None:
        _note(group + ' grad mask', AO._ratio(AO._err(_np(grads[1]), gm_ref), bm))
    _reach(f'{group} D', D)
    _reach(f'{group} K', K)
    _reach(f'{group} T', T)
    if _psd_smem(D, K) > 48 * 1024:
        _reach(f'{group} D with more than 48 KB of shared memory', D)


def _psd_inputs(F, D, K, T, seed, dtype=np.complex128):
    rng = np.random.default_rng(seed)
    y = (_cplx(rng, F, D, T) * 10.0 ** (-2 * rng.random((F, 1, T)))).astype(dtype)
    m = rng.uniform(size=(F, K, T))
    if K >= 2:
        m[0, 0] *= 1e-11 / m[0, 0].sum()  # sums below 1e-10: the clamped branch
        m[F - 1, K - 1] = 0.0              # exactly zero
    return y, m


@pytest.mark.parametrize('D', range(1, 35))
def test_psd_backward_over_d_k_and_t(D):
    """Every K in PSD_K at every D; T cycles through PSD_T (every T at D = 20, 21 and 34 with K = 2 and 19)."""
    for i, K in enumerate(PSD_K):
        for T in (PSD_T if D in (20, 21, 34) and K in (2, 19) else (PSD_T[(D + i) % len(PSD_T)],)):
            y, m = _psd_inputs(2, D, K, T, 100 * D + K)
            _check_psd(y, m, True, D + K + T, 'psd')


@pytest.mark.parametrize('D', [1, 2, 7, 20, 21, 33, 34])
def test_psd_backward_without_mask_without_normalize_and_complex64(D):
    for T in (1, 64, 65, 1000):
        y, m = _psd_inputs(2, D, 3, T, D + T)
        _check_psd(y, None, True, D, 'psd, no mask')
        _check_psd(y, m, False, D + 1, 'psd, no normalize')
        _check_psd(y.astype(np.complex64), m, True, D + 2, 'psd, complex64')


def test_psd_backward_broadcast_mask_and_source_dim():
    """A (K, T) mask broadcast over F sums its per-bin gradients; source_dim = 0 (mask (K, F, T)) and a leading
    batch dim (observation (2, 3, D, T)) give the gradients of contiguous (F, K, T) copies bitwise."""
    F, D, K, T = 5, 4, 3, 70
    y, m = _psd_inputs(F, D, K, T, 1)
    rng = np.random.default_rng(2)
    G = _cplx(rng, F, K, D, D)
    Gd = torch.from_numpy(G).to(DEV)
    mb = _t(m[:1])                                                         # (1, K, T)
    yd = _t(y)
    gy, gm = torch.autograd.grad(B.get_power_spectral_density_matrix(yd, mb), (yd, mb), Gd)
    gy_ref, gm_ref, by, bm = AO.psd_grad_ld(y, np.broadcast_to(m[:1], (F, K, T)), G)
    _note('psd, broadcast mask grad y', AO._ratio(AO._err(_np(gy), gy_ref), by))
    gm_sum, bm_sum = AO.reduce_rows(gm_ref, bm, np.zeros(F, dtype=np.int64), 1)
    _note('psd, broadcast mask grad mask', AO._ratio(AO._err(_np(gm), gm_sum), bm_sum))
    # source_dim = 0: mask (K, F, T), PSD (K, F, D, D)
    ms = _t(m.transpose(1, 0, 2).copy())
    mc = _t(m)
    g0 = torch.autograd.grad(B.get_power_spectral_density_matrix(yd, ms, source_dim=0), (yd, ms), Gd.transpose(0, 1))
    gc = torch.autograd.grad(B.get_power_spectral_density_matrix(yd, mc), (yd, mc), Gd)
    assert torch.equal(g0[0], gc[0]) and torch.equal(g0[1].transpose(0, 1), gc[1])
    # permuted observation view and leading batch dims
    yt = _t(y.transpose(0, 2, 1).copy())                                  # (F, T, D)
    gt = torch.autograd.grad(B.get_power_spectral_density_matrix(yt.transpose(1, 2), mc), (yt, mc), Gd)
    assert torch.equal(gt[0].transpose(1, 2), gc[0]) and torch.equal(gt[1], gc[1])
    y6, m6 = _psd_inputs(6, D, K, T, 3)
    y23, m23 = _t(y6.reshape(2, 3, D, T)), _t(m6.reshape(2, 3, K, T))
    G6 = torch.from_numpy(_cplx(rng, 6, K, D, D)).to(DEV)
    g23 = torch.autograd.grad(B.get_power_spectral_density_matrix(y23, m23), (y23, m23), G6.reshape(2, 3, K, D, D))
    y6d, m6d = _t(y6), _t(m6)
    g6 = torch.autograd.grad(B.get_power_spectral_density_matrix(y6d, m6d), (y6d, m6d), G6)
    assert torch.equal(g23[0].reshape(6, D, T), g6[0]) and torch.equal(g23[1].reshape(6, K, T), g6[1])


def test_psd_backward_bin_does_not_depend_on_the_batch():
    F, D, K, T = 257, 6, 2, 130
    y, m = _psd_inputs(F, D, K, T, 4)
    G = torch.from_numpy(_cplx(np.random.default_rng(5), F, K, D, D)).to(DEV)
    yd, md = _t(y), _t(m)
    gb = torch.autograd.grad(B.get_power_spectral_density_matrix(yd, md), (yd, md), G)
    for f in (0, 100, 256):
        y1, m1 = _t(y[f:f + 1]), _t(m[f:f + 1])
        g1 = torch.autograd.grad(B.get_power_spectral_density_matrix(y1, m1), (y1, m1), G[f:f + 1].clone())
        assert torch.equal(g1[0][0], gb[0][f]) and torch.equal(g1[1][0], gb[1][f])


# ---- Souden MVDR (souden_backward_kernel, solve_kernel on N^H, souden_noise_backward_kernel) -----------------------
def _solve_warps(D):
    """solve_kernel's warps per CTA for the D right-hand sides of the backward solve (solve_smem_per_warp, warps_for)."""
    b = (D * D + D * D) * 16
    if D <= 40:
        b += (2 * D * D + D * D) * 16 + ((D + 1) // 2) * 6 * 8
    b = (b + 15) & ~15
    return min(max((96 * 1024) // b, 1), 4)


def _souden_inputs(n, D, seed):
    rng = np.random.default_rng(seed)
    t = synth.pos_def_hermitian(n, D, D, seed=seed)
    # a non-Hermitian noise matrix: the backward solves with N^H, not the Hermitian part
    nz = synth.pos_def_hermitian(n, D, D, seed=seed + 1) + 0.05 * _cplx(rng, n, D, D)
    return t, nz, _cplx(rng, n, D)


def _souden_grads(t, nz, g, ref, eps=None):
    td, nd = _t(t), _t(nz)
    w = B.get_mvdr_vector_souden(td, nd, ref_channel=ref, eps=eps)
    return torch.autograd.grad(w, (td, nd), torch.from_numpy(np.asarray(g)).to(DEV))


def _check_souden(t, nz, g, ref, group, eps=None, high_precision=False):
    gt, gn = _souden_grads(t, nz, g, ref, eps)
    _note(group, AO.souden_ratio(_np(gt), _np(gn),
                                 AO.souden_grad_ref(t, nz, ref, g, eps, high_precision=high_precision)))
    return gt, gn


@pytest.mark.parametrize('D', range(1, 65))
def test_souden_backward_over_d(D):
    """n = 7 bins: not a multiple of 2, 3 or 4 warps per CTA, so the last CTA is partial."""
    t, nz, g = _souden_inputs(7, D, D)
    _check_souden(t, nz, g, D // 2, 'souden float64')
    _reach('souden D', D)
    _reach('souden solve warps per CTA', _solve_warps(D))


@pytest.mark.parametrize('D', [2, 8, 17, 18, 33, 41])
def test_souden_backward_ill_conditioned_against_mpmath(D):
    """kappa(N) = 1e12, unitarily (conditioned, positive definite) and by grading (graded, 6 decades), against
    mpmath solves; both kinds below D = 30, one of them above."""
    pytest.importorskip('mpmath')
    rng = np.random.default_rng(D)
    N = [LO.conditioned(D, 1e12, rng, hermitian=True), LO.graded(D, rng, decades=6.0)]
    N = np.stack(N if D < 30 else N[D % 2:][:1])  # mpmath's solves take about 20 s per bin at D = 33
    X = np.stack([LO.from_spectrum(rng.uniform(0.5, 1.0, D), rng) for _ in range(len(N))])
    g = _cplx(rng, len(N), D)
    _check_souden(X, N, g, 0, 'souden mpmath', high_precision=True)
    _reach('souden mpmath D', D)


def test_souden_backward_trace_at_or_below_eps():
    """A user eps: bins with 0 < tr Phi <= eps and with a negative trace take grad Phi = g e_r^T / eps."""
    D, eps = 5, 1e-3
    t, nz, g = _souden_inputs(4, D, 3)
    t[1] *= 0.5 * eps / np.trace(np.linalg.solve(nz[1], t[1])).real
    t[2] = -t[2]
    lam = np.trace(np.linalg.solve(nz, t), axis1=-2, axis2=-1).real
    assert 0 < lam[1] <= eps and lam[2] < 0 and lam[0] > eps and lam[3] > eps
    _check_souden(t, nz, g, 1, 'souden tr <= eps', eps=eps)


def test_souden_backward_broadcast_noise():
    """One (D, D) noise matrix for F bins: its gradient sums the bins'."""
    F, D = 9, 6
    t, nz, g = _souden_inputs(F, D, 4)
    td, nd = _t(t), _t(nz[0])
    w = B.get_mvdr_vector_souden(td, nd, ref_channel=2)
    gt, gn = torch.autograd.grad(w, (td, nd), torch.from_numpy(g).to(DEV))
    gX, gN, bX, bN = AO.souden_grad_ref(t, np.broadcast_to(nz[0], t.shape), 2, g)
    _note('souden broadcast noise', AO._ratio(np.sqrt((AO._err(_np(gt), gX) ** 2).sum((-1, -2))), bX))
    err = np.sqrt((AO._err(_np(gn), gN.sum(0)) ** 2).sum()).astype(np.float64)
    _note('souden broadcast noise', AO._ratio(err, bN.sum() + AO.gamma(F) * np.abs(gN).sum()))


def _souden_backward_entry(phi, nz, g, ref, eps):
    """pbb_souden_backward on device tensors: the only way to a singular bin at D > 40, whose forward raises."""
    n, D = phi.shape[0], phi.shape[-1]
    gt = torch.empty((n, D, D), dtype=torch.complex128, device=DEV)
    gn = torch.empty_like(gt)
    _lib.check(_lib.load().pbb_souden_backward(_device.ptr(phi), _device.ptr(nz), _device.ptr(g), n, D, ref, eps,
                                               _device.ptr(gt), _device.ptr(gn), _device.stream_ptr()),
               'pbb_souden_backward')
    return gt, gn


@pytest.mark.parametrize('D', [3, 40, 41, 64])
def test_souden_backward_nan_only_in_singular_and_non_finite_bins(D):
    """An exactly singular N (bin 2) and an N holding inf (bin 4): NaN gradients there, and the other bins bitwise
    what they are without those bins."""
    n = 7
    t, nz, g = _souden_inputs(n, D, D + 7)
    bad = nz.copy()
    bad[2] = 0.0
    bad[4, 0, 1] = np.inf
    good = [0, 1, 3, 5, 6]
    if D <= 40:
        gt, gn = _souden_grads(t, bad, g, 1)
    else:
        # the forward raises on the singular bin at D > 40 (no minimum-norm fallback)
        # Phi finite everywhere, so the NaN must come from the solve with the singular or non-finite N^H
        phi = torch.from_numpy(np.linalg.solve(nz, t)).to(DEV)
        gt, gn = _souden_backward_entry(phi, torch.from_numpy(bad).to(DEV), torch.from_numpy(g).to(DEV), 1,
                                        float(np.finfo(np.float64).tiny))
        gt_ok, gn_ok = _souden_backward_entry(phi[good].contiguous(), torch.from_numpy(nz[good]).to(DEV),
                                              torch.from_numpy(g[good]).to(DEV), 1, float(np.finfo(np.float64).tiny))
        assert torch.equal(gt[good], gt_ok) and torch.equal(gn[good], gn_ok)
    for x in (gt, gn):
        assert torch.isnan(x[[2, 4]]).all()
        assert torch.isfinite(x[good]).all()
    if D <= 40:
        gt_ok, gn_ok = _souden_grads(t[good], nz[good], g[good], 1)
        assert torch.equal(gt[good], gt_ok) and torch.equal(gn[good], gn_ok)


def test_souden_backward_bin_does_not_depend_on_its_place_in_the_cta():
    for D in (6, 18, 22, 30):
        warps = _solve_warps(D)
        t, nz, g = _souden_inputs(2 * warps + 1, D, D + 11)
        gt, gn = _souden_grads(t, nz, g, 0)
        for m in range(warps):
            g1 = _souden_grads(t[m:m + 1], nz[m:m + 1], g[m:m + 1], 0)
            assert torch.equal(g1[0][0], gt[m]) and torch.equal(g1[1][0], gn[m]), (D, m)


# ---- apply_beamforming_vector (apply_bf_vector_backward_kernel, apply_bf_mix_backward_kernel) ----------------------
def _check_apply(v, y, g, gv, gy, group):
    """v (B, F, D), y (F, D, T), g (B, F, T) against the kernels' gradients in the same layouts."""
    rv, ry, bv, by = AO.apply_grad_ld(v, y, g)
    _note(group + ' grad vector', AO._ratio(AO._err(gv, rv), bv))
    _note(group + ' grad mix', AO._ratio(AO._err(gy, ry), AO._rounded(by, ry, y.dtype)))


@pytest.mark.parametrize('D', range(1, 30))
def test_apply_backward_over_d_and_t(D):
    for T in (1, 31, 32, 33, 1000):
        rng = np.random.default_rng(D * T)
        F = 3
        v, y, g = _cplx(rng, F, D), _cplx(rng, F, D, T), _cplx(rng, F, T)
        for dtype in (np.complex128, np.complex64) if T in (33, 1000) else (np.complex128,):
            vd, yd = _t(v), _t(y.astype(dtype))
            gv, gy = torch.autograd.grad(B.apply_beamforming_vector(vd, yd), (vd, yd), torch.from_numpy(g).to(DEV))
            assert gy.dtype == yd.dtype and gv.dtype == torch.complex128
            _check_apply(v[None], y.astype(dtype), g[None], _np(gv)[None], _np(gy), 'apply')
        _reach('apply D', D)
        _reach('apply T', T)


def test_apply_backward_past_the_grid_y_limit():
    """F = 70 000 bins: the mix gradient strides bins past gridDim.y = 65535."""
    rng = np.random.default_rng(7)
    F, D, T = 70000, 2, 3
    v, y, g = _cplx(rng, F, D), _cplx(rng, F, D, T), _cplx(rng, F, T)
    vd, yd = _t(v), _t(y)
    gv, gy = torch.autograd.grad(B.apply_beamforming_vector(vd, yd), (vd, yd), torch.from_numpy(g).to(DEV))
    _check_apply(v[None], y, g[None], _np(gv)[None], _np(gy), 'apply, F > 65535')
    _reach('apply F', F)


@pytest.mark.parametrize('Bn', [2, 7, 20])
def test_apply_backward_shared_mix_with_broadcast_dim_not_leading(Bn):
    """vector (F, B, D) and one mix (F, 1, D, T): B beamformers share the mix along a dim that is not leading."""
    rng = np.random.default_rng(Bn)
    F, D, T = 5, 4, 100
    for dtype in (np.complex128, np.complex64):
        v, y, g = _cplx(rng, F, Bn, D), _cplx(rng, F, 1, D, T).astype(dtype), _cplx(rng, F, Bn, T)
        vd, yd = _t(v), _t(y)
        out = B.apply_beamforming_vector(vd, yd)
        assert out.shape == (F, Bn, T)
        gv, gy = torch.autograd.grad(out, (vd, yd), torch.from_numpy(g).to(DEV))
        assert gy.dtype == yd.dtype
        _check_apply(v.transpose(1, 0, 2), y[:, 0], g.transpose(1, 0, 2), _np(gv).transpose(1, 0, 2),
                     _np(gy)[:, 0], 'apply, shared mix')
    _reach('apply shared B', Bn)


def test_apply_backward_layout():
    """Leading batch dims and a permuted mix view give the gradients of contiguous (F, D, T) copies bitwise."""
    rng = np.random.default_rng(8)
    D, T = 5, 40
    v, y, g = _cplx(rng, 2, 3, D), _cplx(rng, 2, 3, D, T), _cplx(rng, 2, 3, T)
    vd, yd = _t(v), _t(y)
    gd = torch.from_numpy(g).to(DEV)
    g23 = torch.autograd.grad(B.apply_beamforming_vector(vd, yd), (vd, yd), gd)
    vf, yf = _t(v.reshape(6, D)), _t(y.reshape(6, D, T))
    gf = torch.autograd.grad(B.apply_beamforming_vector(vf, yf), (vf, yf), gd.reshape(6, T))
    assert torch.equal(g23[0].reshape(6, D), gf[0]) and torch.equal(g23[1].reshape(6, D, T), gf[1])
    yt = _t(y.reshape(6, D, T).transpose(0, 2, 1).copy())                   # (F, T, D)
    gt = torch.autograd.grad(B.apply_beamforming_vector(vf, yt.transpose(1, 2)), (vf, yt), gd.reshape(6, T))
    assert torch.equal(gt[0], gf[0]) and torch.equal(gt[1].transpose(1, 2), gf[1])


# ---- SI-SDR (si_sdr_backward_row_kernel, si_sdr_backward_kernel) -----------------------------------------------------
def _own_index(own_shape, lead):
    """The own row each row of the broadcast shape reads."""
    return np.broadcast_to(np.arange(int(np.prod(own_shape))).reshape(own_shape), lead).reshape(-1)


def _check_si_sdr(r, e, seed, group):
    """r and e in their own shapes (broadcastable, last axes n or 1) against the per-row references summed over the
    rows that share an own row."""
    rd, ed = _t(r), _t(e)
    s = si_sdr(rd, ed)
    g = np.random.default_rng(seed).standard_normal(tuple(s.shape))
    gr, ge = torch.autograd.grad(s, (rd, ed), torch.from_numpy(g).to(DEV))
    shape = np.broadcast_shapes(r.shape, e.shape)
    lead, n = shape[:-1], shape[-1]
    rb = np.broadcast_to(r, shape).reshape(-1, n)
    eb = np.broadcast_to(e, shape).reshape(-1, n)
    rr, re, br, be = AO.si_sdr_grad_ld(rb, eb, g.reshape(-1))
    for got, x, ref, bnd in ((gr, r, rr, br), (ge, e, re, be)):
        xs = x.reshape((1,) * (len(shape) - x.ndim) + x.shape)
        own = xs.shape[:-1]
        ref_own, b_own = AO.reduce_rows(ref, bnd, _own_index(own, lead), int(np.prod(own)))
        if xs.shape[-1] != n:  # a broadcast last axis: one sample receives the sum over n
            ref_own, b_own = ref_own.sum(-1, keepdims=True), b_own.sum(-1, keepdims=True) + AO.gamma(n) * np.abs(
                ref_own).astype(np.float64).sum(-1, keepdims=True)
        _note(group, AO._ratio(AO._err(_np(got).reshape(ref_own.shape), ref_own), b_own))
    return gr, ge


def _si_sdr_rows(rows, n, seed):
    rng = np.random.default_rng(seed)
    r = rng.standard_normal((rows, n))
    e = r * rng.uniform(0.5, 2.0, (rows, 1)) + rng.uniform(0.05, 1.0, (rows, 1)) * rng.standard_normal((rows, n))
    return r, e


@pytest.mark.parametrize('n', [8191, 8192, 8193, 3 * 8192 + 1])
def test_si_sdr_backward_at_chunk_edges(n):
    r, e = _si_sdr_rows(3, n, n)
    _check_si_sdr(r, e, n, 'si_sdr')
    _reach('si_sdr n', n)


def test_si_sdr_backward_of_one_sample_is_non_finite_exactly_where_the_value_is():
    """n = 1: alpha r equals e up to rounding, so Q is 0 or of order u^2 |e|^2."""
    r, e = _si_sdr_rows(8, 1, 1)
    rd, ed = _t(r), _t(e)
    s = si_sdr(rd, ed)
    gr, ge = torch.autograd.grad(s, (rd, ed), torch.ones_like(s))
    finite = torch.isfinite(s)
    for x in (gr, ge):
        assert torch.equal(torch.isfinite(x[:, 0]), finite)
    _reach('si_sdr n', 1)


@pytest.mark.parametrize('pattern', ['both broadcast', 'reference 1-D', 'broadcast last axis', 'estimation broadcast'])
def test_si_sdr_backward_broadcast(pattern):
    n = 8193
    rng = np.random.default_rng(len(pattern))
    if pattern == 'both broadcast':
        r, e = rng.standard_normal((3, 1, n)), rng.standard_normal((1, 4, n))
    elif pattern == 'reference 1-D':
        r = rng.standard_normal(n)
        e = r * rng.uniform(0.5, 2.0, (5, 1)) + 0.3 * rng.standard_normal((5, n))
    elif pattern == 'broadcast last axis':
        r, e = rng.standard_normal((4, 1)), rng.standard_normal((4, n)) + 1.0
    else:
        r, e = rng.standard_normal((6, n)), rng.standard_normal(n)
    _check_si_sdr(r, e, 3, f'si_sdr, {pattern}')


def test_si_sdr_backward_non_finite_rows():
    """r = 0 (nan), e = 2 r (inf) and e orthogonal to r (-inf) rows: non-finite gradients in exactly those rows."""
    r, e = _si_sdr_rows(6, 1000, 5)
    r[1] = 0.0
    e[3] = 2 * r[3]
    r[4] = 0.0
    r[4, 0] = 1.0
    e[4, 0] = 0.0
    rd, ed = _t(r), _t(e)
    s = si_sdr(rd, ed)
    assert torch.isnan(s[1]) and s[3] == float('inf') and s[4] == -float('inf')
    gr, ge = torch.autograd.grad(s, (rd, ed), torch.from_numpy(np.linspace(0.5, 1.5, 6)).to(DEV))
    for x in (gr, ge):
        assert (~torch.isfinite(x[[1, 3, 4]])).all()
        assert torch.isfinite(x[[0, 2, 5]]).all()
    ok = [0, 2, 5]
    _check_si_sdr(r[ok], e[ok], 6, 'si_sdr')


def test_si_sdr_backward_row_does_not_depend_on_the_batch_and_layout():
    r, e = _si_sdr_rows(9, 20000, 9)
    rd, ed = _t(r), _t(e)
    g = torch.linspace(-1, 1, 9, dtype=torch.float64, device=DEV)
    gb = torch.autograd.grad(si_sdr(rd, ed), (rd, ed), g)
    for i in (0, 4, 8):
        r1, e1 = _t(r[i]), _t(e[i])
        g1 = torch.autograd.grad(si_sdr(r1, e1), (r1, e1), g[i])
        assert torch.equal(g1[0], gb[0][i]) and torch.equal(g1[1], gb[1][i])
    et = _t(e.T.copy())                                                      # (n, rows): a transposed view
    gt = torch.autograd.grad(si_sdr(rd, et.T), (rd, et), g)
    assert torch.equal(gt[0], gb[0]) and torch.equal(gt[1].T, gb[1])


def test_si_sdr_backward_past_the_grid_cap():
    """rows n > 2^28 (2 GiB per operand): the element kernel's grid is capped at 2^20 CTAs and strides.  Three rows
    repeated: every copy's gradient is bitwise that of the three rows alone."""
    n, reps = 8192, 10923
    rows = 3 * reps
    assert rows * n > (1 << 20) * 256
    r, e = _si_sdr_rows(3, n, 12)
    r3, e3 = _t(r), _t(e)
    g3 = torch.tensor([0.5, -1.0, 2.0], dtype=torch.float64, device=DEV)
    small = torch.autograd.grad(si_sdr(r3, e3), (r3, e3), g3)
    rb = r3.detach().repeat(reps, 1).requires_grad_()
    eb = e3.detach().repeat(reps, 1).requires_grad_()
    big = torch.autograd.grad(si_sdr(rb, eb), (rb, eb), g3.repeat(reps))
    del rb, eb
    try:
        for a, b in zip(big, small):
            assert bool((a.view(reps, 3, n) == b).all())
    finally:
        del big
        torch.cuda.empty_cache()
