"""oracle/autograd_oracle.py on the CPU: its torch forwards equal the NumPy oracles, and the closed-form gradients that
the device backward passes implement (include/pbb.h) equal torch autograd of the restatement in float64."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
from oracle import fft_oracle as FO
from oracle import pb_bss_oracle as O
from oracle import sxr_oracle as SO
from oracle import synth
from oracle import transform_oracle as TO


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a), np.asarray(b)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize('n, size, shift, wl, fading, pad', [
    (1000, 128, 32, None, True, True), (1000, 128, 32, None, False, False), (997, 128, 48, 96, True, False),
    (700, 64, 16, 40, False, True), (30, 128, 32, None, True, True)])
def test_stft_istft_forwards_match_numpy(n, size, shift, wl, fading, pad):
    x = np.random.default_rng(0).standard_normal((2, n))
    X = AO.stft(torch.from_numpy(x), size, shift, window_length=wl, fading=fading, pad=pad)
    ref = TO.stft(x, size, shift, window_length=wl, fading=fading, pad=pad)
    _close(X.numpy(), ref)
    _close(AO.istft(X, size, shift, window_length=wl, fading=fading).numpy(),
           TO.istft(ref, size, shift, window_length=wl, fading=fading))


@pytest.mark.parametrize('mask_shape, normalize', [(None, True), ((5, 40), True), ((5, 3, 40), True),
                                                   ((5, 3, 40), False)])
def test_psd_forward_matches_numpy(mask_shape, normalize):
    rng = np.random.default_rng(1)
    y = rng.standard_normal((5, 4, 40)) + 1j * rng.standard_normal((5, 4, 40))
    m = None if mask_shape is None else rng.uniform(size=mask_shape)
    got = AO.power_spectral_density(torch.from_numpy(y), None if m is None else torch.from_numpy(m), normalize)
    _close(got.numpy(), O.power_spectral_density(y, m, normalize))


def test_souden_and_apply_forwards_match_numpy():
    t = synth.pos_def_hermitian(7, 4, 4, seed=2)
    nz = synth.pos_def_hermitian(7, 4, 4, seed=3)
    for ref in (None, 2):
        w, r = AO.mvdr_vector_souden(torch.from_numpy(t), torch.from_numpy(nz), ref)
        w_ref, r_ref = O.mvdr_vector_souden(t, nz, ref)
        assert r == r_ref
        _close(w.numpy(), w_ref)
    rng = np.random.default_rng(4)
    v = rng.standard_normal((3, 7, 4)) + 1j * rng.standard_normal((3, 7, 4))
    y = rng.standard_normal((7, 4, 50)) + 1j * rng.standard_normal((7, 4, 50))
    _close(AO.apply_beamforming_vector(torch.from_numpy(v), torch.from_numpy(y)).numpy(),
           O.apply_beamforming_vector(v, y))


def test_si_sdr_forward_matches_numpy():
    rng = np.random.default_rng(5)
    r = rng.standard_normal((1, 300))
    e = r + 0.3 * rng.standard_normal((4, 300))
    _close(AO.si_sdr(torch.from_numpy(r), torch.from_numpy(e)).numpy(), SO.si_sdr(r, e))


def test_si_sdr_closed_form_matches_autograd():
    rng = np.random.default_rng(6)
    r = torch.tensor(rng.standard_normal(200), requires_grad=True)
    e = torch.tensor(r.detach().numpy() + 0.5 * rng.standard_normal(200), requires_grad=True)
    AO.si_sdr(r, e).backward(torch.tensor(0.7, dtype=torch.float64))
    gr, ge = AO.si_sdr_grad(r.detach(), e.detach(), 0.7)
    _close(r.grad.numpy(), gr.numpy(), 1e-10)
    _close(e.grad.numpy(), ge.numpy(), 1e-10)


@pytest.mark.parametrize('normalize, zero_source', [(True, False), (False, False), (True, True)])
def test_psd_closed_form_matches_autograd(normalize, zero_source):
    rng = np.random.default_rng(7)
    F, K, D, T = 3, 2, 4, 30
    y = torch.tensor(rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T)), requires_grad=True)
    mn = rng.uniform(size=(F, K, T))
    if zero_source:
        mn[1, 0] = 1e-13  # the sum stays below 1e-10: the clamp is active
    m = torch.tensor(mn, requires_grad=True)
    G = torch.tensor(rng.standard_normal((F, K, D, D)) + 1j * rng.standard_normal((F, K, D, D)))
    phi = AO.power_spectral_density(y, m, normalize)
    (G.conj() * phi).sum().real.backward()
    gy, gm = AO.psd_grad(y.detach(), m.detach(), G, normalize)
    _close(y.grad.numpy(), gy.numpy(), 1e-10)
    _close(m.grad.numpy(), gm.numpy(), 1e-10)


def test_souden_closed_form_matches_autograd():
    rng = np.random.default_rng(8)
    t = torch.tensor(synth.pos_def_hermitian(5, 4, 4, seed=9), requires_grad=True)
    # a non-Hermitian noise matrix: the closed form must not assume symmetry
    nz0 = synth.pos_def_hermitian(5, 4, 4, seed=10) + 0.1 * rng.standard_normal((5, 4, 4))
    nz = torch.tensor(nz0 + 0j, requires_grad=True)
    g = torch.tensor(rng.standard_normal((5, 4)) + 1j * rng.standard_normal((5, 4)))
    w, _ = AO.mvdr_vector_souden(t, nz, 1)
    (g.conj() * w).sum().real.backward()
    gx, gn = AO.souden_grad(t.detach(), nz.detach(), 1, g)
    _close(t.grad.numpy(), gx.numpy(), 1e-10)
    _close(nz.grad.numpy(), gn.numpy(), 1e-10)


# ---- the long-double reference gradients against torch autograd, and the float64 models against the bounds ----------
SIZES = [64, 128, 256, 512, 1024, 2048, 4096]


def _autograd(fn, inputs, g):
    inputs = [torch.tensor(a, requires_grad=True) for a in inputs]
    out = fn(*inputs)
    return [a.resolve_conj() for a in torch.autograd.grad(out, inputs, torch.as_tensor(g))]


def _spectra(rng, rows, T, size):
    X = rng.standard_normal((rows, T, size // 2 + 1)) + 1j * rng.standard_normal((rows, T, size // 2 + 1))
    X *= 10.0 ** (-6 * rng.random((rows, T, 1)))
    X[:, 2::5] = 0
    return X


@pytest.mark.parametrize('n, size, shift, wl, fading, pad', [
    (1000, 128, 32, None, True, True), (1000, 128, 32, None, False, False), (997, 128, 48, 96, True, False),
    (700, 64, 16, 40, False, True), (30, 128, 32, None, True, True), (200, 64, 1, 63, True, True),
    (200, 64, 1, 1, False, True)])
def test_stft_istft_reference_gradients_match_autograd(n, size, shift, wl, fading, pad):
    rng = np.random.default_rng(n + size)
    x = rng.standard_normal((2, n))
    T = TO.num_frames(n, size, shift, wl, fading, pad)
    G = _spectra(rng, 2, T, size)
    (gx,) = _autograd(lambda x: AO.stft(x, size, shift, window_length=wl, fading=fading, pad=pad), [x], G)
    ref, _ = AO.stft_grad_parts(G, n, size, shift, wl, fading)
    _close(ref.astype(np.float64), gx.numpy())
    X = _spectra(rng, 2, T, size)
    out = AO.istft(torch.from_numpy(X), size, shift, window_length=wl, fading=fading)
    g = rng.standard_normal(out.shape)
    (gX,) = _autograd(lambda X: AO.istft(X, size, shift, window_length=wl, fading=fading), [X], g)
    _close(AO.istft_grad(g, T, size, shift, wl, fading).astype(np.complex128), gX.numpy())


@pytest.mark.parametrize('size', SIZES)
def test_model_stft_backward_within_half_the_bound(size):
    """The float64 model of stft_backward_kernel + overlap_add_kernel (the inverse body on G^) against the long-double
    transpose under the inverse bound, per sample; samples under all-zero G frames exactly zero."""
    rng = np.random.default_rng(size)
    worst = 0.0
    for shift, wl in ((size // 4, size), (1, 63), (3, size - 1), (size - 1, size - 1), (1, 1)):
        T = 12 if shift > 3 else 64
        n = (T - 1) * shift + wl
        G = _spectra(rng, 2, T, size)
        for fading in (True, False):
            ref, scale = AO.stft_grad_parts(G, n, size, shift, wl, fading)
            got = AO.model_stft_grad(G, n, size, shift, wl, fading)
            worst = max(worst, FO.inverse_ratio(got, ref, scale, size).max())
    print(f'size {size}: model stft backward ratio {worst:.3f} (bound C_I = {FO.C_I})')
    assert worst <= 0.5


@pytest.mark.parametrize('size', SIZES)
def test_model_istft_backward_within_half_the_bound(size):
    """The float64 model of istft_backward_kernel (the forward body on the windowed gradient, scaled) against the
    long-double rfft under the forward bound, per frame."""
    worst = 0.0
    for shift, wl in ((size // 4, size), (1, 63), (3, size - 1), (size - 1, size - 1), (1, 1)):
        T = 12 if shift > 3 else 64
        for fading in (True, False):
            crop = wl - shift if fading else 0
            g = FO.spread_signal((2, max(T * shift + wl - shift - 2 * crop, 0)), wl, size + shift)
            ratio, _ = FO.forward_ratio(AO.model_istft_grad(g, T, size, shift, wl, fading),
                                        AO.istft_grad(g, T, size, shift, wl, fading), size)
            worst = max(worst, ratio.max())
    print(f'size {size}: model istft backward ratio {worst:.3f} (bound C_F = {FO.C_F})')
    assert worst <= 0.5


@pytest.mark.parametrize('masked, normalize, clamp', [(True, True, False), (True, False, False), (False, True, False),
                                                      (True, True, True)])
def test_psd_reference_gradient_matches_autograd_and_bounds_float64(masked, normalize, clamp):
    rng = np.random.default_rng(40)
    F, K, D, T = 3, 2, 4, 70
    y = rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T))
    m = rng.uniform(size=(F, K, T)) if masked else None
    if clamp:
        m[1, 0] = 1e-13
        m[2, 1] = 0.0
    G = rng.standard_normal((F, K if masked else 1, D, D)) + 1j * rng.standard_normal((F, K if masked else 1, D, D))
    gy, gm, by, bm = AO.psd_grad_ld(y, m, G, normalize)
    if masked:
        ry, rm = _autograd(lambda y, m: AO.power_spectral_density(y, m, normalize), [y, m], G)
        _close(gm.astype(np.float64), rm.numpy())
        # float64 closed form (another summation order) inside half the bound
        _, gm64 = AO.psd_grad(torch.from_numpy(y), torch.from_numpy(m), torch.from_numpy(G), normalize)
        r = AO._ratio(AO._err(gm64.numpy(), gm), bm)
        print(f'psd grad mask, float64 closed form: worst ratio {r.max():.3f}')
        assert r.max() <= 0.5
    else:
        (ry,) = _autograd(lambda y: AO.power_spectral_density(y), [y], G[:, 0])
    _close(gy.astype(np.complex128), ry.numpy())
    r = AO._ratio(AO._err(ry.numpy(), gy), by)
    print(f'psd grad y, float64 autograd: worst ratio {r.max():.3f}')
    assert r.max() <= 0.5


@pytest.mark.parametrize('high_precision', [False, True])
def test_souden_reference_gradient_matches_autograd(high_precision):
    pytest.importorskip('mpmath')
    rng = np.random.default_rng(41)
    n, D, ref = 4, 5, 2
    t = synth.pos_def_hermitian(n, D, D, seed=42)
    nz = synth.pos_def_hermitian(n, D, D, seed=43) + 0.1 * rng.standard_normal((n, D, D))
    g = rng.standard_normal((n, D)) + 1j * rng.standard_normal((n, D))
    rt, rn = _autograd(lambda t, nz: AO.mvdr_vector_souden(t, nz, ref)[0], [t, nz + 0j], g)
    out = AO.souden_grad_ref(t, nz, ref, g, high_precision=high_precision)
    _close(out[0], rt.numpy())
    _close(out[1], rn.numpy())
    # float64 autograd (LAPACK solves) within half the normwise bound
    r = AO.souden_ratio(rt.numpy(), rn.numpy(), out)
    print(f'souden, float64 autograd: worst ratio {r.max():.3f}')
    assert r.max() <= 0.5


def test_souden_reference_of_an_ill_conditioned_bin_bounds_float64():
    """kappa(N) = 1e12: float64 LAPACK solves stay inside half the normwise bound of the mpmath reference."""
    pytest.importorskip('mpmath')
    from oracle import linalg_oracle as LO
    rng = np.random.default_rng(44)
    D = 6
    N = np.stack([LO.conditioned(D, 1e12, rng, hermitian=True), LO.graded(D, rng, decades=5.0)])
    X = np.stack([LO.from_spectrum(rng.uniform(0.5, 1.0, D), rng) for _ in range(2)])
    g = rng.standard_normal((2, D)) + 1j * rng.standard_normal((2, D))
    ref = AO.souden_grad_ref(X, N, 1, g, high_precision=True)
    f64 = AO.souden_grad_ref(X, N, 1, g)
    r = AO.souden_ratio(f64[0], f64[1], ref)
    print(f'souden kappa 1e12, float64: worst ratio {r.max():.3f}')
    assert r.max() <= 0.5


@pytest.mark.parametrize('B', [1, 3])
def test_apply_reference_gradient_matches_autograd(B):
    rng = np.random.default_rng(45 + B)
    F, D, T = 5, 4, 70
    v = rng.standard_normal((B, F, D)) + 1j * rng.standard_normal((B, F, D))
    y = rng.standard_normal((F, D, T)) + 1j * rng.standard_normal((F, D, T))
    g = rng.standard_normal((B, F, T)) + 1j * rng.standard_normal((B, F, T))
    rv, ry = _autograd(AO.apply_beamforming_vector, [v, y], g)
    gv, gy, bv, by = AO.apply_grad_ld(v, y, g)
    _close(gv.astype(np.complex128), rv.numpy())
    _close(gy.astype(np.complex128), ry.numpy())
    r = max(AO._ratio(AO._err(rv.numpy(), gv), bv).max(), AO._ratio(AO._err(ry.numpy(), gy), by).max())
    print(f'apply B = {B}, float64 autograd: worst ratio {r:.3f}')
    assert r <= 0.5


@pytest.mark.parametrize('n', [1, 2, 300, 8193])
def test_si_sdr_reference_gradient_matches_autograd(n):
    rng = np.random.default_rng(46 + n)
    r = rng.standard_normal((3, n))
    e = r + rng.uniform(0.01, 1.0, (3, 1)) * rng.standard_normal((3, n))
    g = rng.standard_normal(3)
    if n == 1:
        e = 3 * r + 1.0  # one sample: q = 0 would be inf; keep it finite
    rr, re = _autograd(AO.si_sdr, [r, e], g)
    gr, ge, br, be = AO.si_sdr_grad_ld(r, e, g)
    if n > 1:
        _close(gr.astype(np.float64), rr.numpy(), 1e-11)
        _close(ge.astype(np.float64), re.numpy(), 1e-11)
        ratio = max(AO._ratio(AO._err(rr.numpy(), gr), br).max(), AO._ratio(AO._err(re.numpy(), ge), be).max())
        print(f'si_sdr n = {n}, float64 autograd: worst ratio {ratio:.3f}')
        assert ratio <= 0.5
    # broadcast reference: its gradient sums the rows
    gsum, bsum = AO.reduce_rows(gr, br, [0, 0, 0], 1)
    assert gsum.shape == (1, n) and np.isfinite(bsum).all() == np.isfinite(br).all()
