"""oracle/autograd_oracle.py on the CPU: its torch forwards equal the NumPy oracles, and the closed-form gradients that
the device backward passes implement (include/pbb.h) equal torch autograd of the restatement in float64."""
import numpy as np
import pytest
import torch

from oracle import autograd_oracle as AO
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
