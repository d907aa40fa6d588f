"""The closed-form WPE gradients of oracle/wpe_autograd_oracle.py (those of include/pbb.h) against torch autograd of
its restatement and against mpmath central differences; CPU only."""
import mpmath
import numpy as np
import pytest
import torch

from oracle import wpe_autograd_oracle as WA
from oracle import wpe_oracle as WO


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _close(got, ref, rel=1e-9):
    err = np.max(np.abs(got - ref)) if np.size(ref) else 0.0
    assert err <= rel * max(1.0, np.max(np.abs(ref))), (err, np.max(np.abs(ref)))


def _autograd(fn, Y, w, xbar):
    Yt = torch.tensor(Y, requires_grad=True)
    wt = None if w is None else torch.tensor(w, requires_grad=True)
    out = fn(Yt, wt)
    (out.conj() * torch.tensor(xbar)).real.sum().backward()
    gy = Yt.grad.resolve_conj().numpy()
    gw = None if wt is None else (np.zeros_like(w) if wt.grad is None else wt.grad.numpy())
    return out.detach().numpy(), gy, gw


@pytest.mark.parametrize('D', range(1, 9))
@pytest.mark.parametrize('taps', range(1, 5))
def test_step_closed_form_matches_autograd(D, taps):
    rng = np.random.default_rng(D * 10 + taps)
    n = D * taps
    for delay in range(4):
        for mode, T in (('full', 3 * n + 7), ('valid', 3 * n + delay + taps + 5), ('valid', delay + taps - 1)):
            if T == 0:
                continue
            Y, xbar = _cplx(rng, D, T), _cplx(rng, D, T)
            w = rng.uniform(0.5, 2.0, T)
            X, gy, gw = _autograd(lambda y, w: WA.wpe_step(y, w, taps, delay, mode)[0], Y, w, xbar)
            Xc, G, R = WA.step_forward(Y, w, taps, delay, mode)
            cy, cw = WA.step_backward(Y, w, G, R, xbar, taps, delay, mode)
            _close(Xc, X)
            _close(cy, gy)
            _close(cw, gw)
            if T <= delay + taps - 1 and mode == 'valid':    # an empty S: X = Y, the identity
                np.testing.assert_array_equal(cy, xbar)
                assert not cw.any()


@pytest.mark.parametrize('D', [1, 2, 3, 5, 8])
@pytest.mark.parametrize('psd_context', [0, 2, np.inf])
@pytest.mark.parametrize('iterations', [1, 2, 3])
@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_wpe_closed_form_matches_autograd(D, psd_context, iterations, mode):
    rng = np.random.default_rng(D + iterations)
    for taps, delay in ((1, 2), (2, 1), (4, 3)):
        T = 3 * D * taps + delay + taps + 6
        Y, xbar = _cplx(rng, D, T), _cplx(rng, D, T)
        X, gy, _ = _autograd(lambda y, _: WA.wpe(y, taps, delay, iterations, psd_context, mode), Y, None, xbar)
        np.testing.assert_allclose(X, WO.wpe_bin(Y, taps, delay, iterations, psd_context, mode), rtol=0,
                                   atol=1e-10 * np.abs(Y).max())
        Xc, stages = WA.wpe_forward(Y, taps, delay, iterations, psd_context, mode)
        _close(Xc, X)
        _close(WA.wpe_backward(Y, stages, xbar, taps, delay, psd_context, mode), gy)


@pytest.mark.parametrize('psd_context', [0, 1, 2, 7, np.inf])
def test_power_closed_forms_match_autograd(psd_context):
    rng = np.random.default_rng(5)
    Y, g = _cplx(rng, 4, 3, 20), rng.standard_normal((4, 20))
    Yt = torch.tensor(Y, requires_grad=True)
    (WA.get_power(Yt, psd_context) * torch.tensor(g)).sum().backward()
    ref = Yt.grad.resolve_conj().numpy()
    _close(np.stack([WA.power_backward(Y[b], g[b], psd_context, 'plain') for b in range(4)]), ref)
    np.testing.assert_allclose(WA.get_power(torch.tensor(Y), psd_context).numpy(), WO.get_power(Y, psd_context),
                               rtol=1e-14)
    # the per-bin inverse, and one bin forced onto the eps branch of the max (lambda_c below 1e-10 max)
    Y[1, :, 3:] *= 1e-7
    Yt = torch.tensor(Y, requires_grad=True)
    (WA.power_inverse_per_bin(Yt, psd_context) * torch.tensor(g)).sum().backward()
    ref = Yt.grad.resolve_conj().numpy()
    got = np.stack([WA.power_backward(Y[b], g[b], psd_context, 'inverse') for b in range(4)])
    _close(got, ref)


def test_power_max_ties_split_evenly():
    """two frames at the max share M's gradient, as torch's amax backward does"""
    Y = np.ones((1, 2, 6), dtype=np.complex128)
    Y[0, :, 2] = 0.5
    Y[0, :, 4] = 1e-6
    g = np.arange(1.0, 7.0)[None]
    Yt = torch.tensor(Y, requires_grad=True)
    (WA.power_inverse_per_bin(Yt) * torch.tensor(g)).sum().backward()
    _close(WA.power_backward(Y[0], g[0], 0, 'inverse')[None], Yt.grad.resolve_conj().numpy())


# ---- mpmath central differences ------------------------------------------------------------------------------------

def _mp_loss(Y, w, xbar, taps, delay):
    """Re sum conj(xbar) X of one step, in mpmath"""
    D, T = len(Y), len(Y[0])
    n = taps * D
    yt = [[(Y[r % D][t - delay - r // D] if t - delay - r // D >= 0 else mpmath.mpc(0)) for t in range(T)]
          for r in range(n)]
    R = mpmath.matrix(n, n)
    P = mpmath.matrix(n, D)
    for i in range(n):
        for j in range(n):
            R[i, j] = mpmath.fsum(w[t] * yt[i][t] * mpmath.conj(yt[j][t]) for t in range(T))
        for d in range(D):
            P[i, d] = mpmath.fsum(w[t] * yt[i][t] * mpmath.conj(Y[d][t]) for t in range(T))
    G = mpmath.matrix(n, D)
    for d in range(D):
        g = mpmath.lu_solve(R, P.column(d))
        for i in range(n):
            G[i, d] = g[i]
    total = mpmath.mpf(0)
    for d in range(D):
        for t in range(T):
            x = Y[d][t] - mpmath.fsum(mpmath.conj(G[r, d]) * yt[r][t] for r in range(n))
            total += mpmath.re(mpmath.conj(xbar[d][t]) * x)
    return total


def test_step_gradient_matches_mpmath_central_differences():
    with mpmath.workdps(40):
        _check_central_differences()


def _check_central_differences():
    rng = np.random.default_rng(7)
    D, taps, delay, T = 2, 2, 1, 12
    Y, xbar = _cplx(rng, D, T), _cplx(rng, D, T)
    w = rng.uniform(0.5, 2.0, T)
    _, G, R = WA.step_forward(Y, w, taps, delay)
    gy, gw = WA.step_backward(Y, w, G, R, xbar, taps, delay)
    Ym = [[mpmath.mpc(complex(v)) for v in row] for row in Y]
    wm = [mpmath.mpf(float(v)) for v in w]
    xm = [[mpmath.mpc(complex(v)) for v in row] for row in xbar]
    h = mpmath.mpf(10) ** -15

    def diff(set_, get):
        old = get()
        set_(old + h)
        hi = _mp_loss(Ym, wm, xm, taps, delay)
        set_(old - h)
        lo = _mp_loss(Ym, wm, xm, taps, delay)
        set_(old)
        return float((hi - lo) / (2 * h))

    for d in range(D):
        for t in range(T):
            def setter(v, d=d, t=t):
                Ym[d][t] = v
            re = diff(lambda v: setter(mpmath.mpc(v, Ym[d][t].imag)), lambda: Ym[d][t].real)
            im = diff(lambda v: setter(mpmath.mpc(Ym[d][t].real, v)), lambda: Ym[d][t].imag)
            assert abs(complex(re, im) - gy[d, t]) <= 1e-10 * np.abs(gy).max(), (d, t)
    for t in range(T):
        def wset(v, t=t):
            wm[t] = v
        assert abs(diff(wset, lambda: wm[t]) - gw[t]) <= 1e-10 * np.abs(gw).max(), t
