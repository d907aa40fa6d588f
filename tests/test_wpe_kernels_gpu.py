"""The offline and online WPE kernels over their whole shape domain, per bin against long-double references
(oracle/wpe_autograd_oracle.py, oracle/wpe_online_oracle.py in np.clongdouble; tests/test_wpe_kernels_oracle.py checks
them against mpmath and checks that the parameter lists below reach every tiling class at its edges).

Bounds (u = 2^-53, kappa_i the 1-norm condition number of iteration i's R, of its live block for a dead channel):

- offline forward, per bin:
      |X_dev - X_ref| <= u (sum_i kappa_i (ceil(span / 4) + parts + n) + n) S + r sqrt(2) 2^-24 max|X_ref|,
  S = max_{d,t} (|Y_dt| + sum_j |G_jd| |Yt_jt|), the magnitude of the terms of an output of the filter.  The
  correlations are sequential m8n8k4 DMMA steps of four frames over a part's span, then the parts summed in order:
  an entry of R or P errs by about (span / 4 + parts) u of the terms it sums, and the solve (LU, or the Jacobi
  eigendecomposition of the minimum-norm fallback) adds n u; both reach G through kappa(R).  The filter sums the
  taps D = n terms of each output.  An iteration's weights come from the previous X, so the iterations' terms add.
  r = 1 for complex64 (the one rounding of the stored output; the input widens exactly), else 0.
- a step's gradients (wpe_step's backward): oracle/wpe_autograd_oracle.grad_bound, as in test_wpe_autograd_gpu.py.
- online, per bin and frame: |Z_dev,t - Z_ref,t| <= 16 n u kappa(R_t) g max|Y_f| (+ one complex64 rounding of Z),
  the per-frame term of test_online_wpe_gpu.py taken at frame t rather than its maximum over the stream (the first
  frames, where R_t is the decayed identity plus a few rank-one terms, have a kappa far above that of the settled
  recursion but errors of the size of their data), and g = 1 + log2(M) with M = min(T, 1 / (1 - alpha)) the frames the
  recursion remembers: a rounding made at frame s stays in Q and G for about M frames; the recursion contracts it
  there (the update of Q is a projection followed by 1 / alpha), so it is not carried at full size, but the errors of
  the remembered frames combine, and a sum over M frames whose weights halve every doubling of age grows with
  log2 M.  At alpha = 1 nothing is forgotten, M = T.
- the online step against the long-double step: 16 n u of the magnitude of the terms behind each output, as in
  test_online_wpe_gpu.py.

With delay = 0 the current frame is among the regressors and X is rounding residue: one iteration only.  The largest
error-to-bound ratio of each group is printed at the end of the module (pytest -s) and recorded in DESIGN.md."""
import collections
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_em_kernels_gpu import Launches  # noqa: E402
from test_online_wpe_gpu import _step_case, _terms  # noqa: E402
from test_wpe_gpu import _reverberant  # noqa: E402
from test_wpe_kernels_oracle import corr_parts, require_extended_precision  # noqa: E402

from oracle import wpe_autograd_oracle as WA  # noqa: E402
from oracle import wpe_online_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
require_extended_precision()

LD = np.clongdouble
U = 2.0 ** -53
U32 = 2.0 ** -24

# ---- the parameter lists (their coverage is checked on the CPU) -----------------------------------------------------
# (D, taps): every (slots, passes) class of wpe_corr at its lowest and highest n + D (2/28, 29/52, 53/76, 77/88,
# 89/104, 105/120); odd n + D gives a padded last 8-row block
CORR_SHAPES = [(1, 1), (4, 6), (7, 3), (1, 28), (4, 12), (1, 52), (4, 18), (7, 10), (8, 10), (1, 88), (8, 12),
               (15, 6), (24, 4), (30, 3)]
# (dtype, statistics_mode, iterations, delay)
CORR_VARIANTS = [('complex128', 'full', 3, 2), ('complex64', 'valid', 2, 1), ('complex128', 'valid', 1, 0)]
# T - tb: the part edges (64-frame chunks, 1024-frame parts), the filter's 128-frame chunk and the 64-part cap
FRAME_COUNTS = [63, 64, 65, 127, 128, 129, 1024, 1025, 65536, 65537, 100000, 131073]
FRAME_SHAPE = (2, 3, 1)              # D, taps, delay
FRAME_BIG_SHAPE = (8, 10, 3)         # n = 80
FRAME_BIG_T = 65537
LSTSQ_SHAPES = [(3, 5), (7, 9), (8, 8), (5, 13), (5, 19)]       # n = 15, 63, 64, 65, 95
PSD_T = 300
MANY_BINS = 65537
# online: R = ceil(n / 16) = 1..6, a full and a partial tile each
ONLINE_SHAPES = [(2, 8), (2, 5), (4, 8), (4, 6), (8, 6), (4, 10), (8, 8), (6, 10), (8, 10), (7, 10), (8, 12),
                 (30, 3)]
STREAM_SHAPES = [(6, 10), (8, 10)]
STREAM_T = 4000
# (D, taps, the largest delay whose ring fits the shared memory of a CTA)
ONLINE_DELAY_EDGES = [(30, 3, 349), (8, 10, 1498)]


def psd_contexts():
    return [129, PSD_T - 1, PSD_T, 10 * PSD_T]


# ---- helpers ----------------------------------------------------------------------------------------------------------
RATIOS = collections.defaultdict(float)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for group, r in sorted(RATIOS.items()):
        print(f'\nwpe kernels: largest error / bound of {group}: {r:.3g}')


def _wpe():
    from pb_bss_b200 import wpe
    return wpe


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def reverberant(F, D, T, delay, seed):
    """(Y (F, D, T), direct path): test_wpe_gpu's STFT-domain reverberation"""
    return _reverberant(F, D, T, max(delay, 1), 12, seed)


def _bins(D, T, delay, seed):
    """two bins: white, and reverberant (where the filter does real work)"""
    rng = np.random.default_rng(seed)
    return np.stack([_cplx(rng, D, T), reverberant(1, D, T, delay, seed)[0][0]])


def forward_bound(Y, G, kappas, span, parts, taps, delay, roundings=0, X=None):
    """the offline forward bound of the module docstring for one bin"""
    D = Y.shape[0]
    n = taps * D
    Yt = np.abs(WA.y_tilde(np.asarray(Y, complex), taps, delay))
    S = float((np.abs(Y) + np.abs(np.asarray(G, complex)).T @ Yt).max())
    top = 0.0 if X is None else float(np.abs(X).max())
    return (U * (sum(kappas) * (math.ceil(span / 4) + parts + n) + n) * S
            + roundings * math.sqrt(2) * U32 * top)


def _check_forward(group, got, Y, taps, delay, iterations, psd_context, mode, single, live=False):
    """per bin, the device X against wpe_forward in long double"""
    D, T = Y.shape[-2:]
    parts, span = corr_parts(T, D, taps, delay, mode == 'valid')
    for b in range(Y.shape[0]):
        X, stages = WA.wpe_forward(Y[b].astype(LD), taps, delay, iterations, psd_context, mode)
        if not stages:
            assert np.array_equal(got[b], Y[b])
            continue
        kap = [(WA.live_kappa if live else WA.kappa)(st[2]) for st in stages]
        bound = forward_bound(Y[b], stages[-1][1], kap, span, parts, taps, delay, int(single), X)
        err = float(np.abs(got[b].astype(LD) - X).max())
        RATIOS[group] = max(RATIOS[group], err / bound)
        assert err <= bound, (group, b, err, bound)


def _device_wpe(Y, taps, delay, iterations, psd_context=0, mode='full'):
    X, status = _wpe()._run(torch.from_numpy(Y).cuda(), taps, delay, iterations, psd_context, mode, False)
    return X.cpu().numpy(), status


# ---- 1. correlation tiling --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D,taps', CORR_SHAPES)
@pytest.mark.parametrize('variant', CORR_VARIANTS)
def test_correlation_tiling_against_long_double(D, taps, variant):
    dtype, mode, iterations, delay = variant
    n = taps * D
    Y = _bins(D, max(200, 4 * n), delay, seed=D * 100 + taps).astype(dtype)
    X, status = _device_wpe(Y, taps, delay, iterations, 0, mode)
    assert status == 0 and X.dtype == Y.dtype
    _check_forward('correlation tiling', X, Y, taps, delay, iterations, 0, mode, dtype == 'complex64')


# ---- 2. frame counts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tv', FRAME_COUNTS)
@pytest.mark.parametrize('mode', ['full', 'valid'])
def test_frame_counts_against_long_double(tv, mode):
    D, taps, delay = FRAME_SHAPE
    T = tv + (delay + taps - 1 if mode == 'valid' else 0)
    Y = _bins(D, T, delay, seed=tv)
    X, status = _device_wpe(Y, taps, delay, 2, 0, mode)
    assert status == 0
    _check_forward('frame counts', X, Y, taps, delay, 2, 0, mode, False)


def test_n80_past_the_part_cap_against_long_double():
    D, taps, delay = FRAME_BIG_SHAPE
    Y = reverberant(1, D, FRAME_BIG_T, delay, seed=80)[0]
    assert corr_parts(FRAME_BIG_T, D, taps, delay, False) == (61, 1088)
    X, status = _device_wpe(Y, taps, delay, 1)
    assert status == 0
    _check_forward('frame counts', X, Y, taps, delay, 1, 0, 'full', False)


def test_step_backward_past_the_part_cap_against_long_double():
    D, taps, delay = FRAME_SHAPE
    T = 65537
    rng = np.random.default_rng(7)
    Y = _bins(D, T, delay, seed=7)
    xbar = _cplx(rng, 2, D, T)
    w = rng.uniform(0.5, 2.0, (2, T))
    Yt, wt = (torch.from_numpy(a).cuda().requires_grad_() for a in (Y, w))
    X = _wpe().wpe_step(Yt, wt, taps, delay)
    gy, gw = (g.cpu().numpy() for g in torch.autograd.grad(X, (Yt, wt), torch.from_numpy(xbar).cuda()))
    n = taps * D
    for b in range(2):
        yl, wl = Y[b].astype(LD), w[b].astype(np.longdouble)
        Xr, G, R = WA.step_forward(yl, wl, taps, delay)
        ry, rw = WA.step_backward(yl, wl, G, R, xbar[b].astype(LD), taps, delay)
        t = float(np.abs(xbar[b]).max())
        for what, got, ref, terms in (('Y', gy[b], ry, t), ('w', gw[b], rw, t / w[b].min())):
            bound = WA.grad_bound(ref, [WA.kappa(R)], n, T, 0, terms)
            err = float(np.abs(got - ref).max())
            RATIOS['step backward'] = max(RATIOS['step backward'], err / bound)
            assert err <= bound, (what, b, err, bound)
        parts, span = corr_parts(T, D, taps, delay, False)
        bound = forward_bound(Y[b], G, [WA.kappa(R)], span, parts, taps, delay)
        err = float(np.abs(X[b].detach().cpu().numpy() - Xr).max())
        RATIOS['frame counts'] = max(RATIOS['frame counts'], err / bound)
        assert err <= bound


# ---- 3. the minimum-norm fallback -----------------------------------------------------------------------------------
@pytest.mark.parametrize('D,taps', LSTSQ_SHAPES)
def test_lstsq_at_odd_n_against_long_double(D, taps):
    """a dead channel makes R exactly singular: wpe_lstsq_kernel's Jacobi eigensolver, with a dummy player for odd n
    and more than 32 pairs per round above n = 64"""
    n, delay = taps * D, 3
    Y = _bins(D, 5 * n, delay, seed=n)
    Y[:, 1] = 0
    X, status = _device_wpe(Y, taps, delay, 3)
    assert status == _wpe().LSTSQ
    assert np.all(X[:, 1] == 0)
    _check_forward('lstsq', X, Y, taps, delay, 3, 0, 'full', False, live=True)


# ---- 4. psd_context -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('c', psd_contexts())
def test_psd_context_against_inf_and_long_double(c):
    D, taps, delay = 4, 5, 2
    Y = _bins(D, PSD_T, delay, seed=c)
    X, status = _device_wpe(Y, taps, delay, 3, c)
    assert status == 0
    _check_forward('psd_context', X, Y, taps, delay, 3, c, 'full', False)
    if c >= PSD_T - 1:   # every window holds every frame: the mean over all frames, up to the order of the sums
        _check_forward('psd_context', X, Y, taps, delay, 3, math.inf, 'full', False)
        Xinf, _ = _device_wpe(Y, taps, delay, 3, math.inf)
        _check_forward('psd_context', Xinf, Y, taps, delay, 3, c, 'full', False)


# ---- 5. more bins than one group ------------------------------------------------------------------------------------
def test_more_than_65535_bins_run_a_tail_group_and_are_bitwise_per_bin():
    wpe = _wpe()
    D, taps, delay, T, iterations = 2, 3, 1, 64, 2
    rng = np.random.default_rng(65537)
    Y = torch.from_numpy(_cplx(rng, MANY_BINS, D, T)).cuda()
    w = torch.from_numpy(rng.uniform(0.5, 2.0, (MANY_BINS, T))).cuda()
    xbar = torch.from_numpy(_cplx(rng, MANY_BINS, D, T)).cuda()

    def grads(Ys, ws, xb):
        Yg, wg = Ys.clone().requires_grad_(), ws.clone().requires_grad_()
        X = wpe.wpe_step(Yg, wg, taps, delay)
        return [X.detach()] + list(torch.autograd.grad(X, (Yg, wg), xb))

    with Launches() as rec:
        X = wpe.wpe(Y, taps=taps, delay=delay, iterations=iterations)
    assert rec.names.count('wpe_corr_kernel') == 2 * iterations          # a full group and the tail group
    assert rec.names.count('wpe_solve_kernel') == 2 * iterations
    with Launches() as rec:
        step = grads(Y, w, xbar)
    assert rec.names.count('wpe_corr_kernel') == 4                       # forward and backward, two groups each
    assert rec.names.count('wpe_gbar_kernel') == 2
    assert rec.names.count('wpe_step_backward_kernel') == 2
    for b0 in range(0, MANY_BINS, 8192):
        sl = slice(b0, b0 + 8192)
        assert torch.equal(wpe.wpe(Y[sl], taps=taps, delay=delay, iterations=iterations).view(torch.float64),
                           X[sl].view(torch.float64))
        for a, b in zip(grads(Y[sl], w[sl], xbar[sl]), step):
            assert torch.equal(a, b[sl])
    keep = [0, 65534, 65535, MANY_BINS - 1]
    Yk = Y[keep].cpu().numpy()
    _check_forward('many bins', X[keep].cpu().numpy(), Yk, taps, delay, iterations, 0, 'full', False)


# ---- 6. online ------------------------------------------------------------------------------------------------------
def _online_bound(Y, kappa, taps, alpha, single=False, Z=None):
    """(T, F): the online bound of the module docstring, per frame and bin"""
    T, _, D = Y.shape
    M = T if alpha == 1 else min(T, 1 / (1 - alpha))
    g = 1 + math.log2(max(M, 1))
    b = 16 * taps * D * U * kappa * g * np.abs(Y).max(axis=(0, 2))
    if single:
        b = b + math.sqrt(2) * U32 * np.abs(Z).max(axis=(0, 2)).astype(float)
    return b


def _check_stream(group, Y, taps, delay, alpha, single=False):
    wpe = _wpe()
    Z, _ = wpe.online_wpe(Y, taps, delay, alpha)
    assert Z.dtype == Y.dtype
    Zr, _, kappa = O.online_wpe(Y.astype(LD), taps, delay, alpha, details=True)
    bound = _online_bound(Y, kappa, taps, alpha, single, Zr)
    err = np.abs(Z.astype(LD) - Zr).max(axis=2).astype(float)
    RATIOS[group] = max(RATIOS[group], float((err / bound).max()))
    assert (err <= bound).all(), (group, (err / bound).max())


@pytest.mark.parametrize('D,taps', ONLINE_SHAPES)
def test_online_step_every_tile_against_long_double(D, taps):
    delay = 2
    buf, power, Q, G, alpha = _step_case(3, D, taps, delay, seed=D * taps)
    got = _wpe().online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    want = O.online_wpe_step(buf.astype(LD), power.astype(np.longdouble), Q.astype(LD), G.astype(LD), alpha, taps,
                             delay)
    for g, w, scale in zip(got, want, _terms(buf, power, Q, G, alpha, taps, delay)):
        err = np.abs(g.astype(LD) - w).reshape(w.shape[0], -1).max(axis=1).astype(float)
        bound = 16 * taps * D * U * scale
        RATIOS['online step'] = max(RATIOS['online step'], float((err / bound).max()))
        assert (err <= bound).all(), (err, bound)


@pytest.mark.parametrize('D,taps', ONLINE_SHAPES)
def test_online_stream_every_tile_against_long_double(D, taps):
    rng = np.random.default_rng(D * taps)
    _check_stream('online streams', _cplx(rng, 300, 2, D), taps, 2, 0.99)


@pytest.mark.parametrize('D,taps', STREAM_SHAPES)
@pytest.mark.parametrize('alpha', [0.99, 0.9999, 1.0])
@pytest.mark.parametrize('source', ['white', 'reverberant'])
def test_online_long_stream_against_long_double(D, taps, alpha, source):
    delay = 2
    if source == 'white':
        Y = _cplx(np.random.default_rng(D), STREAM_T, 1, D)
    else:
        Y = reverberant(1, D, STREAM_T, delay, seed=D)[0].transpose(2, 0, 1)
    _check_stream(f'online long streams (alpha {alpha})', np.ascontiguousarray(Y), taps, delay, alpha)


def test_online_complex64_against_long_double():
    D, taps = 6, 10
    Y = _cplx(np.random.default_rng(64), 1000, 2, D).astype(np.complex64)
    _check_stream('online complex64', Y, taps, 2, 0.9999, single=True)


@pytest.mark.parametrize('D,taps,delay', ONLINE_DELAY_EDGES)
def test_online_largest_delay_runs_and_the_next_raises(D, taps, delay):
    # alpha = 1 keeps Q = I over the frames before the delayed window reaches the data; with alpha < 1 the state would
    # be alpha^-delay I there, a start no per-frame kappa describes (measured: 1e3 times the per-frame bound at
    # alpha = 0.99, against 4e-8 times the bound with the stream's largest kappa)
    rng = np.random.default_rng(delay)
    Y = _cplx(rng, delay + 4 * taps * D, 1, D)      # past the delay, enough frames for R_t to settle
    _check_stream('online delay edge', Y, taps, delay, 1.0)
    with pytest.raises(NotImplementedError):
        _wpe().online_wpe(Y, taps, delay + 1, 0.99)
