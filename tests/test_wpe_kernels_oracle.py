"""The long-double WPE references of tests/test_wpe_kernels_gpu.py, checked on the CPU.

- The references (oracle/wpe_autograd_oracle.py: step_forward, wpe_forward, lstsq_solve; oracle/wpe_online_oracle.py:
  online_wpe in np.clongdouble) against mpmath at 40 digits at tiny shapes, and lstsq_solve against np.linalg.lstsq.
- A restatement of the device's shape choices (pbb's wpe_shape, wpe_corr's slot count, wpe_online_run's tile count
  R and the online kernel's shared memory), and the claim that the GPU file's parameter lists reach every class at
  its edges.
- That the forward bound of the GPU file rejects real defects at its longest T: an R that leaves out one frame and an
  R rounded to complex64."""
import importlib
import math
import os
import sys

import numpy as np
import pytest

from oracle import wpe_autograd_oracle as WA
from oracle import wpe_online_oracle as O

LD = np.clongdouble


def require_extended_precision():
    """The references are only worth more than float64 where long double is wider than double."""
    assert np.finfo(np.longdouble).eps <= 2.0 ** -60, 'np.longdouble is not an extended type on this platform'


require_extended_precision()

# ---- the device's shape choices (csrc/wpe.cuh, csrc/wpe_online.cuh, csrc/api_wpe.cu) -------------------------------
CHUNK = 64               # kWpeChunk: frames per staged chunk of wpe_corr_kernel, and the span's granule
PART_FRAMES = 1024       # kWpePartFrames
MAX_PARTS = 64           # kWpeMaxParts
CORR_WARPS = 16          # kWpeCorrWarps
SLOTS = (2, 6, 12, 16, 22)
FILTER_CHUNK = 128       # kWpeFilterChunk
ONLINE_MAX_SMEM = 232448
MAX_N = 96


def corr_parts(T, D, taps, delay, valid):
    """(parts, span) of wpe_shape: the frames T - tb of the statistics in parts of about 1024, at most 64, the span
    rounded up to whole 64-frame chunks (which can leave fewer than 64 parts)"""
    tb = delay + taps - 1 if valid else 0
    tv = T - tb
    if tv <= 0:
        return 1, CHUNK
    parts = min(-(-tv // PART_FRAMES), MAX_PARTS)
    span = -(-tv // parts)
    span = -(-span // CHUNK) * CHUNK
    return -(-tv // span), span


def corr_class(D, taps):
    """(slots per warp, passes) of wpe_corr: the lower-triangle 8 x 8 tiles of the 2 (n + D) real rows over 16 warps"""
    t8 = -(-2 * (taps * D + D) // 8)
    ntiles = t8 * (t8 + 1) // 2
    tpw = -(-ntiles // CORR_WARPS)
    slots = next((s for s in SLOTS if tpw <= s), SLOTS[-1])
    return slots, -(-ntiles // (CORR_WARPS * slots))


def online_tiles(n):
    """R of wpe_online_kernel<R>: each of the 16 x 16 threads holds R x R entries of Q"""
    return min(-(-n // 16), 6)


def online_smem_bytes(D, taps, delay):
    n, L = taps * D, taps + delay + 1
    return 16 * (11 * MAX_N + D * n + L * D) + 8 * (L + 1)


def max_online_delay(D, taps):
    """the largest delay whose ring of taps + delay + 1 frames fits a CTA's shared memory"""
    delay = 0
    while online_smem_bytes(D, taps, delay + 1) <= ONLINE_MAX_SMEM:
        delay += 1
    return delay


def test_shape_restatement_at_known_points():
    # the examples of the part cap: 65 537 frames give 61 parts of 1088, 100 000 give 63 of 1600, 131 073 63 of 2112
    assert corr_parts(65536, 2, 3, 1, False) == (64, 1024)
    assert corr_parts(65537, 2, 3, 1, False) == (61, 1088)
    assert corr_parts(100000, 2, 3, 1, False) == (63, 1600)
    assert corr_parts(131073, 2, 3, 1, False) == (63, 2112)
    assert corr_parts(1025, 2, 3, 1, False) == (2, 576)
    assert corr_parts(10, 2, 3, 1, True) == (1, 64) and corr_parts(3, 2, 3, 1, True) == (1, 64)
    # the slot classes split n + D at 28 / 52 / 76 / 88 / 104, and n + D = 120 takes two passes
    assert [corr_class(1, t - 1) for t in (2, 28)] == [(2, 1)] * 2
    assert corr_class(1, 28) == (6, 1) and corr_class(4, 12) == (6, 1)
    assert corr_class(1, 52) == (12, 1) and corr_class(4, 18) == (12, 1)
    assert corr_class(7, 10) == (16, 1) and corr_class(8, 10) == (16, 1)
    assert corr_class(1, 88) == (22, 1) and corr_class(8, 12) == (22, 1)
    assert corr_class(15, 6) == (22, 2) and corr_class(30, 3) == (22, 2)
    assert max_online_delay(30, 3) == 349 and max_online_delay(8, 10) == 1498
    assert [online_tiles(n) for n in (1, 16, 17, 49, 64, 65, 96)] == [1, 1, 2, 4, 4, 5, 6]


def _gpu_file():
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    return importlib.import_module('test_wpe_kernels_gpu')


def test_gpu_parameters_reach_every_class_at_its_edges():
    G = _gpu_file()
    # wpe_corr: every (slots, passes) class at the lowest and the highest n + D it takes, and padded 8-row blocks
    edges = {}
    for D in range(1, 31):
        for taps in range(1, MAX_N // D + 1):
            c, m = corr_class(D, taps), taps * D + D
            lo, hi = edges.get(c, (m, m))
            edges[c] = (min(lo, m), max(hi, m))
    assert len(edges) == 6
    reached = {}
    for D, taps in G.CORR_SHAPES:
        reached.setdefault(corr_class(D, taps), set()).add(taps * D + D)
    for c, (lo, hi) in edges.items():
        assert {lo, hi} <= reached.get(c, set()), (c, lo, hi, reached.get(c))
    assert any((taps * D + D) % 4 for D, taps in G.CORR_SHAPES)                 # a padded last 8-row block
    assert {v[0] for v in G.CORR_VARIANTS} == {'complex64', 'complex128'}
    assert {v[1] for v in G.CORR_VARIANTS} == {'full', 'valid'}
    assert {v[2] for v in G.CORR_VARIANTS} == {1, 2, 3}
    assert all(v[3] > 0 or v[2] == 1 for v in G.CORR_VARIANTS)                   # delay = 0: one iteration
    # frame counts: part and filter-chunk edges, and a part count below 64 after the cap
    tvs = set(G.FRAME_COUNTS)
    assert {63, 64, 65, 1024, 1025, 65536, 65537, 100000, 131073} <= tvs
    assert {FILTER_CHUNK - 1, FILTER_CHUNK, FILTER_CHUNK + 1} <= tvs
    D, taps, delay = G.FRAME_SHAPE
    parts = [corr_parts(tv, D, taps, delay, False)[0] for tv in tvs]
    assert 64 in parts and any(p < 64 and tv > 64 * PART_FRAMES for p, tv in zip(parts, tvs))
    assert corr_parts(G.FRAME_BIG_T, *G.FRAME_BIG_SHAPE[:2], G.FRAME_BIG_SHAPE[2], False)[0] < MAX_PARTS
    assert G.FRAME_BIG_SHAPE[0] * G.FRAME_BIG_SHAPE[1] == 80
    # lstsq: odd n, n = 64 and n above 64 (more than 32 rotation pairs)
    ns = {D * taps for D, taps in G.LSTSQ_SHAPES}
    assert {15, 63, 64, 65, 95} <= ns
    # psd_context beyond a filter chunk, at T - 1, T and 10 T
    assert G.PSD_T - 1 in G.psd_contexts() and G.PSD_T in G.psd_contexts() and 10 * G.PSD_T in G.psd_contexts()
    assert any(FILTER_CHUNK < c < G.PSD_T - 1 for c in G.psd_contexts())
    # the online kernel: every R with a full and a partial tile, n = 60 and 70 among them
    tiles = {}
    for D, taps in G.ONLINE_SHAPES:
        n = taps * D
        tiles.setdefault(online_tiles(n), set()).add(n % 16 == 0)
    assert tiles == {R: {True, False} for R in range(1, 7)}, tiles
    assert {(6, 10), (7, 10), (8, 10)} <= set(G.ONLINE_SHAPES)
    assert {D * taps for D, taps in G.STREAM_SHAPES} == {60, 80}
    assert online_tiles(60) == 4
    # the largest accepted delay of the ring, next to the first rejected one
    for D, taps, delay in G.ONLINE_DELAY_EDGES:
        assert delay == max_online_delay(D, taps)
        assert online_smem_bytes(D, taps, delay) <= ONLINE_MAX_SMEM < online_smem_bytes(D, taps, delay + 1)
    # more than 65 535 bins: a tail group
    assert G.MANY_BINS > 65535


# ---- the references against mpmath ----------------------------------------------------------------------------------
mp = pytest.importorskip('mpmath')
DPS = 40


def _mpc(z):
    """z (any complex dtype, long double included) exactly enough: the shortest repr that reads back to it"""
    def f(x):
        return mp.mpf(np.format_float_scientific(np.longdouble(x), unique=True))
    return mp.mpc(f(z.real), f(z.imag))


def _cplx(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _mp_step(Y, w, taps, delay):
    """one WPE step at 40 digits, w a list of mpf: R, P of the weighted statistics, G = R^-1 P, X = Y - G^H Yt"""
    Yt = WA.y_tilde(Y, taps, delay)
    n, D, T = Yt.shape[0], Y.shape[0], Y.shape[1]
    yt = [[_mpc(Yt[i, t]) for t in range(T)] for i in range(n)]
    y = [[_mpc(Y[d, t]) for t in range(T)] for d in range(D)]
    wm = list(w)
    R = mp.matrix(n, n)
    P = mp.matrix(n, D)
    for i in range(n):
        for j in range(n):
            R[i, j] = mp.fsum(wm[t] * yt[i][t] * mp.conj(yt[j][t]) for t in range(T))
        for d in range(D):
            P[i, d] = mp.fsum(wm[t] * yt[i][t] * mp.conj(y[d][t]) for t in range(T))
    G = mp.matrix(n, D)
    for d in range(D):
        g = mp.lu_solve(R, P.column(d))
        for i in range(n):
            G[i, d] = g[i]
    X = np.empty((D, T), complex)
    exact = []
    for d in range(D):
        for t in range(T):
            x = y[d][t] - mp.fsum(mp.conj(G[i, d]) * yt[i][t] for i in range(n))
            X[d, t] = complex(x)
            exact.append(x)
    return X, exact


def test_offline_iteration_against_mpmath():
    """one iteration of wpe (weights from Y's power) in long double against 40 digits"""
    with mp.workdps(DPS):
        rng = np.random.default_rng(1)
        D, taps, delay, T = 2, 3, 1, 24
        Y = _cplx(rng, D, T)
        X, stages = WA.wpe_forward(Y.astype(LD), taps, delay, 1, 0, 'full')
        w = stages[0][0]
        lam = [mp.fsum(abs(_mpc(Y[d, t])) ** 2 for d in range(D)) / D for t in range(T)]
        wmp = [1 / max(v, mp.mpf(WA.EPS_POWER) * max(lam)) for v in lam]
        assert max(abs(_mpc(a) - b) / b for a, b in zip(w, wmp)) < 1e-18
        _, exact = _mp_step(Y, wmp, taps, delay)
        err = max(float(abs(_mpc(X[d, t]) - exact[d * T + t]))
                  for d in range(D) for t in range(T))
        kap = WA.kappa(stages[0][2])
        # long double's unit (2^-64) times n kappa, far below what float64 could reach (2^-53)
        assert err <= 64 * taps * D * kap * 2.0 ** -64 * np.abs(Y).max(), err


def test_online_recursion_against_mpmath():
    with mp.workdps(DPS):
        rng = np.random.default_rng(2)
        T, D, taps, delay, alpha = 20, 2, 2, 1, 0.9
        Y = _cplx(rng, T, 1, D)
        Z, _ = O.online_wpe(Y.astype(LD), taps, delay, alpha)
        n, L = taps * D, taps + delay + 1
        stream = [[mp.mpc(0)] * D for _ in range(L - 1)] + [[_mpc(v) for v in Y[t, 0]] for t in range(T)]
        Q = mp.eye(n)
        G = mp.matrix(n, D)
        a = mp.mpf(alpha)
        err = 0.0
        for t in range(T):
            buf = stream[t:t + L]
            lam = mp.fsum(abs(v) ** 2 for f in buf for v in f) / (L * D)
            win = [buf[L - delay - 2 - k][d] for d in range(D) for k in range(taps)]   # index d taps + k
            pred = [buf[-1][d] - mp.fsum(mp.conj(G[i, d]) * win[i] for i in range(n)) for d in range(D)]
            u = [mp.fsum(Q[i, j] * win[j] for j in range(n)) for i in range(n)]
            den = a * lam + mp.fsum(mp.conj(win[i]) * u[i] for i in range(n))
            k = [v / den for v in u]
            v = [mp.fsum(mp.conj(win[j]) * Q[j, m] for j in range(n)) for m in range(n)]
            Q = mp.matrix([[(Q[i, m] - k[i] * v[m]) / a for m in range(n)] for i in range(n)])
            G = mp.matrix([[G[i, d] + k[i] * mp.conj(pred[d]) for d in range(D)] for i in range(n)])
            for d in range(D):
                z = Z[t, 0, d]
                err = max(err, float(abs(_mpc(z) - pred[d])))
        assert err <= 1e-16 * np.abs(Y).max(), err


def test_reduced_block_lstsq_against_mpmath_and_numpy():
    """a dead channel: the minimum-norm solution through mpmath's Hermitian eigendecomposition (the device's route),
    and np.linalg.lstsq in float64, against lstsq_solve"""
    rng = np.random.default_rng(3)
    D, taps, delay, T = 3, 2, 1, 30
    Y = _cplx(rng, D, T)
    Y[1] = 0
    w = rng.uniform(0.5, 2.0, T)
    _, G, R = WA.step_forward(Y.astype(LD), w.astype(np.longdouble), taps, delay)
    assert WA.lu_solve(R, np.eye(taps * D, dtype=LD)) is None                 # the zero pivot that takes lstsq
    Yt = WA.y_tilde(Y, taps, delay)
    P = (Yt * w) @ Y.conj().T
    ls = np.linalg.lstsq((Yt * w) @ Yt.conj().T, P, rcond=None)[0]
    assert np.abs(G.astype(complex) - ls).max() <= 1e-12 * np.abs(ls).max()
    with mp.workdps(DPS):
        n = taps * D
        Rm = mp.matrix([[_mpc(complex(R[i, j])) for j in range(n)] for i in range(n)])
        Rm = (Rm + Rm.H) / 2
        E, V = mp.eighe(Rm)
        cut = mp.mpf(2) ** -100 * max(abs(e) for e in E)
        Pm = mp.matrix([[_mpc(P[i, d]) for d in range(D)] for i in range(n)])
        Dinv = mp.diag([1 / e if abs(e) > cut else 0 for e in E])
        Gm = V * Dinv * V.H * Pm
        err = max(float(abs(_mpc(G[i, d]) - Gm[i, d]))
                  for i in range(n) for d in range(D))
        # R holds long-double sums of float64 data, P float64 sums: the long-double R is exact to its unit
        assert err <= 1e-14 * float(mp.norm(Gm, 'inf')), err


# ---- the forward bound rejects real defects at the longest T --------------------------------------------------------
def test_bound_rejects_defective_statistics_at_the_longest_t():
    G = _gpu_file()
    D, taps, delay = G.FRAME_SHAPE
    T = max(G.FRAME_COUNTS)
    Y = G.reverberant(1, D, T, delay, seed=5)[0][0]
    yl = Y.astype(LD)
    X, stages = WA.wpe_forward(yl, taps, delay, 1, 0, 'full')
    w, Gref, R = stages[0][:3]
    parts, span = corr_parts(T, D, taps, delay, False)
    bound = G.forward_bound(Y, Gref, [WA.kappa(R)], span, parts, taps, delay)
    Yt = WA.y_tilde(yl, taps, delay)
    P = (Yt * w) @ yl.conj().T
    wr = w.copy()
    wr[T // 2] = 0
    defects = {'one frame left out of R': (Yt * wr) @ Yt.conj().T,
               'R rounded to complex64': R.astype(np.complex64).astype(LD)}
    for what, Rbad in defects.items():
        Xbad = yl - WA.lu_solve(Rbad, P).conj().T @ Yt
        err = float(np.abs(Xbad - X).max())
        assert err > 100 * bound, (what, err, bound)
    # and the long-double X itself, rounded to float64, is inside it
    assert float(np.abs(X.astype(complex) - X).max()) < 1e-3 * bound
