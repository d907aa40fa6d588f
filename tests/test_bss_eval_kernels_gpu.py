"""BSS Eval's kernels stage by stage (csrc/bss_eval.cuh), read from the workspace of a one-group pbb_bss_eval call at the
offsets of bss_layout (restated in oracle/bss_eval_kernels_oracle.py, which tests/test_bss_eval_kernels_oracle.py checks
on the CPU together with the claim that the lists below reach every shape class at its edges).

Bounds (u = 2^-53):

- lag correlations R: integer signals with |x| <= 2^10 give integer products and partial sums below 2^42, so R must
  equal the exact correlation bit for bit; real signals: |R - R*| <= u (span + parts) sum_v |a[v - d]| |b[v]| against
  the long-double R*, one rounding per product along a part's span and one per part of the ordered sum.
- the solves of G and of every diagonal block G_jj, rebuilt from the device's own R: every stored |l| <= 1 (partial
  pivoting), and per estimate column ||D - G c||_inf <= 3 n u || |L| (|U| |c|) ||_inf (Higham, Thm. 9.4), the
  residual taken in long double.  The growth factor max|U| / max|G| is recorded.
- the tile energies of P_j x, x - P_j x, P_all x - P_j x, P_all x and x - P_all x from the device's own c, against long
  double: per sample |P - P*| <= u (K L + 1) sum |c| |s| (L for P_j), and a tile's energy within
  sum_t (2 |d_t| delta_t + delta_t^2) plus the rounding of its fixed-order sum (oracle tile_energies).
- the (estimate, reference) ratios within 4 ulp of mir_eval's _safe_db of the device's own tile totals, and the
  selection equal to the host restatement (itertools order, np.mean, np.argmax) of the device's own SIR matrix.

The largest error-to-bound ratio of each group and the largest growth factor are printed at the end of the module
(pytest -s) and recorded in DESIGN.md."""
import collections
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_bss_eval_gpu import speech_like  # noqa: E402
from test_wpe_kernels_oracle import require_extended_precision  # noqa: E402

from oracle import bss_eval_kernels_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
require_extended_precision()

L = O.L
BIG_T = 1 << 22
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bss_eval.npz')

# ---- the parameter lists (their coverage is checked on the CPU) -----------------------------------------------------
# (K, E, T) of integer signals: T < 128 and < 512, T mod 128 in {0, 1, 127} at K >= 2, one part, a partial last part,
# the 64-part cap and the drop to span 256 (8064, 8065, 8192, 8193), 2^22 - 1 and 2^22 for every K, and NS = 1 / 2 / 3
INT_CASES = ([(1, 2, 1), (1, 1, 127), (1, 2, 128), (2, 3, 129), (3, 3, 511), (2, 2, 512), (4, 5, 513),
              (4, 4, 8064), (6, 7, 8065), (7, 7, 8191), (8, 9, 8192), (3, 4, 8193), (5, 5, 100001),
              (1, 2, BIG_T - 1), (8, 9, BIG_T - 1)]
             + [(K, K + K % 2, BIG_T) for K in range(1, 9)])
# (signal kind, K, E, T) of real signals, every stage against long double: the smallest valid T = 512 K - 510 of each
# K >= 2, full and partial projection tiles, the reference's periodic doctest (kappa(G) ~ 1e19), pivot-forcing
# references, and K = 8 (N = 4096) with E = 8 and 9
STAGE_CASES = [('white', 1, 2, 1), ('ar', 1, 1, 100), ('white', 1, 2, 513), ('speech', 1, 2, 20000),
               ('white', 2, 3, 514), ('speech', 2, 2, 4000), ('periodic', 2, 2, 4000), ('ar', 2, 3, 20000),
               ('pivot', 2, 3, 3000), ('white', 3, 3, 1026), ('pivot', 3, 4, 6000), ('speech', 4, 5, 1538),
               ('ar', 4, 4, 8064), ('pivot', 5, 5, 2050), ('white', 6, 7, 2562), ('speech', 7, 7, 3074),
               ('pivot', 8, 8, 4200), ('speech', 8, 9, 3586)]
ALL_TILES_UP_TO = 20000        # every projection tile up to this T, else SPOT_TILES
LD_CORR_UP_TO = 20000          # the long-double correlation reference up to this T


def spot_tiles(T):
    """tiles 0, 1, the middle one, the last full one and the (partial) last one"""
    n = O.bss_shape(T, 1, 1)['tiles']
    full = (T + L - 1) % O.TILE == 0
    return sorted({0, min(1, n - 1), n // 2, n - 1 if full else max(0, n - 2), n - 1})


# ---- helpers ----------------------------------------------------------------------------------------------------------
RATIOS = collections.defaultdict(float)
GROWTH = collections.defaultdict(float)


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    for group, r in sorted(RATIOS.items()):
        print(f'\nbss_eval kernels: largest error / bound of {group}: {r:.3g}')
    for group, g in sorted(GROWTH.items()):
        print(f'\nbss_eval kernels: largest growth factor max|U| / max|G| of {group}: {g:.3g}')


def signals(kind, K, E, T, seed):
    """(references (K, T), estimates (E, T))"""
    rng = np.random.default_rng(seed)
    if kind == 'periodic':
        with np.load(GOLDEN) as g:
            ref, est = g['doctest_reference'], g['doctest_estimation']
        assert ref.shape == (K, T) and est.shape == (E, T)
        return ref.astype(np.float64), est.astype(np.float64)
    if kind == 'speech':
        return speech_like(rng, K, E, T)
    return {'white': O.white, 'ar': O.ar_coloured, 'pivot': O.pivoting, 'int': O.integers}[kind](rng, K, E, T)


def run(x, K, E, permute=True, group=None):
    """pbb_bss_eval on x (items, K + E, T) with `pairs` requested, on a workspace filled with NaN bytes; returns the
    outputs as NumPy and the stages of the last group (oracle stages)"""
    from pb_bss_b200 import _lib
    lib = _lib.load()
    items, S, T = x.shape
    assert S == K + E
    group = group or items
    nbytes = lib.pbb_bss_eval_workspace_bytes(group, K, E, T)
    assert nbytes == O.bss_layout(group, K, E, T)['total']
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device='cuda')
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float64)).cuda()
    f64 = dict(dtype=torch.float64, device='cuda')
    sdr, sir, sar = (torch.empty((items, K), **f64) for _ in range(3))
    sel = torch.empty((items, K), dtype=torch.int64, device='cuda')
    pairs = torch.empty((items, 3, E, K), **f64)
    status = torch.zeros(1, dtype=torch.int64, device='cuda')
    rc = lib.pbb_bss_eval(xd.data_ptr(), items, K, E, T, int(permute), group, ws.data_ptr(), nbytes, sdr.data_ptr(),
                          sir.data_ptr(), sar.data_ptr(), sel.data_ptr() if permute else None, pairs.data_ptr(),
                          status.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'pbb_bss_eval')
    torch.cuda.synchronize()
    last = items - (items - 1) // group * group
    out = dict(sdr=sdr.cpu().numpy(), sir=sir.cpu().numpy(), sar=sar.cpu().numpy(), pairs=pairs.cpu().numpy(),
               selection=sel.cpu().numpy() if permute else None, status=int(status.item()))
    out['stages'] = O.stages(ws.cpu().numpy(), group, K, E, T, last)
    return out


def _ratio(group, err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    if err.size == 0:
        return
    ok = err <= bound
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(err == 0, 0.0, err / bound)
    RATIOS[group] = max(RATIOS[group], float(r.max()))
    assert ok.all(), (group, float(r.max()), np.argwhere(~ok)[:5])


def check_correlations(R, ref, sig, T):
    R_ld = O.lag_correlations(ref, sig)
    mag = O.lag_correlations(np.abs(ref), np.abs(sig), np.float64)
    _ratio('correlations', np.abs(R.astype(O.LD) - R_ld).astype(np.float64), O.corr_bound(mag, T))


def check_solves(what, R, G, Gb, K, E):
    A, D = O.assemble(R, K, E)
    systems = [('G', A, D, G)]
    if K > 1:
        systems += [(f'G_{j}{j}', *O.assemble(R, K, E, block=j), Gb[j]) for j in range(K)]
    for name, A, D, F in systems:
        assert np.isfinite(F[:, :A.shape[0] + E]).all(), name
        err, bound, lmax, growth = O.solve_check(A, D, F)
        assert lmax <= 1.0, (what, name, lmax)
        _ratio('solves (G)' if name == 'G' else 'solves (diagonal blocks)', err, bound)
        GROWTH[what] = max(GROWTH[what], growth)


def check_projections(st, i, sig, K, E, T, tiles):
    c_all, c_one = O.solutions(st['G'][i], st['Gb'][i] if K > 1 else None, K, E)
    ref, bound = O.tile_energies(sig, K, E, T, c_all, c_one, tiles)
    got = st['sums'][i][tiles][..., :E]
    _ratio('tile energies', np.abs(got.astype(O.LD) - ref).astype(np.float64), bound)
    if K == 1:
        assert np.all(got[:, 0, 2] == 0)               # P_all - P_1 is identically zero


def check_ratios(out, st, i, item, K, E, permute=True):
    """the ratios and the selection of output item `item` against the tile sums of stage slot i"""
    tot = O.tile_totals(st['sums'][i])
    i = item
    for want, got in zip(O.pairs_from_totals(tot, K, E), out['pairs'][i]):
        fin = np.isfinite(want)
        np.testing.assert_array_equal(got[~fin], want[~fin])
        err = np.abs(got[fin] - want[fin])
        _ratio('ratios (ulp / 4)', err, 4 * np.spacing(np.abs(want[fin])))
    if K == 1:
        assert np.all(out['pairs'][i, 1] == np.inf)
    if permute:
        _, perm = O.select(out['pairs'][i, 1])
        np.testing.assert_array_equal(out['selection'][i], perm)
        k = np.arange(K)
        for q, name in enumerate(('sdr', 'sir', 'sar')):
            np.testing.assert_array_equal(out[name][i], out['pairs'][i, q][perm, k])


def check_item(what, out, i, ref, est, K, E, T, corr, item=None):
    """every stage of stage slot i (of the last group) and the outputs of batch item `item` (default i)"""
    item = i if item is None else item
    st = out['stages']
    sig = np.concatenate([ref, est])
    R = st['R'][i]
    assert np.isfinite(R).all()
    if corr == 'exact':
        np.testing.assert_array_equal(R, O.exact_int_correlations(ref, sig))
    else:
        check_correlations(R, ref, sig, T)
    if T + L - 1 <= K * L:     # the shifted references span every signal: G is singular or nearly so
        return
    assert st['flags'][i] == 0 and out['status'] == 0
    check_solves(what, R, st['G'][i], st['Gb'][i] if K > 1 else None, K, E)
    tiles = list(range(O.bss_shape(T, K, E)['tiles'])) if T <= ALL_TILES_UP_TO else spot_tiles(T)
    check_projections(st, i, sig, K, E, T, tiles)
    assert np.isfinite(st['sums'][i]).all()
    check_ratios(out, st, i, item, K, E)


# ---- 1. integer signals: exact correlations ---------------------------------------------------------------------------
@pytest.mark.parametrize('K,E,T', INT_CASES)
def test_integer_correlations_are_exact(K, E, T):
    ref, est = signals('int', K, E, T, seed=K * 100 + T % 1000)
    out = run(np.concatenate([ref, est])[None], K, E)
    check_item('integer signals', out, 0, ref, est, K, E, T, 'exact')


# ---- 2. real signals: every stage against long double -----------------------------------------------------------------
@pytest.mark.parametrize('kind,K,E,T', STAGE_CASES)
def test_stages_against_long_double(kind, K, E, T):
    ref, est = signals(kind, K, E, T, seed=K * 1000 + E * 10 + T % 7)
    out = run(np.concatenate([ref, est])[None], K, E)
    assert T <= LD_CORR_UP_TO
    check_item(kind, out, 0, ref, est, K, E, T, 'ld')


# ---- 3. the permutation scan ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 8])
def test_duplicated_estimates_tie_and_the_first_permutation_wins(K):
    """E = K + 1 estimates: estimate e is reference K - e (e >= 1) plus a little of the others, and estimate 0 is a
    bitwise copy of estimate 1.  The two best permutations, (K, ..., 2, 1) and (K, ..., 2, 0), then tie; at K = 8 they
    are the last two of 362 880 ranks, taken by threads 126 and 127 of the 256-thread stride in their last round."""
    E, T = K + 1, 4000
    rng = np.random.default_rng(K)
    ref, _ = O.white(rng, K, K, T)
    est = np.empty((E, T))
    for e in range(1, E):
        est[e] = ref[K - e] + 0.05 * ref.sum(0) * (e % 3 + 1) / 3 + 0.01 * rng.standard_normal(T)
    est[0] = est[1]
    out = run(np.concatenate([ref, est])[None], K, E)
    check_item('duplicated estimates', out, 0, ref, est, K, E, T, 'ld')
    pairs = out['pairs'][0]
    np.testing.assert_array_equal(pairs[:, 0], pairs[:, 1])      # bitwise equal rows for the duplicated estimate
    perms = O.permutations(E, K)
    means = O.np_mean_rows(pairs[1][perms, np.arange(K)])
    best = np.flatnonzero(means == means.max())
    assert len(best) == 2 and best[0] == len(perms) - 2, best
    np.testing.assert_array_equal(out['selection'][0], perms[best[0]])
    np.testing.assert_array_equal(out['selection'][0], np.r_[np.arange(K, 1, -1), 0])


# ---- 4. invariants ----------------------------------------------------------------------------------------------------
SCALES = [(-200, 200), (200, -200), (57, -133), (-3, 0)]


def test_power_of_two_scaling_is_exact():
    """references times 2^a and estimates times 2^b: R scales by 2^2a (reference columns) and 2^(a + b), the
    multipliers stay, U by 2^2a, c by 2^(b - a), the energies by 2^2b, and the ratios and the selection do not move"""
    K, E, T = 3, 4, 3000
    ref, est = signals('speech', K, E, T, seed=11)
    x = [np.concatenate([ref, est])] + [np.concatenate([ref * 2.0 ** a, est * 2.0 ** b]) for a, b in SCALES]
    out = run(np.stack(x), K, E)
    st = out['stages']
    N = K * L
    for n, (a, b) in enumerate(SCALES, start=1):
        np.testing.assert_array_equal(st['R'][n][:, :K], st['R'][0][:, :K] * 2.0 ** (2 * a))
        np.testing.assert_array_equal(st['R'][n][:, K:], st['R'][0][:, K:] * 2.0 ** (a + b))
        for F, F0, m in [(st['G'][n], st['G'][0], N)] + [(st['Gb'][n][j], st['Gb'][0][j], L) for j in range(K)]:
            np.testing.assert_array_equal(np.tril(F[:, :m], -1), np.tril(F0[:, :m], -1))
            np.testing.assert_array_equal(np.triu(F[:, :m]), np.triu(F0[:, :m]) * 2.0 ** (2 * a))
            np.testing.assert_array_equal(F[:, m:m + E], F0[:, m:m + E] * 2.0 ** (b - a))
        np.testing.assert_array_equal(st['sums'][n], st['sums'][0] * 2.0 ** (2 * b))
        for name in ('pairs', 'sdr', 'sir', 'sar', 'selection'):
            np.testing.assert_array_equal(out[name][n], out[name][0])
    check_item('scaling', out, 0, ref, est, K, E, T, 'ld')


def test_flagged_items_and_a_partial_last_group():
    """five items in groups of two: exactly singular systems at items 2 and 4, the last in the partial last group.  Two
    bitwise identical references make twin rows of [G | D] that the elimination updates alike, so the copy of a pivot
    row is eliminated to exact zeros and a later pivot is exactly zero.  The status names item 2 with flag 4, the
    flagged items are NaN with permutation 0, and the other items equal one-item runs bit for bit.  Then a zero estimate (flag 1) and a NaN sample (flag 2), and the
    stage contents of an item in a partial last group against its one-item run."""
    K, E, T = 2, 3, 3000
    items = []
    for i in range(5):
        ref, est = signals('speech', K, E, T, seed=50 + i)
        if i in (2, 4):
            ref[1] = ref[0]
        items.append(np.concatenate([ref, est]))
    x = np.stack(items)
    out = run(x, K, E, group=2)
    assert out['status'] == (3 << 3) | 4
    assert out['stages']['flags'][0] == 4                      # item 4, alone in the last group
    for i in range(5):
        if i in (2, 4):
            for name in ('sdr', 'sir', 'sar', 'pairs'):
                assert np.isnan(out[name][i]).all(), (i, name)
            np.testing.assert_array_equal(out['selection'][i], np.arange(K))
            continue
        one = run(x[i:i + 1], K, E)
        assert one['status'] == 0
        for name in ('sdr', 'sir', 'sar', 'pairs', 'selection'):
            np.testing.assert_array_equal(out[name][i], one[name][0])
    # a zero estimate and a non-finite sample
    bad = x[[0, 1, 3]].copy()
    bad[1, K + 1] = 0
    bad[2, 0, 17] = np.nan
    out = run(bad, K, E, group=2)
    assert out['status'] == (2 << 3) | 1
    assert out['stages']['flags'][0] & 2
    for i in (1, 2):
        assert np.isnan(out['pairs'][i]).all()
        np.testing.assert_array_equal(out['selection'][i], np.arange(K))
    # the stages of the item alone in the last group (regular) against its one-item run
    good = x[[0, 1, 3]]
    out = run(good, K, E, group=2)
    one = run(good[2:], K, E)
    for name in ('flags', 'R', 'G', 'Gb', 'sums'):
        np.testing.assert_array_equal(out['stages'][name], one['stages'][name])
    for name in ('pairs', 'selection'):
        np.testing.assert_array_equal(out[name][2], one[name][0])
    check_item('partial group', out, 0, x[3, :K], x[3, K:], K, E, T, 'ld', item=2)
