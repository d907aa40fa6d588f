"""The references of tests/test_bss_eval_kernels_gpu.py, checked on the CPU (oracle/bss_eval_kernels_oracle.py).

- The restated shape choices and workspace layout equal the library's (pbb_bss_eval_workspace_bytes, which needs no
  GPU), and the GPU file's parameter lists reach every shape class at its edges.
- The exact integer correlations against int64 sums, and the long-double ones against them.
- Float64 models of the chunked, part-ordered correlation and of the tile energies stay within half the GPU file's
  bounds, and mutated models (a partial chunk dropped, a lag off by one, the last part skipped; the samples past T
  dropped, a tap off by one, P_j from the wrong filter) exceed them: the bounds can fail.
- The solve bound holds for LAPACK's factors, and the GPU file's pivot-forcing inputs make LAPACK pivot off the
  diagonal in many columns.
- The host restatement of the permutation scan equals np.mean / np.argmax and the NumPy restatement's select."""
import importlib
import os
import sys

import numpy as np
import pytest
import scipy.linalg

from oracle import bss_eval_kernels_oracle as O
from oracle import bss_eval_oracle as BO

L = O.L


def _gpu_file():
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    return importlib.import_module('test_bss_eval_kernels_gpu')


# ---- shapes and layout ------------------------------------------------------------------------------------------------
def test_shape_restatement_at_known_points():
    def sp(T):
        s = O.bss_shape(T, 1, 1)
        return s['span'], s['parts']
    assert sp(1) == (128, 1) and sp(128) == (128, 1) and sp(129) == (128, 2)
    assert sp(8064) == (128, 63) and sp(8065) == (128, 64) and sp(8192) == (128, 64)
    assert sp(8193) == (256, 33)
    assert sp((1 << 22) - 1) == (65536, 64) and sp(1 << 22) == (65536, 64)
    assert O.bss_shape(1, 1, 1)['tiles'] == 4 and O.bss_shape(1 << 22, 1, 1)['tiles'] == 32772
    assert [O.corr_ns(K, E) for K, E in ((4, 4), (4, 5), (8, 8), (8, 9))] == [1, 2, 2, 3]
    assert O.sums_width(8) == 8 and O.sums_width(9) == 16


def _sweep():
    G = _gpu_file()
    shapes = {(K, E, T) for K, E, T in G.INT_CASES}
    shapes |= {(K, E, T) for _, K, E, T in G.STAGE_CASES}
    Ts = [1, 2, 127, 128, 129, 511, 512, 513, 4096, 8063, 8064, 8065, 8191, 8192, 8193, 8320, 100001, 160000,
          (1 << 22) - 1, 1 << 22]
    shapes |= {(K, E, T) for K in range(1, 9) for E in (K, K + 1) for T in Ts}
    return sorted(shapes)


def test_layout_equals_the_library():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    for K, E, T in _sweep():
        for group in (1, 3, 7):
            want = lib.pbb_bss_eval_workspace_bytes(group, K, E, T)
            lay = O.bss_layout(group, K, E, T)
            assert want == lay['total'], (group, K, E, T)
            assert all(v % 256 == 0 for k, v in lay.items() if k != 'total')
    assert lib.pbb_bss_eval_workspace_bytes(1, 9, 9, 100) == 0
    assert lib.pbb_bss_eval_workspace_bytes(1, 2, 4, 100) == 0


def test_stage_views_fill_the_layout():
    """the views of `stages` cover the workspace exactly up to the 256-byte padding"""
    for K, E, T, group in ((1, 2, 513, 2), (3, 4, 8193, 1), (8, 9, 3586, 1)):
        lay = O.bss_layout(group, K, E, T)
        ws = np.zeros(lay['total'], np.uint8)
        st = O.stages(ws, group, K, E, T)
        assert st['R'].shape == (group, K, K + E, L)
        assert st['G'].shape == (group, K * L, K * L + 16)
        assert (st['Gb'] is None) == (K == 1)
        end = st['sums'].ctypes.data + st['sums'].nbytes
        assert end == ws.ctypes.data + lay['total']
        assert st['R'].ctypes.data - ws.ctypes.data == lay['R']


def test_gpu_parameters_reach_every_class_at_its_edges():
    G = _gpu_file()
    ints = G.INT_CASES
    Ts = {T for _, _, T in ints}
    assert any(T < 128 for T in Ts) and any(128 < T < 512 for T in Ts)
    for r in (0, 1, 127):                                          # partial chunks at K >= 2 too
        assert any(T % 128 == r and K >= 2 for K, _, T in ints), r
    parts = {O.bss_shape(T, 1, 1)['parts'] for T in Ts}
    assert 1 in parts and 64 in parts
    assert any(T % O.bss_shape(T, 1, 1)['span'] for T in Ts)        # a partial last part
    assert {8064, 8065, 8192, 8193, (1 << 22) - 1, 1 << 22} <= Ts
    assert {K for K, _, T in ints if T == 1 << 22} == set(range(1, 9))
    assert {K + E for K, E, _ in ints} >= {8, 9, 16, 17}
    assert {O.corr_ns(K, E) for K, E, _ in ints} == {1, 2, 3}
    stage = [(K, E, T) for _, K, E, T in G.STAGE_CASES]
    for K in range(2, 9):                                          # the smallest valid T of each K >= 2
        assert (K, 512 * K - 510) in {(k, T) for k, _, T in stage}, K
    for K, E, T in stage + ints:
        if T + L - 1 > K * L:
            assert T >= 512 * K - 510
    tails = {(T + L - 1) % O.TILE for _, _, T in stage} | {(T + L - 1) % O.TILE for _, _, T in ints}
    assert {0, 1, 127} <= tails                                    # full and partial last projection tiles
    assert {(8, 8), (8, 9)} <= {(K, E) for K, E, _ in stage}       # E = 8 against E = 9 at N = 4096
    assert {O.sums_width(E) for _, E, _ in stage} == {8, 16}
    assert {K for K, _, _ in stage} == set(range(1, 9)) and {K for K, _, _ in ints} == set(range(1, 9))
    assert {E - K for K, E, _ in stage} == {0, 1} and {E - K for K, E, _ in ints} == {0, 1}
    assert {k for k, *_ in G.STAGE_CASES} == {'white', 'ar', 'speech', 'periodic', 'pivot'}
    assert max(T for *_, T in G.STAGE_CASES) <= G.LD_CORR_UP_TO
    assert G.spot_tiles(1 << 22) == [0, 1, 16386, 32770, 32771]
    assert G.spot_tiles(100001) == [0, 1, 393, 784, 785]


# ---- correlations -----------------------------------------------------------------------------------------------------
def _int64_correlations(refs, sigs):
    K, T = refs.shape
    r, s = refs.astype(np.int64), sigs.astype(np.int64)
    out = np.zeros((K, s.shape[0], L), np.int64)
    for a in range(K):
        for d in range(min(L, T)):
            out[a, :, d] = s[:, d:] @ r[a, :T - d]
    return out


@pytest.mark.parametrize('T', [1, 127, 513, 1025, 5000])
def test_exact_correlations_against_int64(T):
    rng = np.random.default_rng(T)
    refs, est = O.integers(rng, 2, 3, T)
    sigs = np.concatenate([refs, est])
    want = _int64_correlations(refs, sigs)
    np.testing.assert_array_equal(O.exact_int_correlations(refs, sigs), want.astype(np.float64))
    np.testing.assert_array_equal(O.lag_correlations(refs, sigs), want.astype(O.LD))


def test_exact_correlations_at_full_magnitude():
    """|x| = 2^10 everywhere over 2^20 samples: sums of 2^40, still within 1/4 of the integer before rounding"""
    T = 1 << 20
    rng = np.random.default_rng(3)
    refs = 1024.0 * rng.choice([-1.0, 1.0], (1, T))
    sigs = np.concatenate([refs, 1024.0 * np.ones((1, T))])
    got = O.exact_int_correlations(refs, sigs)
    assert got[0, 0, 0] == T * 2.0 ** 20
    np.testing.assert_array_equal(got[0, 1], [1024.0 * refs[0, :T - d].sum() for d in range(L)])


def test_correlation_model_within_half_the_bound_and_mutants_exceed_it():
    T = 10000                           # span 256, 40 parts, a 16-sample last part: a partial chunk at K >= 2
    rng = np.random.default_rng(1)
    refs, est = O.ar_coloured(rng, 2, 3, T)
    sigs = np.concatenate([refs, est])
    ref = O.lag_correlations(refs, sigs)
    bound = O.corr_bound(O.lag_correlations(np.abs(refs), np.abs(sigs), np.float64), T)
    s = O.bss_shape(T, 2, 3)
    assert s['parts'] == 40 and T % s['span'] % O.CHUNK
    model = O.chunked_correlation_model(refs, sigs, T)
    assert np.all(np.abs(model - ref) <= 0.5 * bound)
    for kw in (dict(drop_partial_chunk=True), dict(lag_shift=1), dict(skip_last_part=True)):
        bad = O.chunked_correlation_model(refs, sigs, T, **kw)
        assert np.any(np.abs(bad - ref) > bound), kw


# ---- solves -----------------------------------------------------------------------------------------------------------
def _system(kind, K, E, T, seed):
    G = _gpu_file()
    refs, est = G.signals(kind, K, E, T, seed)
    R = O.lag_correlations(refs, np.concatenate([refs, est]), np.float64)
    return refs, est, R


def test_pivoting_inputs_pivot_off_the_diagonal():
    """LAPACK's getrf on the GPU file's pivot-forcing systems: many pivots leave the diagonal"""
    G = _gpu_file()
    for kind, K, E, T in G.STAGE_CASES:
        if kind != 'pivot':
            continue
        _, _, R = _system(kind, K, E, T, seed=K * 1000 + E * 10 + T % 7)
        A, _ = O.assemble(R, K, E)
        _, piv = scipy.linalg.lu_factor(A)
        moved = int(np.sum(piv != np.arange(len(piv))))
        assert moved >= len(piv) // 4, (K, moved, len(piv))


def test_solve_bound_holds_for_lapack_and_rejects_a_perturbed_solution():
    refs, est, R = _system('pivot', 3, 4, 3000, seed=2)
    K, E = 3, 4
    A, D = O.assemble(R, K, E)
    lu, piv = scipy.linalg.lu_factor(A)
    c = scipy.linalg.lu_solve((lu, piv), D)
    F = np.concatenate([lu, c], axis=1)
    err, bound, lmax, growth = O.solve_check(A, D, F)
    assert lmax <= 1 and growth >= 1 and np.all(err <= 0.5 * bound), err / bound
    c2 = c * (1 + 1e-9)
    err2, *_ = O.solve_check(A, D, np.concatenate([lu, c2], axis=1))
    assert np.all(err2 > bound)
    # the blocks the same way
    Aj, Dj = O.assemble(R, K, E, block=1)
    np.testing.assert_array_equal(Aj, A[L:2 * L, L:2 * L])
    np.testing.assert_array_equal(Dj, D[L:2 * L])


# ---- projections ------------------------------------------------------------------------------------------------------
def _solutions(R, K, E):
    A, D = O.assemble(R, K, E)
    c_all = np.linalg.solve(A, D).reshape(K, L, E)
    if K == 1:
        return c_all, c_all
    return c_all, np.stack([np.linalg.solve(*O.assemble(R, K, E, block=j)) for j in range(K)])


@pytest.mark.parametrize('K,E,T', [(1, 2, 700), (2, 3, 1700)])
def test_projection_model_within_half_the_bound_and_mutants_exceed_it(K, E, T):
    rng = np.random.default_rng(K)
    refs, est = O.white(rng, K, E, T)
    sig = np.concatenate([refs, est])
    R = O.lag_correlations(refs, sig, np.float64)
    c_all, c_one = _solutions(R, K, E)
    tiles = list(range(O.bss_shape(T, K, E)['tiles']))
    ref, bound = O.tile_energies(sig, K, E, T, c_all, c_one, tiles)
    model = O.projection_model(sig, K, E, T, c_all, c_one, tiles)
    assert np.all(np.abs(model - ref) <= 0.5 * bound)
    mutants = [dict(drop_tail=True), dict(tap_shift=1)] + ([dict(own_block_from_all=True)] if K > 1 else [])
    for kw in mutants:
        bad = O.projection_model(sig, K, E, T, c_all, c_one, tiles, **kw)
        assert np.any(np.abs(bad - ref) > bound), kw
    # the pair matrices of the model's totals against the NumPy restatement of BSS Eval
    tot = np.zeros((K + 1, 3, O.sums_width(E)))
    tot[..., :E] = model.sum(axis=0)
    for got, want in zip(O.pairs_from_totals(tot, K, E), BO.pair_matrices(refs, est)):
        fin = np.isfinite(want)
        np.testing.assert_array_equal(np.isfinite(got), fin)
        np.testing.assert_allclose(got[fin], want[fin], rtol=1e-9, atol=1e-9)


# ---- ratios and the permutation ---------------------------------------------------------------------------------------
def test_mean_and_argmax_restatement_equal_numpy():
    rng = np.random.default_rng(4)
    for K in range(1, 9):
        v = rng.standard_normal((4000, K)) * 10.0 ** rng.integers(-8, 9, (4000, K))
        v[rng.random((4000, K)) < 0.05] = np.inf
        v[rng.random((4000, K)) < 0.05] = -np.inf
        v[rng.random((4000, K)) < 0.02] = np.nan
        with np.errstate(invalid='ignore'):
            want = np.array([np.mean(r) for r in v])
            got = O.np_mean_rows(v)
        np.testing.assert_array_equal(got, want)
        for m in (got, np.nan_to_num(got, nan=0.0), np.round(np.nan_to_num(got, nan=0.0, posinf=1, neginf=0))):
            assert O.first_argmax(m) == int(np.argmax(m))


def test_selection_restatement_equals_the_numpy_select():
    rng = np.random.default_rng(5)
    inf = np.inf
    cases = [rng.standard_normal((E, K)) for K in range(1, 8) for E in (K, K + 1)]
    cases += [np.array([[1.0, inf], [-inf, 0.0], [2.0, 2.0]]), np.ones((3, 2)), np.full((9, 8), np.nan),
              np.round(rng.standard_normal((9, 8)))]
    for sir in cases:
        E, K = sir.shape
        r, perm = O.select(sir)
        np.testing.assert_array_equal(perm, BO.select(sir, sir, sir)[3])
        assert tuple(O.permutations(E, K)[r]) == tuple(perm)


def test_safe_db_and_tile_totals():
    assert O.safe_db(1.0, 0.0) == np.inf and O.safe_db(0.0, 0.0) == np.inf and O.safe_db(0.0, 1.0) == -np.inf
    assert O.safe_db(10.0, 1.0) == 10.0
    sums = np.array([[[[1.0]]], [[[2.0 ** -60]]], [[[-1.0]]]])
    assert O.tile_totals(sums)[0, 0, 0] == 0.0          # ((1 + 2^-60) - 1): in order, not pairwise
