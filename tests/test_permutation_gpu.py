"""DHTV permutation alignment on the device: integer mappings must be EXACTLY
the reference's (golden fixtures produced by the unmodified reference)."""
import os
import sys

import numpy as np
import pytest

from conftest import load_golden
from oracle import pb_bss_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu


def test_mapping_matches_reference_golden():
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    g = load_golden('permutation')
    for tag, stft in (('a', 512), ('b', 1024)):
        al = DHTVPermutationAlignment.from_stft_size(stft)
        assert al.alignment_plan == g[f'{tag}_plan'].tolist()
        mask = g[f'{tag}_mask']
        mapping = al.calculate_mapping(mask)
        assert mapping.dtype == np.int64 and mapping.shape == g[f'{tag}_mapping'].shape
        np.testing.assert_array_equal(mapping, g[f'{tag}_mapping'])
        np.testing.assert_array_equal(al.apply_mapping(mask, mapping), g[f'{tag}_aligned'])
        np.testing.assert_array_equal(al(mask), g[f'{tag}_aligned'])
    al = DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                  main_iterations=5, sub_iterations=2)
    assert al.alignment_plan == g['c_plan'].tolist()
    np.testing.assert_array_equal(al.calculate_mapping(g['c_mask']), g['c_mapping'])


@pytest.mark.parametrize('metric', ['cos', 'multiply', 'euclidean'])
@pytest.mark.parametrize('algorithm', ['greedy', 'optimal'])
def test_dhtv_options_match_reference_golden(metric, algorithm):
    """similarity_metric / algorithm of DHTVPermutationAlignment (permutation_alignment.py:133-163,380-420,556-585)."""
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    g = load_golden('permutation')
    al = DHTVPermutationAlignment(stft_size=512, segment_start=70, segment_width=100, segment_shift=20,
                                  main_iterations=20, sub_iterations=2, similarity_metric=metric, algorithm=algorithm)
    np.testing.assert_array_equal(al.calculate_mapping(g['a_mask']), g[f'opt_{metric}_{algorithm}'])


def test_dhtv_option_errors():
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    kw = dict(stft_size=512, segment_start=70, segment_width=100, segment_shift=20, main_iterations=2, sub_iterations=2)
    with pytest.raises(AttributeError):
        DHTVPermutationAlignment(similarity_metric='coss', **kw)
    with pytest.raises(ValueError):
        DHTVPermutationAlignment(algorithm='best', **kw).calculate_mapping(load_golden('permutation')['a_mask'])


def test_full_size_alignment_recovers_a_random_permutation():
    """K=3, F=513, T=500 (BASELINE.json config 3): permute a consistent mask per
    bin, align, and check against the oracle and the sortedness property
    (every bin ends up in the same global order)."""
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment, apply_mapping
    rng = np.random.RandomState(0)
    K, F, T = 3, 513, 500
    proto = rng.uniform(size=(K, 1, T)) ** 4
    mask = proto + 0.3 * rng.uniform(size=(K, F, T))
    mask /= mask.sum(0, keepdims=True)
    perm = np.stack([rng.permutation(K) for _ in range(F)], axis=1)
    permuted = mask[perm, np.arange(F)]
    al = DHTVPermutationAlignment.from_stft_size(1024)
    mapping = al.calculate_mapping(permuted)
    np.testing.assert_array_equal(mapping, O.dhtv_calculate_mapping(permuted, O.dhtv_plan_from_stft_size(1024)))
    aligned = apply_mapping(permuted, mapping)
    # up to ONE global permutation the original order is restored
    order = np.argmax(np.einsum('kft,lft->kl', aligned, mask), axis=1)
    assert sorted(order.tolist()) == [0, 1, 2]
    np.testing.assert_array_equal(aligned, mask[order])
    # permutations: every column of the mapping is a permutation of range(K)
    assert np.all(np.sort(mapping, axis=0) == np.arange(K)[:, None])


def test_apply_mapping_trailing_dims_and_device_tensors():
    import torch
    from pb_bss_b200.permutation_alignment import apply_mapping, sample_random_mapping
    rng = np.random.RandomState(1)
    K, F = 4, 9
    mask = rng.uniform(size=(K, F, 5, 3))
    mapping = sample_random_mapping(K, F, rng)
    np.testing.assert_array_equal(apply_mapping(mask, mapping), mask[mapping, range(F)])
    out = apply_mapping(torch.from_numpy(mask).cuda(), torch.from_numpy(mapping).cuda())
    assert out.is_cuda
    np.testing.assert_array_equal(out.cpu().numpy(), mask[mapping, range(F)])


METRICS = ('cos', 'euclidean', 'multiply')


@pytest.mark.parametrize('metric', METRICS)
def test_greedy_and_oracle_alignment_match_reference_golden(metric):
    """GreedyPermutationAlignment / OraclePermutationAlignment (permutation_alignment.py:592-786):
    exact integer equality with the mappings of the unmodified reference."""
    from pb_bss_b200.permutation_alignment import GreedyPermutationAlignment, OraclePermutationAlignment
    g = load_golden('permutation_greedy_oracle')
    for tag, mask, ref in (('', g['mask'], g['reference_mask']), ('noise_', g['noise'], g['noise_reference'])):
        got = GreedyPermutationAlignment(metric).calculate_mapping(mask)
        assert got.dtype == np.int64
        np.testing.assert_array_equal(got, g[f'greedy_{tag}{metric}'])
        for alg in ('greedy', 'optimal'):
            al = OraclePermutationAlignment(metric, alg)
            np.testing.assert_array_equal(al.calculate_mapping(mask, ref), g[f'oracle_{tag}{metric}_{alg}'])
    # the oracle alignment undoes the random permutation of the synthetic mask
    aligned = OraclePermutationAlignment(metric)(g['mask'], g['reference_mask'])
    np.testing.assert_array_equal(aligned, g['reference_mask'])


def test_mapping_from_score_matrix_known_answers_and_errors():
    from pb_bss_b200.permutation_alignment import (GreedyPermutationAlignment, OraclePermutationAlignment,
                                                   _mapping_from_score_matrix)
    sm = np.array([[11, 10, 0], [4, 5, 10], [6, 0, 5]])  # doctest, permutation_alignment.py:475-508
    np.testing.assert_array_equal(_mapping_from_score_matrix(sm, 'optimal'), [1, 2, 0])
    np.testing.assert_array_equal(_mapping_from_score_matrix(sm, 'greedy'), [0, 2, 1])
    np.testing.assert_array_equal(_mapping_from_score_matrix([sm, sm], 'optimal'), [[1, 1], [2, 2], [0, 0]])
    with pytest.raises(ValueError, match='infeasible'):
        _mapping_from_score_matrix([[np.inf, 0], [1, 2]])
    with pytest.raises(ValueError):
        _mapping_from_score_matrix(sm, 'hungarian')
    with pytest.raises(ValueError):
        GreedyPermutationAlignment('coss')
    with pytest.raises(AttributeError, match='Suggestions'):
        OraclePermutationAlignment('coss')
    with pytest.raises(AssertionError):
        GreedyPermutationAlignment('cos').calculate_mapping(np.ones((3, 4, 5)))  # even F


def test_full_size_greedy_alignment_against_the_oracle():
    """F=513, K=3, T=500 (C3 shapes): the device mapping equals the NumPy restatement."""
    from pb_bss_b200.permutation_alignment import GreedyPermutationAlignment
    rng = np.random.RandomState(5)
    K, F, T = 3, 513, 500
    proto = rng.uniform(size=(K, 1, T)) ** 4
    mask = proto + 0.5 * rng.uniform(size=(K, F, T))
    mask /= mask.sum(0, keepdims=True)
    perm = np.stack([rng.permutation(K) for _ in range(F)], axis=1)
    mask = mask[perm, np.arange(F)]
    got = GreedyPermutationAlignment('cos').calculate_mapping(mask)
    np.testing.assert_array_equal(got, O.greedy_permutation_alignment(mask, 'cos'))
    aligned = mask[got, np.arange(F)]
    # every bin now carries the same source order as bin 0
    assert (np.argmax(np.einsum('kft,jt->fkj', aligned, aligned[:, 0]), axis=-1) == np.arange(K)).all()


# ---- every DHTV kernel on the same inputs ---------------------------------------------------------------------------
# pbb_dhtv_mapping_ex runs dhtv_cluster_kernel when the widest segment fits one thread-block cluster (templated for
# K = 2, 3, 4, generic for K = 5..9), and dhtv_coop_kernel (grid barriers) when it does not or with PBB_DHTV_COOP=1.
# The switch is read once per process, so each path runs in a child process of its own (this file run as a script)
# over the same cases.
#
# The kernels add the centroid in different orders and apply the cos normalisation differently, so a decision within
# rounding of a tie may legitimately differ between them.  Generated cases therefore assert the oracle's decision
# margin (relative to the largest |score| of the bin) before their mappings are compared exactly; the fixture's cases
# carry that check in tests/test_oracle_golden.py, and its exact-tie cases (tie_*) must follow the reference's first
# maximum in row-major order on every path.
MARGIN = 1e-9
ALGORITHMS = ('greedy', 'optimal')
ALL = tuple((m, a) for m in METRICS for a in ALGORITHMS)
GREEDY = tuple((m, 'greedy') for m in METRICS)
SOME = (('cos', 'greedy'), ('multiply', 'greedy'), ('euclidean', 'optimal'))
MULTIPLY = (('multiply', 'greedy'), ('multiply', 'optimal'))
KERNELS = {'cluster': 'dhtv_cluster_kernel', 'coop': 'dhtv_coop_kernel'}


def _generated_dhtv_cases():
    """name -> (mask builder, plan, (metric, algorithm) pairs, kernel the default dispatch picks)."""
    p512, p1024 = O.dhtv_plan_from_stft_size(512), O.dhtv_plan_from_stft_size(1024)

    def pm(K, F, T, seed):
        return lambda: synth.permuted_mask(K, F, T, seed=seed)[0]

    cases = {
        # long utterances: (2 + ceil(widest / 16)) K T 8 B > 200 KB, so the segments do not fit the cluster
        'long_f513_k3_t1000': (pm(3, 513, 1000, 1), p1024, ALL, 'coop'),
        'long_f257_k4_t1000': (pm(4, 257, 1000, 2), p512, ALL, 'coop'),
        'long_f257_k9_t400': (pm(9, 257, 400, 3), p512, GREEDY, 'coop'),
        # dispatch boundaries: 16 bins per CTA of a 16-CTA cluster or one more; (2 + 8) K T 8 B = 200 KB at T = 853
        'seg256': (pm(3, 257, 200, 4), [[3, 0, 256], [2, 1, 257]], SOME, 'cluster'),
        'seg257': (pm(3, 257, 200, 4), [[3, 0, 257]], SOME, 'coop'),
        't853': (pm(3, 513, 853, 5), p1024, SOME, 'cluster'),
        't854': (pm(3, 513, 854, 5), p1024, SOME, 'coop'),
        # K T 8 B just under 200 KB: one CTA per SM, so the grid is smaller than the segment's 1025 bins
        'wide_k3_t8533': (pm(3, 1025, 8533, 6), [[2, 0, 1025]], SOME, 'coop'),
        # K T 8 B at 200 KB exactly, and just under it for K = 9
        'limit_k4_t6400': (pm(4, 3, 6400, 7), [[2, 0, 3]], SOME, 'coop'),
        'limit_k9_t2844': (pm(9, 3, 2844, 8), [[2, 0, 3]], GREEDY, 'coop'),
        # degenerate plans: one bin; 0-iteration and 1-bin segments (there the centroid is the bin itself, so the cos
        # and euclidean diagonals tie: 'multiply' only)
        'f1_k3': (pm(3, 1, 40, 9), [[2, 0, 1]], MULTIPLY, 'cluster'),
        'f1_k9': (pm(9, 1, 40, 10), [[2, 0, 1]], MULTIPLY, 'cluster'),
        'plan_edge_k6': (pm(6, 33, 50, 11), [[0, 0, 33], [2, 7, 8], [3, 0, 33], [0, 3, 9], [1, 32, 33]], MULTIPLY,
                         'cluster'),
    }
    # K = 5..9 on the generic cluster kernel: T <= 150 and segments <= 128 bins fit an 8-CTA cluster as well
    for K in range(5, 10):
        cases[f'cluster_k{K}'] = (pm(K, 129, 150, 20 + K), [[5, 0, 128], [2, 40, 129], [1, 100, 129]],
                                  ALL if K <= 7 else GREEDY, 'cluster')
    for K in (8, 9):  # 'optimal' tries all K! permutations: a few bins
        cases[f'cluster_k{K}_optimal'] = (pm(K, 5, 150, 30 + K), [[2, 0, 5]],
                                          tuple((m, 'optimal') for m in METRICS), 'cluster')
    # frame counts around the warp width and the 512-frame chunks of the row loads and score loops.  At T = 1 every cos
    # feature is 1 up to rounding, and euclidean permutation sums such as |x_a - c_1| + |x_b - c_2| and
    # |x_b - c_1| + |x_a - c_2| are equal up to rounding
    for T in (1, 31, 33, 512, 513):
        for K in (3, 5):
            combos = ALL if T > 1 else MULTIPLY + (('euclidean', 'greedy'),)
            cases[f'frames_k{K}_t{T}'] = (pm(K, 33, T, 40 + T + K), [[3, 0, 20], [2, 10, 33]], combos, 'cluster')
    return cases


def _dhtv_cases(golden):
    """(name, mask, plan, combos, default kernel) for the fixture's cases, then the generated ones."""
    for name in golden['dhtv_cases'].tolist():
        combos = tuple((m, a) for m in METRICS for a in ALGORITHMS if f'{name}_{m}_{a}' in golden)
        yield name, golden[f'{name}_mask'], golden[f'{name}_plan'].tolist(), combos, 'cluster'
    for name, (build, plan, combos, kernel) in _generated_dhtv_cases().items():
        yield name, build(), plan, combos, kernel


def _aligner(plan, metric, algorithm):
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment

    class PlanAligner(DHTVPermutationAlignment):
        @property
        def alignment_plan(self):
            return [list(map(int, p)) for p in plan]

    return PlanAligner(stft_size=0, segment_start=0, segment_width=0, segment_shift=1, main_iterations=0,
                       sub_iterations=0, similarity_metric=metric, algorithm=algorithm)


def _recorded_launches(lib):
    """Names of the launches recorded since the last pbb_profile_reset (pbb_profile_dump prints them on fd 2)."""
    import tempfile
    import torch
    torch.cuda.synchronize()
    sys.stderr.flush()
    with tempfile.TemporaryFile(mode='w+') as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            lib.pbb_profile_dump()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        names = [line.split()[1] for line in tmp.read().splitlines() if line.startswith('[pbb]')]
    lib.pbb_profile_reset()
    return names


def _run_dhtv_cases(out_path):
    """Child process: every case on the path this process's environment selects -> mappings and launched kernels."""
    import torch
    from pb_bss_b200 import _lib
    lib = _lib.load()
    lib.pbb_profile_enable(1)
    out = {}
    for name, mask, plan, combos, _ in _dhtv_cases(load_golden('permutation_classes')):
        m = torch.from_numpy(mask).cuda()
        for metric, algorithm in combos:
            lib.pbb_profile_reset()
            key = f'{name}_{metric}_{algorithm}'
            out[key] = _aligner(plan, metric, algorithm).calculate_mapping(m).cpu().numpy()
            out[f'kernels_{key}'] = np.array(','.join(_recorded_launches(lib)))
        del m
    np.savez(out_path, **out)


PATHS = {'default': {}, 'coop': {'PBB_DHTV_COOP': '1'}}


@pytest.fixture(scope='module')
def dhtv_paths(tmp_path_factory):
    """Runs the two child processes (concurrently, while the oracle runs here) -> (expected, results, kernels):
    the fixture's mapping for its cases, the oracle's for the generated ones."""
    import subprocess
    tmp = tmp_path_factory.mktemp('dhtv')
    procs = {}
    try:
        for path, env in PATHS.items():
            e = {k: v for k, v in os.environ.items() if k != 'PBB_DHTV_COOP'}
            e.update(env)
            procs[path] = subprocess.Popen([sys.executable, os.path.abspath(__file__), str(tmp / f'{path}.npz')], env=e)
        g = load_golden('permutation_classes')
        expected, kernels = {}, {}
        for name, mask, plan, combos, kernel in _dhtv_cases(g):
            for metric, algorithm in combos:
                key = f'{name}_{metric}_{algorithm}'
                kernels[key] = kernel
                if key in g:
                    expected[key] = g[key]
                    continue
                expected[key], margin = O.dhtv_calculate_mapping(mask, plan, metric, algorithm, return_margin=True)
                assert margin > MARGIN, (key, margin)  # precondition: no decision within rounding of a tie
        for path, p in procs.items():
            assert p.wait(timeout=600) == 0, path
    finally:
        for p in procs.values():
            if p.poll() is None:
                p.kill()
                p.wait()
    results = {path: dict(np.load(tmp / f'{path}.npz')) for path in PATHS}
    return expected, results, kernels


@pytest.mark.parametrize('path', list(PATHS))
def test_dhtv_every_kernel_matches_the_oracle(dhtv_paths, path):
    """Each path on every case: K = 2..9 on the cluster kernel (templated and generic), long utterances and the
    dispatch boundaries on the coop kernel by default, exact ties, degenerate plans, frame-count edges; every metric
    and assignment.  Asserts which kernel ran, so the coverage cannot silently move to another kernel."""
    expected, results, kernels = dhtv_paths
    got = results[path]
    assert sorted(k for k in got if not k.startswith('kernels_')) == sorted(expected)
    ran = {}
    for key in expected:
        launched = got[f'kernels_{key}'].item().split(',')
        want = KERNELS[kernels[key] if path == 'default' else path]
        assert want in launched and not (set(KERNELS.values()) - {want}) & set(launched), (path, key, launched)
        ran.setdefault(want, []).append(key)
        np.testing.assert_array_equal(got[key], expected[key], err_msg=f'{path}: {key}')
    if path == 'default':
        # the generic cluster kernel ran for every K = 5..9, the coop kernel on the long utterances
        for K in range(5, 10):
            assert any(k.startswith((f'k{K}_', f'cluster_k{K}_')) for k in ran['dhtv_cluster_kernel']), K
        assert sum(k.startswith('long_') for k in ran['dhtv_coop_kernel']) == 2 * 6 + 3


@pytest.mark.parametrize('K,T', [(3, 8534), (9, 2845)])
def test_dhtv_centroid_size_limit(K, T):
    """K T 8 B one element over the 200 KB of the shared-memory centroid: ValueError before any launch (K T 8 B at or
    just under the limit runs: limit_k4_t6400, limit_k9_t2844, wide_k3_t8533 above)."""
    import torch
    from pb_bss_b200 import _lib
    lib = _lib.load()
    mask = torch.full((K, 3, T), 1.0 / K, dtype=torch.float64, device='cuda')
    torch.cuda.synchronize()
    before = lib.pbb_launch_count()
    with pytest.raises(ValueError, match='too large'):
        _aligner([[2, 0, 3]], 'cos', 'greedy').calculate_mapping(mask)
    assert lib.pbb_launch_count() == before


@pytest.mark.parametrize('K', range(2, 10))
def test_greedy_and_oracle_alignment_all_class_counts(K):
    """GreedyPermutationAlignment / OraclePermutationAlignment (score_matrix_kernel, mapping_from_score_kernel,
    chain_mapping_kernel) for K = 2..9: the reference's fixtures, then generated inputs against the oracle with T = 1,
    an odd T and leading dims of the Oracle alignment."""
    import torch
    from pb_bss_b200.permutation_alignment import GreedyPermutationAlignment, OraclePermutationAlignment
    g = load_golden('permutation_classes')
    mask, perm = g[f'k{K}_mask'], g[f'k{K}_perm']
    reference = mask[np.argsort(perm, axis=0), np.arange(mask.shape[1])]
    for tag, m, ref in (('k', mask, reference), ('noise_k', g[f'noise_k{K}_mask'], g[f'noise_k{K}_reference'])):
        for metric in METRICS:
            np.testing.assert_array_equal(GreedyPermutationAlignment(metric).calculate_mapping(m),
                                          g[f'{tag}{K}_greedy_{metric}'])
            for alg in ALGORITHMS:
                key = f'{tag}{K}_oracle_{metric}_{alg}'
                if key in g:
                    np.testing.assert_array_equal(OraclePermutationAlignment(metric, alg).calculate_mapping(m, ref),
                                                  g[key], err_msg=key)
    for T in (1, 37):
        F = 33 if K <= 7 else 9
        mask, clean, _ = synth.permuted_mask(K, F, T, seed=200 + K + T)
        lead = synth.permuted_mask(K, 15, T, seed=300 + K + T)[0].reshape(K, 3, 5, T)
        lead_ref = np.random.RandomState(K + T).uniform(size=lead.shape)
        # T = 1: every cos feature is 1 up to rounding, and euclidean permutation sums tie up to rounding
        metrics = METRICS if T > 1 else ('multiply', 'euclidean')
        for metric in metrics:
            want, margin = O.greedy_permutation_alignment(mask, metric, return_margin=True)
            assert margin > MARGIN, (T, metric, margin)
            np.testing.assert_array_equal(GreedyPermutationAlignment(metric).calculate_mapping(mask), want)
            for alg in ALGORITHMS if K <= 8 and (T > 1 or metric == 'multiply') else ('greedy',):
                al = OraclePermutationAlignment(metric, alg)
                want, margin = O.oracle_permutation_alignment(mask, clean, metric, alg, return_margin=True)
                assert margin > MARGIN, (T, metric, alg, margin)
                np.testing.assert_array_equal(al.calculate_mapping(mask, clean), want)
                want, margin = O.oracle_permutation_alignment(lead.reshape(K, 15, T), lead_ref.reshape(K, 15, T),
                                                              metric, alg, return_margin=True)
                assert margin > MARGIN, (T, metric, alg, margin)
                got = al.calculate_mapping(torch.from_numpy(lead).cuda(), torch.from_numpy(lead_ref).cuda())
                assert got.is_cuda and tuple(got.shape) == (K, 3, 5)
                np.testing.assert_array_equal(got.cpu().numpy(), want.reshape(K, 3, 5))


if __name__ == '__main__':
    _run_dhtv_cases(sys.argv[1])
