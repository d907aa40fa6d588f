"""Pins the oracle (oracle/pb_bss_oracle.py) to the reference: every function
is checked against fixtures produced by the unmodified reference
(oracle/make_golden.py) and against the known answers in the reference's own
doctests / unit tests.  CPU only."""
import numpy as np
import pytest

from oracle import pb_bss_oracle as O
from conftest import load_golden, cos_similarity

CACGMM_CASES = [
    'cacgmm_d4k2', 'cacgmm_d8k3', 'cacgmm_d8k3_structured',
    'cacgmm_opt_saliency', 'cacgmm_opt_mask', 'cacgmm_opt_trace',
    'cacgmm_opt_nonorm', 'cacgmm_opt_w2', 'cacgmm_opt_eps0',
    'cacgmm_opt_bcast',
]


def _kwargs(g):
    kw = {}
    for k, v in g.items():
        if not k.startswith('kw_'):
            continue
        name = k[3:]
        if name == 'covariance_norm':
            v = str(v) if v.dtype.kind in 'US' else False
        elif name == 'weight_constant_axis':
            v = int(v)
        elif name in ('affiliation_eps', 'eigenvalue_floor'):
            v = float(v)
        kw[name] = v
    return kw


@pytest.mark.parametrize('name', CACGMM_CASES)
def test_cacgmm_fit_matches_reference(name):
    g = load_golden(name)
    kw = _kwargs(g)
    model = O.cacgmm_fit(g['y'], g['init'], int(g['iterations']), **kw)
    np.testing.assert_allclose(model['weight'], g['weight'], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(model['eigenvalues'], g['eigenvalues'], rtol=1e-7, atol=1e-13)
    cov = O.cacg_covariance_from_eig(model['eigenvectors'], model['eigenvalues'])
    np.testing.assert_allclose(cov, g['covariance'], rtol=1e-7, atol=1e-10)
    aff, q = O.cacgmm_predict(g['y'], model, True, kw.get('source_activity_mask'))
    np.testing.assert_allclose(aff, g['affiliation'], rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(q, g['quadratic_form'], rtol=1e-7)
    np.testing.assert_allclose(O.cacgmm_log_likelihood(g['y'], model),
                               g['log_likelihood'], rtol=1e-9)


@pytest.mark.parametrize('name,axis', [('cacgmm_tied_time', (-3,)), ('cacgmm_tied', (-3, -1))])
def test_cacgmm_frequency_tied_weights(name, axis):
    g = load_golden(name)
    m = O.cacgmm_fit(g['y'], g['init'], int(g['iterations']), weight_constant_axis=axis)
    assert m['weight'].shape == g['weight'].shape
    np.testing.assert_allclose(m['weight'], g['weight'], rtol=1e-9)
    np.testing.assert_allclose(O.cacg_covariance_from_eig(m['eigenvectors'], m['eigenvalues']), g['covariance'],
                               rtol=1e-7, atol=1e-10)


def test_cacgmm_inline_permutation_alignment():
    g = load_golden('cacgmm_inline_pa')
    m = O.cacgmm_fit(g['y'], g['init'], 5, weight_constant_axis=(-3,), inline_permutation_plan=g['plan'].tolist())
    np.testing.assert_allclose(m['weight'], g['weight'], rtol=1e-9)
    np.testing.assert_allclose(O.cacg_covariance_from_eig(m['eigenvectors'], m['eigenvalues']), g['covariance'],
                               rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(O.cacgmm_predict(g['y'], m), g['affiliation'], rtol=1e-7, atol=1e-10)


def test_cacgmm_warm_start():
    g = load_golden('cacgmm_warm')
    m3 = dict(weight=g['w3'], eigenvectors=g['V3'], eigenvalues=g['l3'])
    m5 = O.cacgmm_fit(g['y'], m3, 2)
    np.testing.assert_allclose(m5['weight'], g['w5'], rtol=1e-9)
    np.testing.assert_allclose(m5['eigenvalues'], g['l5'], rtol=1e-7, atol=1e-13)
    cov = O.cacg_covariance_from_eig(m5['eigenvectors'], m5['eigenvalues'])
    np.testing.assert_allclose(cov, g['cov5'], rtol=1e-7, atol=1e-10)


def test_cacg_single_steps():
    g = load_golden('cacg_steps')
    z = O.normalize_observation_cacg(g['y'])
    np.testing.assert_allclose(z, g['z'], rtol=1e-14)
    V, lam = O.cacg_from_covariance(g['cov'].copy(), 1e-10)
    np.testing.assert_allclose(lam, g['lam'], rtol=1e-10)
    log_pdf, q = O.cacg_log_pdf(z[..., None, :, :], g['V'], g['lam'])
    np.testing.assert_allclose(log_pdf, g['log_pdf'], rtol=1e-11)
    np.testing.assert_allclose(q, g['q'], rtol=1e-11)
    aff = O.log_pdf_to_affiliation(g['w'], g['log_pdf'], None, 1e-10)
    np.testing.assert_allclose(aff, g['aff'], rtol=1e-12)
    cov = O.cacg_covariance(z[..., None, :, :], g['aff'], g['q'])
    V2, lam2 = O.cacg_from_covariance(cov, 1e-10)
    np.testing.assert_allclose(lam2, g['fit_lam'], rtol=1e-9)
    np.testing.assert_allclose(O.cacg_covariance_from_eig(V2, lam2),
                               g['fit_cov'], rtol=1e-9, atol=1e-12)


def test_reference_doctest_known_answers():
    # complex_angular_central_gaussian.py:278-289 (_fit doctest)
    y = np.array([[1, 0, 0], [1, 0, 0], [0, 1, 0], [0, 1, 0]],
                 dtype=np.complex128).T
    q = np.array([[1, 0], [1, 0], [1, 0], [1, 0]], dtype=np.float64).T
    cov = O.cacg_covariance(y, np.ones_like(q), q)
    _, lam = O.cacg_from_covariance(cov, 1e-10)
    np.testing.assert_allclose(lam, [[1e-10, 1, 1], [1e-10, 1, 1]])
    # mixture_model_utils.py:157-175 (estimate_mixture_weight doctest)
    a = np.array([[0.4, 1, 0.4], [0.6, 0, 0.6]])
    np.testing.assert_allclose(O.estimate_mixture_weight(a), [[0.6], [0.4]])
    np.testing.assert_allclose(O.estimate_mixture_weight(a, weight_constant_axis=-2), [[0.5], [0.5]])
    np.testing.assert_allclose(
        O.estimate_mixture_weight(np.array([a, a]), weight_constant_axis=-3),
        [[[0.4, 1., 0.4], [0.6, 0., 0.6]]])
    # distribution/utils.py:232-244 (_unit_norm 'where')
    s = np.array([[1, 1], [1e-20, 1e-20], [0, 0]], dtype=np.complex128)
    z = O.normalize_observation_cacg(s)
    np.testing.assert_allclose(z.T, [[0.70710678, 0.70710678],
                                     [0.70710678, 0.70710678], [0, 0]], atol=1e-8)
    # pb_bss/utils.py:114-124 (get_pca)
    vec, val = O.principal_component(np.array([[2., 0], [0, 1]]))
    np.testing.assert_allclose(np.abs(vec), [1, 0]); assert val == 2
    # complex_watson.py:268-271 (hypergeometric_ratio_inverse doctest)
    sp = O.cw_spline(5)
    np.testing.assert_allclose(
        sp([0, 1 / 5, 1 / 5 + 1e-4, 0.9599999, 1]),
        [0, 0, 3.74879525e-03, 9.99997522e+01, 5e+02], rtol=1e-7)
    # permutation_alignment.py:475-508 (greedy assignment doctest)
    sm = np.array([[11, 10, 0], [4, 5, 10], [6, 0, 5]])
    np.testing.assert_array_equal(O.greedy_mapping_from_score_matrix(sm), [0, 2, 1])
    # permutation_alignment.py:223-232 (alignment_plan doctest, stft 512)
    assert O.dhtv_plan_from_stft_size(512) == [
        [20, 70, 170], [2, 90, 190], [2, 50, 150], [2, 110, 210],
        [2, 30, 130], [2, 130, 230], [2, 0, 110], [2, 150, 257]]
    assert O.dhtv_alignment_plan(512, 0, 257, 20, 20, 2) == [[20, 0, 257]]


@pytest.mark.parametrize('name', ['cwmm_d6k4', 'cwmm_d4k2'])
def test_cwmm_fit_matches_reference(name):
    g = load_golden(name)
    model = O.cwmm_fit(g['y'], g['init'], int(g['iterations']))
    np.testing.assert_allclose(model['weight'], g['weight'], rtol=1e-8)
    np.testing.assert_allclose(model['concentration'], g['concentration'], rtol=1e-7)
    np.testing.assert_allclose(cos_similarity(model['mode'], g['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(O.cwmm_predict(g['y'], model), g['affiliation'],
                               rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('name,axis', [('cwmm_tied_time', (-3,)), ('cwmm_tied', (-3, -1)), ('cwmm_inline_pa', (-3,))])
def test_cwmm_coupled_fit_matches_reference(name, axis):
    # frequency-tied weights / inline permutation alignment, cwmm.py:152-184
    g = load_golden(name)
    plan = g['plan'].tolist() if 'plan' in g else None
    model = O.cwmm_fit(g['y'], g['init'], int(g['iterations']), weight_constant_axis=axis,
                       inline_permutation_plan=plan)
    assert model['weight'].shape == g['weight'].shape
    np.testing.assert_allclose(model['weight'], g['weight'], rtol=1e-9)
    np.testing.assert_allclose(model['concentration'], g['concentration'], rtol=1e-7)
    np.testing.assert_allclose(cos_similarity(model['mode'], g['mode']), 1, atol=1e-9)
    np.testing.assert_allclose(O.cwmm_predict(g['y'], model), g['affiliation'], rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('D', [4, 6, 8])
def test_cw_spline_and_log_norm(D):
    g = load_golden(f'cw_spline_d{D}')
    np.testing.assert_allclose(O.cw_spline(D)(g['lam']), g['kappa'], rtol=1e-12)
    np.testing.assert_allclose(O.cw_log_norm(g['kappa_grid'], D), g['log_norm'], rtol=1e-13)


def test_permutation_alignment():
    g = load_golden('permutation')
    for tag in 'ab':
        plan = g[f'{tag}_plan'].tolist()
        stft = {257: 512, 513: 1024}[g[f'{tag}_mask'].shape[1]]
        assert O.dhtv_plan_from_stft_size(stft) == plan
        mapping = O.dhtv_calculate_mapping(g[f'{tag}_mask'], plan)
        np.testing.assert_array_equal(mapping, g[f'{tag}_mapping'])
        np.testing.assert_array_equal(O.apply_mapping(g[f'{tag}_mask'], mapping),
                                      g[f'{tag}_aligned'])
    plan = O.dhtv_alignment_plan(128, 20, 20, 5, 5, 2)
    assert plan == g['c_plan'].tolist()
    np.testing.assert_array_equal(O.dhtv_calculate_mapping(g['c_mask'], plan), g['c_mapping'])
    np.testing.assert_array_equal(O.greedy_mapping_from_score_matrix(g['score']), g['score_greedy'])


def test_beamformer_chain():
    g = load_golden('beamformer')
    Y, mask = g['Y'], g['mask']
    np.testing.assert_allclose(O.power_spectral_density(Y, mask), g['psd'], rtol=1e-12)
    np.testing.assert_allclose(O.power_spectral_density(Y, mask, False), g['psd_nonorm'], rtol=1e-12)
    np.testing.assert_allclose(O.power_spectral_density(Y, mask[:, 0]), g['psd_single'], rtol=1e-12)
    np.testing.assert_allclose(O.power_spectral_density(Y), g['psd_nomask'], rtol=1e-12)
    pca = O.pca_vector(g['target'])
    np.testing.assert_allclose(cos_similarity(pca, g['pca']), 1, atol=1e-12)
    np.testing.assert_allclose(O.mvdr_vector(g['pca'], g['noise']), g['mvdr'], rtol=1e-10)
    np.testing.assert_allclose(O.gev_vector(g['target'], g['noise']), g['gev'], rtol=1e-12)
    s, ch = O.mvdr_vector_souden(g['target'], g['noise'])
    assert ch == int(g['ref_channel'])
    np.testing.assert_allclose(s, g['souden'], rtol=1e-10)
    np.testing.assert_allclose(O.blind_analytic_normalization(g['gev'], g['noise']), g['ban'], rtol=1e-12)
    np.testing.assert_allclose(O.apply_beamforming_vector(g['gev'], Y), g['applied'], rtol=1e-12)
    # Souden golden vector of the reference's own unit test
    # (tests/test_extraction/test_beamformer.py:205-209)
    obs = np.array([[0, 0, 1], [0, 0.1, 1], [0.1, 0, 1]])
    w, _ = O.mvdr_vector_souden((obs.T.conj() @ obs)[None], np.eye(3)[None])
    np.testing.assert_allclose(w[0], [0.03311258, 0.03311258, 0.99337748], atol=1e-8)


METRICS = ('cos', 'euclidean', 'multiply')


@pytest.mark.parametrize('metric', METRICS)
def test_greedy_and_oracle_permutation_alignment(metric):
    # GreedyPermutationAlignment / OraclePermutationAlignment, permutation_alignment.py:592-786
    g = load_golden('permutation_greedy_oracle')
    np.testing.assert_allclose(O.score_matrix(g['noise'], g['noise_reference'], metric), g[f'scores_{metric}'],
                               rtol=1e-13, atol=1e-15)
    for tag, mask, ref in (('', g['mask'], g['reference_mask']), ('noise_', g['noise'], g['noise_reference'])):
        np.testing.assert_array_equal(O.greedy_permutation_alignment(mask, metric), g[f'greedy_{tag}{metric}'])
        for alg in ('greedy', 'optimal'):
            np.testing.assert_array_equal(O.oracle_permutation_alignment(mask, ref, metric, alg),
                                          g[f'oracle_{tag}{metric}_{alg}'])


@pytest.mark.parametrize('metric', ['cos', 'multiply', 'euclidean'])
@pytest.mark.parametrize('algorithm', ['greedy', 'optimal'])
def test_dhtv_options(metric, algorithm):
    # DHTVPermutationAlignment's similarity_metric / algorithm (permutation_alignment.py:133-163,295-355), K = 3
    g = load_golden('permutation')
    mapping, margin = O.dhtv_calculate_mapping(g['a_mask'], O.dhtv_plan_from_stft_size(512), metric, algorithm,
                                               return_margin=True)
    np.testing.assert_array_equal(mapping, g[f'opt_{metric}_{algorithm}'])
    assert margin > MARGIN


# smallest decision margin (relative to the largest |score| of the bin) for which the device kernels must reproduce
# the reference's integer mapping: the kernels sum in other orders, so closer decisions may legitimately differ
MARGIN = 1e-9
CLASS_CASES = ('k2', 'k3', 'k4', 'k5', 'k6', 'k7', 'k8', 'k9', 'k8s', 'k9s', 'plan_edge',
               'tie_const_k3', 'tie_const_k9', 'tie_pair_k3', 'tie_pair_k9', 'tie_zero_k3', 'tie_zero_k9')


def test_permutation_classes_inputs_are_the_generators():
    from oracle.make_golden import permutation_classes_cases
    g = load_golden('permutation_classes')
    assert sorted(g['dhtv_cases'].tolist()) == sorted(CLASS_CASES)
    for name, (mask, plan) in permutation_classes_cases().items():
        np.testing.assert_array_equal(g[f'{name}_mask'], mask)
        assert g[f'{name}_plan'].tolist() == plan


@pytest.mark.parametrize('name', CLASS_CASES)
def test_dhtv_classes_and_ties(name):
    """DHTV alignment, K = 2..9, every metric and assignment the fixture holds.  Exact ties (tie_*) follow the first
    maximum in row-major order; every other decision is far from a tie, so any correct kernel reproduces it."""
    g = load_golden('permutation_classes')
    mask, plan = g[f'{name}_mask'], g[f'{name}_plan'].tolist()
    combos = [(m, a) for m in METRICS for a in ('greedy', 'optimal') if f'{name}_{m}_{a}' in g]
    keys = [f'{name}_{m}_{a}' for m, a in combos]
    assert len(keys) >= 2
    for key, (metric, algorithm) in zip(keys, combos):
        mapping, margin = O.dhtv_calculate_mapping(mask, plan, metric, algorithm, return_margin=True)
        np.testing.assert_array_equal(mapping, g[key], err_msg=key)
        if name.startswith('tie_'):
            assert margin == 0, key
        else:
            assert margin > MARGIN, (key, margin)
    if name.startswith('tie_const'):
        # every score ties: the first iteration keeps the identity and the reference stops there
        assert all((g[k] == np.arange(mask.shape[0])[:, None]).all() for k in keys)


@pytest.mark.parametrize('K', range(2, 10))
def test_greedy_and_oracle_alignment_classes(K):
    g = load_golden('permutation_classes')
    mask, perm = g[f'k{K}_mask'], g[f'k{K}_perm']
    reference = mask[np.argsort(perm, axis=0), np.arange(mask.shape[1])]
    for tag, m, ref in (('k', mask, reference), ('noise_k', g[f'noise_k{K}_mask'], g[f'noise_k{K}_reference'])):
        for metric in METRICS:
            got, margin = O.greedy_permutation_alignment(m, metric, return_margin=True)
            np.testing.assert_array_equal(got, g[f'{tag}{K}_greedy_{metric}'])
            assert margin > MARGIN
            for alg in ('greedy', 'optimal'):
                key = f'{tag}{K}_oracle_{metric}_{alg}'
                if key in g:
                    got, margin = O.oracle_permutation_alignment(m, ref, metric, alg, return_margin=True)
                    np.testing.assert_array_equal(got, g[key], err_msg=key)
                    assert margin > MARGIN, key
    # the Oracle alignment undoes the shuffle
    np.testing.assert_array_equal(O.apply_mapping(mask, g[f'k{K}_oracle_euclidean_greedy']), reference)


def test_assignment_margins_and_the_vectorised_brute_force():
    import itertools
    sm = np.array([[11, 10, 0], [4, 5, 10], [6, 0, 5]])  # permutation_alignment.py:475-508
    assert O.greedy_mapping_from_score_matrix(sm, return_margin=True)[1] == 1  # 11 over 10; then 10 over 5
    p, m = O.optimal_mapping_from_score_matrix(sm, return_margin=True)
    np.testing.assert_array_equal(p, [1, 2, 0])
    assert m == 5  # 26 over 21
    rng = np.random.RandomState(3)
    for K in (1, 2, 3, 4, 5, 6):
        for _ in range(20):
            score = rng.randint(0, 3, size=(K, K)).astype(np.float64)  # many exact ties
            if rng.rand() < 0.5:
                score = rng.uniform(-1, 1, size=(K, K))
            best, best_perm = float('-inf'), None
            for perm in itertools.permutations(range(K)):  # the reference's loop
                s = sum(score[range(K), perm])
                if s > best:
                    best, best_perm = s, perm
            np.testing.assert_array_equal(O.optimal_mapping_from_score_matrix(score), best_perm)
    assert O.greedy_mapping_from_score_matrix(np.zeros((4, 4)), return_margin=True)[1] == 0
    np.testing.assert_array_equal(O.greedy_mapping_from_score_matrix(np.zeros((4, 4))), np.arange(4))


def test_mapping_from_score_matrix_doctest():
    # permutation_alignment.py:475-508: 'optimal' and 'greedy' differ on this matrix
    g = load_golden('permutation_greedy_oracle')
    np.testing.assert_array_equal(O.greedy_mapping_from_score_matrix(g['score']), [0, 2, 1])
    np.testing.assert_array_equal(O.optimal_mapping_from_score_matrix(g['score']), [1, 2, 0])
    np.testing.assert_array_equal(g['score_greedy'], [0, 2, 1])
    np.testing.assert_array_equal(g['score_optimal'], [1, 2, 0])
    with pytest.raises(ValueError, match='infeasible'):
        O.mapping_from_score_matrix(np.array([[[np.inf, 0], [1, 2]]]), 'optimal')
