"""BinaryGMM / BinaryGMMTrainer on the device (pbb_kmeans_fit / pbb_kmeans_predict) against the reference's outputs
in tests/golden/kmeans.npz and against the NumPy restatement (oracle/kmeans_oracle.py)."""
import warnings

import numpy as np
import pytest

from oracle import kmeans_oracle as KO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold(golden):
    return golden('kmeans')


def _trainer():
    from pb_bss_b200.distribution import BinaryGMMTrainer
    return BinaryGMMTrainer()


def _fit(x, K, saliency=None, init=None):
    from pb_bss_b200.distribution import BinaryGMM, gmm
    if init is None:
        return _trainer().fit(x, K, saliency=saliency)
    return BinaryGMM(kmeans=gmm._kmeans_fit(x, K, init=init))


def _check(km, want_labels, want_centres, want_inertia, want_n_iter, x, rtol=1e-12):
    np.testing.assert_array_equal(km.labels_, want_labels)
    assert km.labels_.dtype == np.int32
    assert km.n_iter_ == want_n_iter and isinstance(km.n_iter_, int)
    assert km.cluster_centers_.dtype == np.float64
    np.testing.assert_allclose(km.cluster_centers_, want_centres, rtol=rtol, atol=rtol * np.abs(want_centres).max())
    assert isinstance(km.inertia_, float)
    np.testing.assert_allclose(km.inertia_, want_inertia, rtol=rtol, atol=rtol * KO.inertia_scale(x))


@pytest.mark.parametrize('name', list(KO.CASES))
def test_fixtures(gold, name):
    seed, N, E, K, _ = KO.CASES[name]
    x, saliency, held, init = KO.case_input(name)
    np.random.seed(seed)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        model = _fit(x, K, saliency, init)
    after = np.random.get_state()
    # the duplicates case: sklearn leaves the empty cluster in place when every point sits on its centre
    assert any('Number of distinct clusters' in str(c.message) for c in caught) == bool(gold[f'{name}_warned'])
    rtol = 1e-5 if x.dtype == np.float32 else 1e-12   # sklearn computes float32 input in float32
    _check(model.kmeans, gold[f'{name}_labels'], gold[f'{name}_centres'], gold[f'{name}_inertia'],
           gold[f'{name}_n_iter'], x if saliency is None else x[saliency], rtol)
    if init is None:   # the RNG state after the fit is the reference's
        np.testing.assert_array_equal(after[1], gold[f'{name}_state_keys'])
        assert after[2] == gold[f'{name}_state_pos'] and after[3] == gold[f'{name}_state_has_gauss']
        assert after[4] == gold[f'{name}_state_gauss']
    aff = model.predict(held)
    assert aff.dtype == held.dtype and aff.shape == (K, held.shape[0])
    np.testing.assert_array_equal(aff, gold[f'{name}_predict'].astype(held.dtype))


SHAPES = [(1, 3, 1), (2, 1, 2), (5, 2, 5), (16, 64, 16), (129, 3, 4), (1000, 64, 16), (4097, 7, 11), (33333, 17, 9),
          (70000, 2, 13), (100000, 40, 4), (2 ** 20, 8, 5)] + [(3000, 10, k) for k in (1, 2, 3, 6, 7, 8, 10, 12, 14, 15,
                                                                                       16)]


def _safe_case(N, E, K):
    """Seeded blobs (and their fit seed) whose oracle fit has no decision within 1e-9 of its boundary."""
    for seed in range(20):
        x = KO.blobs(1000 + seed + N + E + K, N, E, K, 3.0)
        np.random.seed(seed)
        want = KO.fit(x, K)
        if want['margin'] > 1e-9:
            return x, seed, want
    pytest.fail('no seeded case clear of rounding')


@pytest.mark.parametrize('N,E,K', SHAPES)
def test_against_the_oracle(N, E, K):
    x, seed, want = _safe_case(N, E, K)
    np.random.seed(seed)
    model = _fit(x, K)
    _check(model.kmeans, want['labels'], want['centres'], want['inertia'], want['n_iter'], x)
    held = x[:: max(1, N // 500)] + 0.25
    np.testing.assert_array_equal(model.kmeans.predict(held), KO.predict(held, model.kmeans.cluster_centers_))
    np.testing.assert_array_equal(model.predict(held),
                                  KO.one_hot(KO.predict(held, model.kmeans.cluster_centers_), K, np.float64))


def test_cuda_in_cuda_out_and_bitwise_repeatable():
    import torch
    x = KO.blobs(5, 50000, 20, 3, 4.0)
    np.random.seed(1)
    a = _fit(x, 3).kmeans
    np.random.seed(1)
    b = _fit(x, 3).kmeans
    np.random.seed(1)
    c = _fit(torch.from_numpy(x).cuda(), 3)
    km = c.kmeans
    assert km.labels_.device.type == 'cuda' and km.labels_.dtype == torch.int32
    assert km.cluster_centers_.device.type == 'cuda' and km.inertia_.device.type == 'cuda'
    for u, v in ((a, b), (a, km)):
        np.testing.assert_array_equal(u.labels_, np.asarray(torch.as_tensor(v.labels_).cpu()))
        np.testing.assert_array_equal(u.cluster_centers_, np.asarray(torch.as_tensor(v.cluster_centers_).cpu()))
        assert u.inertia_ == float(v.inertia_) and u.n_iter_ == int(v.n_iter_)
    xt = torch.from_numpy(x[:100]).cuda()
    aff = c.predict(xt)
    assert aff.device.type == 'cuda' and aff.dtype == torch.float64
    np.testing.assert_array_equal(aff.cpu().numpy(), _fit_predict_numpy(a, x[:100]))
    lab = km.predict(xt)
    assert lab.device.type == 'cuda' and lab.dtype == torch.int32


def _fit_predict_numpy(km, x):
    from pb_bss_b200.distribution import BinaryGMM
    return BinaryGMM(kmeans=km).predict(x)


def test_cuda_fit_does_not_synchronise():
    import torch
    import pb_bss_b200
    x = torch.from_numpy(KO.blobs(6, 20000, 16, 4, 4.0)).cuda()
    np.random.seed(2)
    want = _fit(x, 4).kmeans
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    np.random.seed(2)
    torch.cuda.set_sync_debug_mode('error')
    try:
        with pb_bss_b200.deferred_status():
            got = _fit(x, 4).kmeans
            torch.cuda.set_sync_debug_mode(prev)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert torch.equal(got.labels_, want.labels_) and torch.equal(got.cluster_centers_, want.cluster_centers_)


def test_cuda_saliency_selects_rows():
    import torch
    x = KO.blobs(7, 9000, 6, 3, 5.0)
    sal = np.random.default_rng(0).random(9000) < 0.5
    np.random.seed(4)
    a = _fit(x, 3, sal).kmeans
    np.random.seed(4)
    b = _fit(torch.from_numpy(x).cuda(), 3, torch.from_numpy(sal).cuda()).kmeans
    np.testing.assert_array_equal(a.labels_, b.labels_.cpu().numpy())
    assert a.labels_.shape == (sal.sum(),)


@pytest.mark.parametrize('case', ['blobs', 'relocation', 'duplicates'])
def test_results_do_not_depend_on_the_grid(case):
    """One CTA working every chunk, a few CTAs, and the device's full grid give the same bits."""
    from pb_bss_b200.distribution import gmm
    if case == 'blobs':
        x, K, init = KO.blobs(21, 100000, 12, 6, 1.0), 6, None
    else:
        x, _, _, init = KO.case_input(case)
        K = KO.CASES[case][3]
    fits = []
    for max_ctas in (0, 1, 3, 37):
        np.random.seed(5)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            fits.append(gmm._kmeans_fit(x, K, init=init, max_ctas=max_ctas))
    for km in fits[1:]:
        np.testing.assert_array_equal(km.labels_, fits[0].labels_)
        np.testing.assert_array_equal(km.cluster_centers_, fits[0].cluster_centers_)
        assert km.inertia_ == fits[0].inertia_ and km.n_iter_ == fits[0].n_iter_


def test_two_empty_clusters_take_tied_points_in_index_order():
    """Two points at the same distance from their old centre, held by different warps of one CTA (index 40 by
    warp 1, index 128 by warp 0): the lower index fills the first empty cluster, as in the oracle."""
    from pb_bss_b200.distribution import gmm
    x = np.zeros((40000, 1))
    x[40, 0], x[128, 0] = 50.0, -50.0
    init = np.array([[0.0], [1e4], [2e4]])
    km = gmm._kmeans_fit(x, 3, init=init)
    want = KO.fit(x, 3, init=init)
    np.testing.assert_array_equal(km.cluster_centers_[1:, 0], [50.0, -50.0])
    np.testing.assert_array_equal(km.labels_, want['labels'])
    np.testing.assert_allclose(km.cluster_centers_, want['centres'], rtol=0, atol=1e-12)


def test_fewer_distinct_points_than_clusters_warns():
    from pb_bss_b200.distribution.gmm import ConvergenceWarning
    x = np.repeat(np.array([[0.0, 1.0], [5.0, 5.0], [9.0, -3.0]]), 40, axis=0)
    np.random.seed(0)
    with pytest.warns(ConvergenceWarning, match=r'Number of distinct clusters \(3\) found smaller than n_clusters \(4\)'):
        km = _fit(x, 4).kmeans
    assert len(set(km.labels_.tolist())) == 3


@pytest.mark.parametrize('x,K,match', [
    (np.zeros(10), 2, '2D'),
    (np.zeros((2, 5, 3)), 2, '2D'),
    (np.zeros((10, 3), complex), 2, 'Complex'),
    (np.zeros((3, 3)), 4, 'n_samples=3 should be >= n_clusters=4'),
    (np.zeros((30, 65)), 2, 'E=65 > 64'),
    (np.zeros((30, 3)), 17, '1 <= K <= 16'),
    (np.zeros((30, 3)), 0, '1 <= K <= 16'),
])
def test_errors(x, K, match):
    with pytest.raises(ValueError, match=match):
        _trainer().fit(x, K)


def test_non_finite_input_raises():
    for bad in (np.nan, np.inf):
        x = KO.blobs(8, 500, 4, 2, 3.0)
        x[17, 2] = bad
        with pytest.raises(ValueError, match='NaN or infinity'):
            _trainer().fit(x, 2)


def test_saliency_must_be_a_boolean_vector():
    x = KO.blobs(9, 100, 4, 2, 3.0)
    with pytest.raises(AssertionError, match='Only boolean saliency supported. Current dtype: float64.'):
        _trainer().fit(x, 2, saliency=np.ones(100))
    with pytest.raises(AssertionError):
        _trainer().fit(x, 2, saliency=np.ones(99, bool))
    with pytest.raises(AssertionError):
        _fit_predict_numpy(_trainer().fit(x, 2).kmeans, x.astype(complex))
