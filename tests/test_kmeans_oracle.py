"""The NumPy restatement of BinaryGMMTrainer's k-means (oracle/kmeans_oracle.py) against the reference's outputs in
tests/golden/kmeans.npz: labels and n_iter exact, centres and inertia to 1e-12 (of the data's scale near 0), and the global RandomState left as
the reference leaves it."""
import numpy as np
import pytest

from oracle import kmeans_oracle as KO


@pytest.fixture(scope='module')
def gold(golden):
    return golden('kmeans')


def _state(gold, name):
    return ('MT19937', gold[f'{name}_state_keys'], int(gold[f'{name}_state_pos']),
            int(gold[f'{name}_state_has_gauss']), float(gold[f'{name}_state_gauss']))


def test_fixture_records_the_sklearn_version(gold):
    assert str(gold['sklearn_version']).count('.') >= 1


@pytest.mark.parametrize('name', list(KO.CASES))
def test_oracle_reproduces_the_reference(gold, name):
    seed, N, E, K, _ = KO.CASES[name]
    x, saliency, held, init = KO.case_input(name)
    fit_x = x if saliency is None else x[saliency]
    np.random.seed(seed)
    got = KO.fit(fit_x, K, init=init)
    after = np.random.get_state()
    np.testing.assert_array_equal(got['labels'], gold[f'{name}_labels'])
    assert got['n_iter'] == gold[f'{name}_n_iter']
    # sklearn computes float32 input in float32
    rtol = 1e-5 if x.dtype == np.float32 else 1e-12
    np.testing.assert_allclose(got['centres'], gold[f'{name}_centres'], rtol=rtol,
                               atol=rtol * np.abs(gold[f'{name}_centres']).max())
    np.testing.assert_allclose(got['inertia'], gold[f'{name}_inertia'], rtol=rtol, atol=rtol * KO.inertia_scale(fit_x))
    if init is None:
        want = _state(gold, name)
        assert after[0] == want[0] and after[2:] == want[2:]
        np.testing.assert_array_equal(after[1], want[1])
    pred = KO.one_hot(KO.predict(held, got['centres']), K, np.uint8)
    np.testing.assert_array_equal(pred, gold[f'{name}_predict'])


def test_draws_depend_on_the_shape_only():
    np.random.seed(3)
    a = KO.draws(1000, 7)
    np.random.seed(3)
    b = KO.draws(1000, 7)
    assert a[0] == b[0] and a[1].shape == (6, 3)
    np.testing.assert_array_equal(a[1], b[1])


def test_two_empty_clusters_take_the_two_farthest_points():
    """Largest distance first; both relocated points keep their labels for this pass."""
    x = np.array([[0.0], [1.0], [2.0], [10.0], [11.0]])
    init = np.array([[5.0], [100.0], [200.0]])
    got = KO.fit(x, 3, init=init, max_iter=1)
    xc = x - x.mean(0)
    # pass 1: all points in cluster 0 (centre 5); farthest from it: 11 (6), then 10 and 0 (5), the lower index wins
    c0 = (xc[[1, 2, 3]].sum() / 3) + x.mean()
    np.testing.assert_allclose(np.sort(got['centres'][:, 0]), np.sort([c0, 11.0, 0.0]), rtol=1e-14)
