"""Generate tests/golden/kmeans.npz: the reference's BinaryGMMTrainer (sklearn's KMeans) on the cases of
oracle/kmeans_oracle.py.CASES.

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_kmeans [OUT_DIR]

The unmodified reference is imported through oracle/ref_shim.py (it needs scikit-learn).  Each case is fitted under
np.random.seed(seed) with ``BinaryGMMTrainer().fit(x, K, saliency)``; the relocation case, which needs explicit
initial centres, with ``KMeans(n_clusters=K, init=init, n_init=1).fit`` as the reference's model holds it.  The inputs
are regenerated from their seeds by ``kmeans_oracle.case_input``, so only outputs are stored, per case <name>_*:
labels (int8), centres, inertia, n_iter, the MT19937 state after the fit (keys, pos, has_gauss, gauss), the
reference's ``BinaryGMM.predict`` one-hot of the held-out points (uint8) and whether the fit warned of fewer distinct
clusters than K (the duplicates case, where sklearn leaves an empty cluster in place).  ``sklearn_version`` records the version.
The generator checks that the NumPy restatement reproduces every case and that no decision of it lies within 1e-9
(relative) of its boundary.
"""
import os
import sys
import warnings

import numpy as np

from . import kmeans_oracle as KO
from . import ref_shim
from .make_golden_transform import OUT

MIN_MARGIN = 1e-9


def main(out_dir=OUT):
    import sklearn
    from sklearn.cluster import KMeans
    ref = ref_shim.load()
    out = {'sklearn_version': np.array(sklearn.__version__)}
    for name, (seed, N, E, K, _) in KO.CASES.items():
        x, saliency, held, init = KO.case_input(name)
        np.random.seed(seed)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter('always')
            if init is None:
                model = ref.distribution.BinaryGMMTrainer().fit(x, K, saliency=saliency)
            else:
                model = ref.distribution.BinaryGMM(kmeans=KMeans(n_clusters=K, init=init, n_init=1).fit(x))
        state = np.random.get_state()
        warned = any('Number of distinct clusters' in str(c.message) for c in caught)
        if name == 'duplicates':
            # sklearn's guard: with every point on its centre no point is relocated, and the empty cluster takes the
            # heaviest cluster's centre in _average_centers
            assert warned, 'the duplicate-points case must leave a cluster empty'
            heaviest = np.argmax(np.bincount(model.kmeans.labels_, minlength=K))
            assert np.array_equal(model.kmeans.cluster_centers_[K - 1], model.kmeans.cluster_centers_[heaviest])
        km = model.kmeans
        fit_x = x if saliency is None else x[saliency]
        np.random.seed(seed)
        orc = KO.fit(fit_x, K, init=init)
        assert orc['margin'] > MIN_MARGIN, (name, orc['margin'])
        assert np.array_equal(orc['labels'], km.labels_), name
        assert orc['n_iter'] == km.n_iter_, (name, orc['n_iter'], km.n_iter_)
        rtol = 1e-5 if x.dtype == np.float32 else 1e-12
        np.testing.assert_allclose(orc['centres'], km.cluster_centers_, rtol=rtol, atol=rtol * np.abs(fit_x).max())
        irtol = 1e-5 if x.dtype == np.float32 else 1e-10
        np.testing.assert_allclose(orc['inertia'], km.inertia_, rtol=irtol, atol=irtol * KO.inertia_scale(fit_x))
        if init is None:
            assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), state)), name
        if name == 'overlapping':
            assert not orc['strict'], 'the overlapping case must stop on the tolerance'
        pred = model.predict(held)
        out[f'{name}_labels'] = km.labels_.astype(np.int8)
        out[f'{name}_centres'] = np.asarray(km.cluster_centers_, dtype=np.float64)
        out[f'{name}_inertia'] = np.float64(km.inertia_)
        out[f'{name}_n_iter'] = np.int64(km.n_iter_)
        out[f'{name}_state_keys'] = state[1]
        out[f'{name}_state_pos'] = np.int64(state[2])
        out[f'{name}_state_has_gauss'] = np.int64(state[3])
        out[f'{name}_state_gauss'] = np.float64(state[4])
        out[f'{name}_predict'] = pred.astype(np.uint8)
        out[f'{name}_warned'] = np.bool_(warned)
        print(f'{name}: N={fit_x.shape[0]} E={E} K={K} n_iter={km.n_iter_} strict={orc["strict"]} '
              f'margin={orc["margin"]:.2e}')
    path = os.path.join(out_dir, 'kmeans.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path} ({os.path.getsize(path)} bytes)')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
