"""NumPy restatement of the k-means behind BinaryGMMTrainer (pb_bss/distribution/gmm.py:201-230), which calls
sklearn's ``KMeans(n_clusters=K).fit`` with its defaults: one k-means++ seeding, then Lloyd iterations.

The steps, as the device computes them (csrc/kmeans.cuh), all in float64:
  - tol = 1e-4 * mean over the columns of var(x); the data are centred on their column mean, which is added back
    to the centres at the end;
  - k-means++ with L = 2 + int(log K) trials per round.  The random draws come from NumPy's global RandomState
    (``draws``): the first centre's index from ``choice(N, p=w / w.sum())`` with w = ones in sklearn's dtype for x,
    then one ``uniform(size=L)`` per further centre.  Squared distances are (-2 a.x + |a|^2) + |x|^2, clipped at 0.
    A round scales the uniforms by the current potential, finds each target in the running sum of the closest
    distances (searchsorted, left, clipped to N - 1), and keeps the first candidate of least potential;
  - Lloyd, at most 300 passes: the label of a point is the first argmin of |c|^2 - 2 x.c.  A cluster left empty
    takes the point farthest from its old centre (largest first, ties to the lower index), which leaves its old
    cluster's sum but keeps its label; when that largest distance is 0 no point moves, as in sklearn.  Centres are the sums times 1 / weight; a still empty cluster copies the
    heaviest cluster's row as it stands at that moment.  The loop stops when no label changed, or when the summed
    squared centre shift is <= tol; in the second case the labels are computed once more.  The inertia is the sum of
    the squared distances to the assigned centres.

``fit`` also returns ``margin``: the smallest relative distance of any decision (an argmin, a searchsorted position
or the tolerance test) from its boundary, so that fixtures can avoid cases decided by rounding.
"""
import numpy as np

MAX_ITER = 300


def trials(K):
    return 2 + int(np.log(K))


def draws(N, K, sklearn_dtype=np.float64):
    """The first centre's index and the (K - 1, L) uniforms, from the global RandomState in sklearn's order."""
    w = np.ones(N, dtype=sklearn_dtype)
    first = int(np.random.choice(N, p=w / w.sum()))
    u = np.array([np.random.uniform(size=trials(K)) for _ in range(K - 1)]).reshape(K - 1, trials(K))
    return first, u


def _sq_dist(a, an, X, xn):
    return np.maximum((-2.0 * (X @ a) + an) + xn, 0.0)


def _gap(values, scale):
    """Relative gap between the least value and the next one that is not equal to it."""
    v = np.sort(values)
    rest = v[v > v[0]]
    return np.inf if rest.size == 0 else (rest[0] - v[0]) / scale


def _assign(xc, xn, centres, track):
    cn = np.einsum('ke,ke->k', centres, centres)
    d = cn[None, :] - 2.0 * (xc @ centres.T)
    labels = np.argmin(d, axis=1)
    if track is not None and centres.shape[0] > 1:
        uniq = np.unique(centres, axis=0, return_index=True)[1]
        du = np.sort(d[:, np.sort(uniq)], axis=1)
        if du.shape[1] > 1:
            scale = xn + cn.max()
            track.append(float(np.min((du[:, 1] - du[:, 0]) / np.maximum(scale, 1e-300))))
    return labels


def plusplus(xc, xn, K, first, u, track=None):
    N = xc.shape[0]
    centres = [xc[first]]
    closest = _sq_dist(xc[first], xn[first], xc, xn)
    pot = closest.sum()
    for r in range(1, K):
        targets = u[r - 1] * pot
        cum = np.cumsum(closest)
        cand = np.minimum(np.searchsorted(cum, targets), N - 1)
        if track is not None and pot > 0:
            track.append(float(np.min(np.abs(cum[None, :] - targets[:, None])) / pot))
        dist = np.minimum(closest[None, :], np.stack([_sq_dist(xc[c], xn[c], xc, xn) for c in cand]))
        pots = dist.sum(axis=1)
        best = int(np.argmin(pots))
        if track is not None:
            distinct = np.unique(cand, return_index=True)[1]
            track.append(_gap(pots[distinct], max(pot, 1e-300)))
        pot = pots[best]
        closest = dist[best]
        centres.append(xc[cand[best]])
    return np.array(centres)


def lloyd(xc, xn, centres, tol, max_iter=MAX_ITER, track=None):
    N, E = xc.shape
    K = centres.shape[0]
    labels = np.full(N, -1)
    strict = False
    for i in range(max_iter):
        previous = labels
        labels = _assign(xc, xn, centres, track)
        sums = np.zeros((K, E))
        np.add.at(sums, labels, xc)
        weight = np.bincount(labels, minlength=K).astype(np.float64)
        empty = np.flatnonzero(weight == 0)
        if empty.size:
            dist = ((xc - centres[labels]) ** 2).sum(axis=1)
            if dist.max() > 0:
                far = np.lexsort((np.arange(N), -dist))[:empty.size]
                for new, f in zip(empty, far):
                    sums[labels[f]] -= xc[f]
                    sums[new] = xc[f]
                    weight[new] = 1.0
                    weight[labels[f]] -= 1.0
        heaviest = int(np.argmax(weight))
        for k in range(K):
            if weight[k] > 0:
                sums[k] *= 1.0 / weight[k]
            else:
                sums[k] = sums[heaviest]
        shift = (np.sqrt(((sums - centres) ** 2).sum(axis=1)) ** 2).sum()
        centres = sums
        if np.array_equal(labels, previous):
            strict = True
            break
        if track is not None and tol > 0:
            track.append(abs(shift - tol) / tol)
        if shift <= tol:
            break
    if not strict:
        labels = _assign(xc, xn, centres, track)
    inertia = ((xc - centres[labels]) ** 2).sum()
    return labels, centres, inertia, i + 1, strict


def fit(x, K, init=None, max_iter=MAX_ITER):
    """KMeans(n_clusters=K).fit(x) (draws from the global RandomState), or with explicit initial centres init (K, E)
    as KMeans(n_clusters=K, init=init, n_init=1).fit(x) (no draws)."""
    x = np.asarray(x)
    X = x.astype(np.float64)
    N, E = X.shape
    tol = np.mean(np.var(X, axis=0)) * 1e-4
    mean = X.mean(axis=0)
    xc = X - mean
    xn = np.einsum('ij,ij->i', xc, xc)
    track = []
    if init is None:
        first, u = draws(N, K, np.float32 if x.dtype == np.float32 else np.float64)
        centres = plusplus(xc, xn, K, first, u, track)
    else:
        centres = np.asarray(init, dtype=np.float64) - mean
    labels, centres, inertia, n_iter, strict = lloyd(xc, xn, centres, tol, max_iter, track)
    return dict(centres=centres + mean, labels=labels.astype(np.int32), inertia=float(inertia), n_iter=n_iter,
                strict=strict, margin=min(track) if track else np.inf)


def predict(x, centres):
    """KMeans.predict on raw x: the first argmin of |c|^2 - 2 x.c."""
    X = np.asarray(x, dtype=np.float64)
    cn = np.einsum('ke,ke->k', centres, centres)
    return np.argmin(cn[None, :] - 2.0 * (X @ centres.T), axis=1).astype(np.int32)


def inertia_scale(x):
    """The inertia of one cluster at the mean: the absolute scale of the rounding in an inertia (an inertia that is
    0 in exact arithmetic comes out as rounding noise of this size)."""
    X = np.asarray(x, dtype=np.float64)
    return float(((X - X.mean(axis=0)) ** 2).sum())


def one_hot(labels, K, dtype):
    out = np.zeros((K, labels.size), dtype=dtype)
    out[labels, np.arange(labels.size)] = 1
    return out


# ---- the fixture cases: inputs are regenerated from their seeds, only outputs are stored ------------------------
def blobs(seed, N, E, K, spread, noise=1.0):
    rng = np.random.default_rng(seed)
    centres = rng.normal(0.0, spread, (K, E))
    return centres[rng.integers(0, K, N)] + rng.normal(0.0, noise, (N, E))


# name: (seed, N, E, K, spread of the blob centres)
CASES = {
    'separated': (0, 256500, 20, 3, 10.0),
    'overlapping': (1, 256500, 40, 4, 0.3),
    'long': (2, 20000, 8, 6, 0.0),
    'k1': (3, 3000, 5, 1, 5.0),
    'k2': (4, 5000, 12, 2, 2.0),
    'k16': (5, 40000, 24, 16, 3.0),
    'e1': (6, 10000, 1, 3, 4.0),
    'e64': (7, 30000, 64, 5, 1.5),
    'saliency': (8, 30000, 20, 3, 10.0),
    'float32': (9, 20000, 20, 3, 10.0),
    'int16': (10, 20000, 20, 3, 10.0),
    'relocation': (12, 5000, 4, 3, 5.0),
    'duplicates': (13, 512, 3, 5, 5.0),
}
HELD_OUT = 1000


def case_input(name):
    """(x to fit, saliency or None, held-out x for predict, init or None) of a fixture case."""
    seed, N, E, K, spread = CASES[name]
    if name == 'long':
        x = np.random.default_rng(seed).uniform(-1.0, 1.0, (N + HELD_OUT, E))
    elif name == 'duplicates':
        # K - 1 = 4 distinct integer points a, -a, b, -b, N / 4 = 128 times each: the mean is 0, every sum and average
        # is exact, so each point lies exactly on its centre and the empty cluster's largest distance is exactly 0
        rng = np.random.default_rng(seed)
        a, b = rng.integers(-int(spread), int(spread) + 1, (2, E)).astype(np.float64)
        pts = np.stack([a, -a, b, -b])
        x = np.concatenate([pts[rng.permutation(np.repeat(np.arange(4), N // 4))], pts[np.arange(HELD_OUT) % 4]])
    else:
        x = blobs(seed, N + HELD_OUT, E, max(K, 2) if name != 'relocation' else 2, spread)
    x, held = x[:N], x[N:]
    saliency = init = None
    if name == 'saliency':
        saliency = np.random.default_rng(seed + 100).random(N) < 0.6
    if name == 'float32':
        x, held = x.astype(np.float32), held.astype(np.float32)
    if name == 'int16':
        x, held = np.round(x * 100).astype(np.int16), np.round(held * 100).astype(np.int16)
    if name == 'relocation':
        # two blobs; the third initial centre lies far from every point, so its cluster is empty at first
        init = np.stack([x[0], x[1], np.full(E, 1e3)])
    return x, saliency, held, init
