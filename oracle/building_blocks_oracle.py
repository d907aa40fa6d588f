"""NumPy restatement of the building blocks of pb_bss.distribution.mixture_model_utils / utils, pb_bss.utils and
pb_bss.evaluation.sxr_module, and the seeded cases of tests/golden/building_blocks.npz
(oracle/make_golden_building_blocks.py).  Results are computed in float64 and rounded once to the output dtype, as
the device kernels do."""
import numpy as np

# ---- cases: (tag, K, lead, weight, mask, eps, dtype, special) -----------------------------------------------------
N_AFF = 37
STORE_MAX = 4000  # larger affiliation outputs are not stored in the fixture
AFF_CASES = []
for K in (1, 2, 3, 6, 7, 16, 64):
    for lead in ((), (5,), (2, 5)):
        AFF_CASES.append((f'aff_k{K}_l{len(lead)}', K, lead, 'k1', False, 0.0, 'float64', None))
for w in ('k1', 'fk1', '1n', 'fkn', 'scalar'):
    for mask in (False, True):
        for eps in (0.0, 1e-3):
            AFF_CASES.append((f'aff_w{w}_m{int(mask)}_e{int(eps > 0)}', 3, (5,), w, mask, eps, 'float64', None))
for K in (3, 7):
    AFF_CASES.append((f'aff_f32_k{K}', K, (5,), 'fk1', True, 0.0, 'float32', None))
AFF_CASES += [
    ('aff_neginf', 3, (5,), 'k1', False, 0.0, 'float64', 'neginf'),
    ('aff_masked_out', 3, (5,), 'k1', True, 0.0, 'float64', 'masked_out'),
    ('aff_pm700', 4, (5,), 'k1', False, 0.0, 'float64', 'pm700'),
    ('aff_transposed', 6, (5,), 'fk1', True, 1e-3, 'float64', 'transposed'),
    ('aff_transposed_k16', 16, (5,), 'fkn', False, 0.0, 'float64', 'transposed'),
]
AFF_ERRORS = [('aff_err_bcast', 'bcast'), ('aff_err_mask', 'mask_dtype')]

INT_CASES = [(f'int_k{K}', K) for K in range(1, 7)]

EMW_AXES = [('m1', -1), ('m2', -2), ('m3', -3), ('t3', (-3,)), ('t31', (-3, -1)), ('t1', (-1,)), ('l31', [-3, -1]),
            ('p1', 2)]
EMW_CASES = [(f'emw_{a}_s{int(s)}', ax, s) for a, ax in EMW_AXES for s in (False, True)]

UNIT_ORDS = [('none', None), ('1', 1), ('2', 2), ('inf', np.inf), ('ninf', -np.inf), ('0', 0), ('3', 3), ('half', 0.5)]
UNIT_CASES = [(f'un_{o}_{st}_{dt}', ordv, st, dt) for o, ordv in UNIT_ORDS for st in ('plus', 'max', 'where')
              for dt in ('complex128', 'float64')]
UNIT_CASES += [(f'un_{st}_f32', None, st, 'float32') for st in ('plus', 'max', 'where')]

ONE_HOT_CASES = [  # tag, labels, categories, axis, keepdims, dtype
    ('oh_a0', [0, 1], 4, 0, False, 'bool'),
    ('oh_am1', [0, 1], 4, -1, False, 'bool'),
    ('oh_2d_am1', [[0, 1], [0, 3]], 4, -1, False, 'bool'),
    ('oh_2d_a1', [[0, 1], [0, 3]], 4, 1, False, 'bool'),
    ('oh_2d_a0', [[0, 1], [0, 3]], 4, 0, False, 'bool'),
    ('oh_keep', [[0], [3], [2]], 4, 1, True, 'bool'),
    ('oh_int64', [[0, 1], [2, 3]], 4, 1, False, 'int64'),
    ('oh_f32', [[0, 1], [2, 3]], 4, -1, False, 'float32'),
    ('oh_neg', [[-1, -4], [2, -2]], 4, 0, False, 'bool'),
]
ONE_HOT_ERRORS = [('oh_err_range', [0, 4], 4, 0, False), ('oh_err_neg', [0, -5], 4, 0, False),
                  ('oh_err_keep', [[0, 1]], 4, 1, True)]


def rng(tag):
    return np.random.default_rng(abs(hash_tag(tag)) % (2 ** 32))


def hash_tag(tag):
    h = 0
    for c in tag.encode():
        h = (h * 131 + c) % (2 ** 61 - 1)
    return h


def aff_input(case):
    """-> (weight, log_pdf, mask or None, eps) of an affiliation case."""
    tag, K, lead, wk, mask, eps, dtype, special = case
    r = rng(tag)
    F = lead[-1] if lead else 1
    lp = r.normal(scale=5.0, size=lead + (K, N_AFF))
    if special == 'pm700':
        lp = np.where(r.random(lp.shape) < 0.5, -700.0, 700.0) + r.normal(size=lp.shape)
    if special == 'neginf':
        lp[..., :, 3] = -np.inf
    w = {'k1': lambda: r.random((K, 1)) + 0.1, 'fk1': lambda: r.random((F, K, 1)) + 0.1,
         '1n': lambda: r.random((1, N_AFF)) + 0.1, 'fkn': lambda: r.random((F, K, N_AFF)) + 0.1,
         'scalar': lambda: np.float64(0.7)}[wk]()
    m = None
    if mask:
        m = r.random(lead + (K, N_AFF)) < 0.7
        if special == 'masked_out':
            m[..., :, 5] = False
    lp = lp.astype(dtype)
    if special == 'transposed':  # the same values read through transposed views
        lp = np.ascontiguousarray(np.swapaxes(lp, -1, -2)).swapaxes(-1, -2)
        if m is not None:
            m = np.ascontiguousarray(np.swapaxes(m, -1, -2)).swapaxes(-1, -2)
        if np.ndim(w) == 3:
            w = np.ascontiguousarray(np.swapaxes(w, -1, -2)).swapaxes(-1, -2)
    return w, lp, m, eps


def aff_error_input(kind):
    r = rng(kind)
    lp = r.normal(size=(3, 11))
    if kind == 'bcast':
        return r.random((2, 3, 1)), lp, None
    return np.ones((3, 1)), lp, (r.random((3, 11)) < 0.5).astype(np.int64)


def int_input(K):
    r = rng(f'int{K}')
    F, T = 5, 23
    return r.random((F, 1, T)) + 0.1, r.normal(scale=3, size=(F, K, T)), r.normal(scale=3, size=(F, K, T))


def emw_input(saliency):
    r = rng(f'emw{int(saliency)}')
    aff = r.random((4, 3, 3, 41))
    aff /= aff.sum(-2, keepdims=True)
    sal = None
    if saliency:
        sal = (r.random((4, 3, 41)) < 0.6).astype(np.float64)
        sal[:, 1, :] = 0  # a bin whose masked sum is 0
    return aff, sal


def unit_input(dtype):
    r = rng('unit' + dtype)
    x = r.normal(size=(4, 6, 5))
    if dtype == 'complex128':
        x = x + 1j * r.normal(size=(4, 6, 5))
    x[0, 1] = 0
    x[0, 2] = 1e-20
    return x.astype(dtype)


def hermitian_input():
    r = rng('herm')
    return r.normal(size=(3, 4, 4)) + 1j * r.normal(size=(3, 4, 4))


def pca_input():
    r = rng('pca')
    a = r.normal(size=(2, 3, 4, 4)) + 1j * r.normal(size=(2, 3, 4, 4))
    return a @ np.conj(np.swapaxes(a, -1, -2))


def snr_input():
    r = rng('snr')
    return r.normal(size=(2, 3, 50)), r.normal(size=(2, 3, 50)) * 0.3


# ---- the restatement ------------------------------------------------------------------------------------------------

def log_pdf_to_affiliation(weight, log_pdf, mask=None, eps=0.0):
    lp = np.asarray(log_pdf, dtype=np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        a = np.exp(lp - np.amax(lp, axis=-2, keepdims=True)) * np.asarray(weight, dtype=np.float64)
        if mask is not None:
            a = a * mask
        a = a / np.maximum(a.sum(-2, keepdims=True), np.finfo(np.asarray(log_pdf).dtype).tiny)
    if eps != 0:
        a = np.clip(a, eps, 1 - eps)
    return a.astype(np.asarray(log_pdf).dtype)


def integration_affiliation(weight, a, b, eps=0.0):
    import itertools
    F, K, T = a.shape
    out = np.zeros((F, K, T))
    w = np.broadcast_to(weight, a.shape)
    for f in range(F):
        best, best_p = -np.inf, None
        for p in itertools.permutations(range(K)):
            lp = a[f, list(p)] + b[f]
            c = np.exp(lp - lp.max(0, keepdims=True))
            c /= np.maximum(c.sum(0, keepdims=True), np.finfo(np.float64).tiny)
            aux = np.sum(c * lp)
            if aux > best:
                best, best_p = aux, p
        out[f] = log_pdf_to_affiliation(w[f], a[f, list(best_p)] + b[f], None, eps)
    return out


def estimate_mixture_weight(aff, sal=None, axis=-1):
    aff = np.asarray(aff)
    if isinstance(axis, int) and axis % aff.ndim - aff.ndim == -2:
        K = aff.shape[-2]
        return np.full([K, 1], 1 / K)
    axis = tuple(axis) if isinstance(axis, list) else axis
    if sal is None:
        return np.mean(aff, axis=axis, keepdims=True)
    return unit_norm(np.sum(aff * sal[..., None, :], axis=axis, keepdims=True), axis=-2, eps=1e-10,
                     eps_style='where', ord=1)


def unit_norm(x, axis=-1, eps=1e-4, eps_style='plus', ord=None):
    dtype = np.asarray(x).dtype
    x64 = np.asarray(x).astype(np.complex128 if np.iscomplexobj(x) else np.float64)
    n = np.linalg.norm(x64, ord=ord, axis=axis, keepdims=True)
    if eps_style == 'plus':
        n = n + eps
    elif eps_style == 'max':
        n = np.maximum(n, eps)
    elif eps_style == 'where':
        n = np.where(n == 0, eps, n)
    else:
        raise AssertionError(eps_style)
    return (x64 / n).astype(dtype)


def force_hermitian(a):
    return (a + np.swapaxes(a.conj(), -1, -2)) / 2


def labels_to_one_hot(labels, categories, axis=0, keepdims=False, dtype=bool):
    labels = np.asarray(labels)
    if keepdims:
        assert labels.shape[axis] == 1
        labels = np.squeeze(labels, axis)
    ax = axis % (labels.ndim + 1)
    c = np.arange(categories).reshape((categories,) + (1,) * labels.ndim)
    if labels.size and not (labels.min() >= -categories and labels.max() < categories):
        raise IndexError('label out of range')
    return np.moveaxis(c == labels % categories, 0, ax).astype(dtype)


def abs_square(x):
    return x.real ** 2 + x.imag ** 2 if np.iscomplexobj(x) else x ** 2


def get_energy(x, axis=None, keepdims=False):
    return np.sum(abs_square(np.asarray(x, dtype=np.complex128)), axis=axis, keepdims=keepdims)


def set_snr_factor(X, N, snr, axis=None):
    pX = np.mean(abs_square(X), axis=axis, keepdims=True)
    pN = np.mean(abs_square(N), axis=axis, keepdims=True)
    return 10 ** (-(snr - 10 * np.log10(pX / pN)) / 20)


def get_pca(m):
    w, v = np.linalg.eigh(m)
    return v[..., -1], w[..., -1]
