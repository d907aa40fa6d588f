"""NumPy restatement of the pb_bss hot path (TEST INFRASTRUCTURE, see oracle/__init__.py).

Every function names the reference lines it follows (paths relative to the
reference checkout, e.g. ``pb_bss/distribution/cacgmm.py:252-278``).  The
arithmetic (einsum expressions, LAPACK entry points, floors, clip constants)
is kept the same as the reference so that (a) results agree to rounding and
(b) the CPU cost is representative when this module is timed as the
``cpu_baseline`` of ``bench.py``.

Parity: PINNED against the live reference, see ``oracle/make_golden.py`` and
``tests/test_oracle_golden.py``.
"""
import math

import numpy as np
import scipy.linalg
import scipy.special
from scipy.interpolate import interp1d

TINY64 = np.finfo(np.float64).tiny


# --------------------------------------------------------------------------
# observation normalisation
# --------------------------------------------------------------------------
def normalize_observation_cacg(y):
    """(..., N, D) -> unit-norm, swapped to (..., D, N).

    pb_bss/distribution/complex_angular_central_gaussian.py:34-55 with
    pb_bss/distribution/utils.py:223-256 (eps_style='where': a zero norm is
    replaced by ``tiny`` so a zero vector stays zero).
    """
    norm = np.linalg.norm(y, axis=-1, keepdims=True)
    norm = np.where(norm == 0, np.finfo(y.dtype).tiny, norm)
    return np.ascontiguousarray(np.swapaxes(y / norm, -2, -1))


def normalize_observation_cw(y):
    """(..., N, D) -> unit norm, layout unchanged.

    pb_bss/distribution/complex_watson.py:16-29 (``max(norm, tiny)``).
    """
    return y / np.maximum(
        np.linalg.norm(y, axis=-1, keepdims=True), np.finfo(y.dtype).tiny)


# --------------------------------------------------------------------------
# cACG: E-step pieces
# --------------------------------------------------------------------------
def cacg_log_pdf(z, eigenvectors, eigenvalues):
    """z (..., D, N) against eigen-decomposed covariances (..., D, D)/(..., D).

    pb_bss/distribution/complex_angular_central_gaussian.py:167-203.
    Returns (log_pdf, quadratic_form), both (..., N).
    """
    D = z.shape[-2]
    q = np.einsum(
        '...dt,...de,...e,...ge,...gt->...t',
        z.conj(), eigenvectors, 1 / eigenvalues, eigenvectors.conj(), z,
        optimize='optimal',
    )
    q = np.maximum(np.abs(q), np.finfo(z.dtype).tiny)
    log_pdf = -D * np.log(q)
    log_pdf -= np.sum(np.log(eigenvalues), axis=-1)[..., None]
    return log_pdf, q


def log_pdf_to_affiliation(weight, log_pdf, source_activity_mask=None,
                           affiliation_eps=0.):
    """Posterior over classes (axis -2).

    pb_bss/distribution/mixture_model_utils.py:7-55.
    """
    a = log_pdf - np.amax(log_pdf, axis=-2, keepdims=True)
    np.exp(a, out=a)
    a = a * weight
    if source_activity_mask is not None:
        a = a * source_activity_mask
    den = np.maximum(np.sum(a, axis=-2, keepdims=True),
                     np.finfo(a.dtype).tiny)
    a = a / den
    if affiliation_eps != 0:
        a = np.clip(a, affiliation_eps, 1 - affiliation_eps)
    return a


def estimate_mixture_weight(affiliation, saliency=None,
                            weight_constant_axis=-1):
    """pb_bss/distribution/mixture_model_utils.py:133-203."""
    affiliation = np.asarray(affiliation)
    if isinstance(weight_constant_axis, int) and \
            weight_constant_axis % affiliation.ndim - affiliation.ndim == -2:
        K = affiliation.shape[-2]
        return np.full([K, 1], 1 / K)
    if isinstance(weight_constant_axis, list):
        weight_constant_axis = tuple(weight_constant_axis)
    if saliency is None:
        return np.mean(affiliation, axis=weight_constant_axis, keepdims=True)
    s = np.sum(affiliation * saliency[..., None, :],
               axis=weight_constant_axis, keepdims=True)
    # _unit_norm(ord=1, axis=-2, eps=1e-10, eps_style='where')
    n = np.linalg.norm(s, ord=1, axis=-2, keepdims=True)
    n = np.where(n == 0, 1e-10, n)
    return s / n


# --------------------------------------------------------------------------
# cACG: M-step pieces
# --------------------------------------------------------------------------
def cacg_covariance(z, masked_affiliation, quadratic_form, hermitize=True):
    """Weighted scatter matrix before the eigendecomposition.

    pb_bss/distribution/complex_angular_central_gaussian.py:295-336.
    z (..., 1, D, N), masked_affiliation / quadratic_form (..., K, N).
    """
    D = z.shape[-2]
    den = np.einsum('...n->...', masked_affiliation)[..., None, None]
    q = np.maximum(quadratic_form,
                   10 * np.finfo(quadratic_form.dtype).tiny)
    cov = D * np.einsum('...dn,...Dn,...n->...dD', z, z.conj(),
                        masked_affiliation / q)
    cov = cov / np.maximum(den, np.finfo(den.dtype).tiny)
    if hermitize:
        cov = (cov + np.swapaxes(cov.conj(), -1, -2)) / 2
    return cov


def cacg_from_covariance(covariance, eigenvalue_floor=0.,
                         covariance_norm='eigenvalue'):
    """pb_bss/distribution/complex_angular_central_gaussian.py:81-132.

    Returns (eigenvectors (..., D, D), eigenvalues (..., D)), ascending.
    """
    if covariance_norm == 'trace':
        tr = np.einsum('...dd', covariance)[..., None, None]
        covariance = covariance / np.maximum(tr, np.finfo(tr.dtype).tiny)
    else:
        assert covariance_norm in ['eigenvalue', False], covariance_norm
    lam, vec = np.linalg.eigh(covariance)
    lam = lam.real
    if covariance_norm == 'eigenvalue':
        lam = lam / np.maximum(np.amax(lam, axis=-1, keepdims=True),
                               np.finfo(lam.dtype).tiny)
        lam = np.maximum(lam, eigenvalue_floor)
    else:
        lam = np.maximum(
            lam, np.amax(lam, axis=-1, keepdims=True) * eigenvalue_floor)
    return vec, lam


def cacg_covariance_from_eig(eigenvectors, eigenvalues):
    """pb_bss/distribution/complex_angular_central_gaussian.py:140-148."""
    return np.einsum('...wx,...x,...zx->...wz', eigenvectors, eigenvalues,
                     eigenvectors.conj(), optimize='greedy')


# --------------------------------------------------------------------------
# cACGMM EM driver
# --------------------------------------------------------------------------
def cacgmm_e_step(z, model, source_activity_mask=None, affiliation_eps=0.):
    """pb_bss/distribution/cacgmm.py:73-95 (``CACGMM._predict``)."""
    log_pdf, q = cacg_log_pdf(z[..., None, :, :], model['eigenvectors'],
                              model['eigenvalues'])
    aff = log_pdf_to_affiliation(model['weight'], log_pdf,
                                 source_activity_mask, affiliation_eps)
    return aff, q, log_pdf


def cacgmm_m_step(z, quadratic_form, affiliation, saliency=None,
                  hermitize=True, covariance_norm='eigenvalue',
                  eigenvalue_floor=1e-10, weight_constant_axis=(-1,)):
    """pb_bss/distribution/cacgmm.py:315-345."""
    weight = estimate_mixture_weight(affiliation, saliency,
                                     weight_constant_axis)
    masked = affiliation if saliency is None \
        else affiliation * saliency[..., None, :]
    cov = cacg_covariance(z[..., None, :, :], masked, quadratic_form,
                          hermitize)
    vec, lam = cacg_from_covariance(cov, eigenvalue_floor, covariance_norm)
    return dict(weight=weight, eigenvectors=vec, eigenvalues=lam)


def cacgmm_fit(y, initialization, iterations=100, *, saliency=None,
               source_activity_mask=None, weight_constant_axis=(-1,),
               hermitize=True, covariance_norm='eigenvalue',
               affiliation_eps=1e-10, eigenvalue_floor=1e-10,
               inline_permutation_plan=None):
    """EM loop of ``CACGMMTrainer.fit`` (pb_bss/distribution/cacgmm.py:142-280).

    ``initialization`` is an affiliation array (..., K, N) (singleton
    independent dims broadcast, cacgmm.py:211-228) or a model dict
    (warm start, cacgmm.py:229-234).  Random initialisation (cacgmm.py:206-210)
    is the caller's job: draw ``np.random.uniform`` and normalise over K.
    ``inline_permutation_plan``: alignment plan of a DHTVPermutationAlignment run
    after every E-step (``inline_permutation_aligner``, cacgmm.py:260-267).
    Returns dict(weight, eigenvectors, eigenvalues).
    """
    assert np.iscomplexobj(y), y.dtype
    assert y.shape[-1] > 1, y.shape
    z = normalize_observation_cacg(y)
    *independent, D, N = z.shape
    model = None
    if isinstance(initialization, dict):
        model = initialization
    else:
        K = initialization.shape[-2]
        shape = (*independent, K, N)
        assert initialization.ndim == len(shape), (initialization.shape, shape)
        affiliation = np.broadcast_to(
            initialization.astype(z.real.dtype), shape)
        quadratic_form = np.ones(shape, dtype=z.real.dtype)
    for _ in range(iterations):
        if model is not None:
            affiliation, quadratic_form, _lp = cacgmm_e_step(
                z, model, source_activity_mask, affiliation_eps)
            if inline_permutation_plan is not None:
                # apply_inline_permutation_alignment, mixture_model_utils.py:264-306
                # (cacgmm.py:260-267): DHTV alignment of the (K, F, T) affiliations,
                # the quadratic forms follow the same mapping
                mask = np.ascontiguousarray(np.transpose(affiliation, (1, 0, 2)))
                mapping = dhtv_calculate_mapping(mask, inline_permutation_plan)
                affiliation = np.transpose(apply_mapping(mask, mapping), (1, 0, 2))
                quadratic_form = np.transpose(
                    apply_mapping(np.transpose(quadratic_form, (1, 0, 2)), mapping), (1, 0, 2))
        model = cacgmm_m_step(
            z, quadratic_form, affiliation, saliency, hermitize,
            covariance_norm, eigenvalue_floor, weight_constant_axis)
    return model


def cacgmm_predict(y, model, return_quadratic_form=False,
                   source_activity_mask=None):
    """pb_bss/distribution/cacgmm.py:64-71 (affiliation_eps = 0)."""
    z = normalize_observation_cacg(y)
    aff, q, _ = cacgmm_e_step(z, model, source_activity_mask, 0.)
    return (aff, q) if return_quadratic_form else aff


def cacgmm_log_likelihood(y, model):
    """pb_bss/distribution/cacgmm.py:97-138 (logsumexp WITHOUT weights)."""
    z = normalize_observation_cacg(y)
    _, _, log_pdf = cacgmm_e_step(z, model)
    return np.sum(scipy.special.logsumexp(log_pdf, axis=-2))


# --------------------------------------------------------------------------
# complex Watson
# --------------------------------------------------------------------------
def cw_log_norm(concentration, D):
    """pb_bss/distribution/complex_watson.py:157-168 (``log_norm_1f1``)."""
    norm = scipy.special.hyp1f1(1, D, concentration) * (
        2 * np.pi ** D / math.factorial(D - 1))
    return np.log(norm)


def cw_log_pdf(z, mode, concentration):
    """z (..., N, D), mode (..., D), concentration (...).

    pb_bss/distribution/complex_watson.py:73-87.
    """
    D = mode.shape[-1]
    r = np.einsum('...d,...d', z, mode[..., None, :].conj())
    r = r.real ** 2 + r.imag ** 2
    r = r * concentration[..., None]
    r = r - cw_log_norm(concentration, D)[..., None]
    return r


def cw_hypergeometric_ratio(concentration, D):
    """pb_bss/distribution/complex_watson.py:258-262."""
    return scipy.special.hyp1f1(2, D + 1, concentration) / (
        D * scipy.special.hyp1f1(1, D, concentration))


def cw_spline(D, max_concentration=500, spline_markers=1000):
    """Inverse of the hypergeometric ratio as a quadratic spline.

    pb_bss/distribution/complex_watson.py:237-256.
    """
    x = np.logspace(-3, np.log10(max_concentration), spline_markers)
    y = cw_hypergeometric_ratio(x, D)
    return interp1d(y, x, kind='quadratic', assume_sorted=True,
                    bounds_error=False, fill_value=(0, max_concentration))


def principal_component(psd):
    """Top eigenpair of Hermitian matrices (..., D, D).

    pb_bss/utils.py:111-169 (``get_pca``, numpy branch).
    """
    lam, vec = np.linalg.eigh(psd)
    return vec[..., -1], lam[..., -1]


def cw_fit_step(z, masked_affiliation, spline):
    """pb_bss/distribution/complex_watson.py:300-315 (saliency branch)."""
    cov = np.einsum('...n,...nd,...nD->...dD', masked_affiliation, z,
                    z.conj())
    den = np.einsum('...n->...', masked_affiliation)[..., None, None]
    cov = cov / den
    mode, lam = principal_component(cov)
    return mode, spline(lam)


def cwmm_predict_normalized(z, model):
    """pb_bss/distribution/cwmm.py:40-52 (``CWMM._predict``)."""
    return log_pdf_to_affiliation(
        model['weight'],
        cw_log_pdf(z[..., None, :, :], model['mode'], model['concentration']),
        None, 0.)


def cwmm_predict(y, model):
    """pb_bss/distribution/cwmm.py:26-38."""
    return cwmm_predict_normalized(normalize_observation_cw(y), model)


def cwmm_fit(y, initialization, iterations=100, *, saliency=None,
             weight_constant_axis=(-1,), max_concentration=500,
             spline_markers=1000, inline_permutation_plan=None):
    """EM loop of ``CWMMTrainer.fit`` (pb_bss/distribution/cwmm.py:76-240).

    ``inline_permutation_plan``: alignment plan of a DHTVPermutationAlignment run after every
    E-step (``inline_permutation_aligner``, cwmm.py:169-174, mixture_model_utils.py:264-306).
    Returns dict(weight, mode, concentration).
    """
    assert np.iscomplexobj(y), y.dtype
    z = normalize_observation_cw(y)
    D = z.shape[-1]
    if saliency is None:
        saliency = np.ones_like(initialization[..., 0, :])  # cwmm.py:129-130
    spline = cw_spline(D, max_concentration, spline_markers)
    affiliation = initialization
    model = None
    for _ in range(iterations):
        if model is not None:
            # CWMM.predict re-normalises y every iteration (cwmm.py:35-37,166)
            affiliation = cwmm_predict(z, model)
            if inline_permutation_plan is not None:
                mask = np.ascontiguousarray(np.transpose(affiliation, (1, 0, 2)))
                mapping = dhtv_calculate_mapping(mask, inline_permutation_plan)
                affiliation = np.transpose(apply_mapping(mask, mapping), (1, 0, 2))
        weight = estimate_mixture_weight(affiliation, saliency,
                                         weight_constant_axis)
        masked = affiliation * saliency[..., None, :]
        mode, kappa = cw_fit_step(z[..., None, :, :], masked, spline)
        model = dict(weight=weight, mode=mode, concentration=kappa)
    return model


# --------------------------------------------------------------------------
# permutation alignment
# --------------------------------------------------------------------------
def _interleave(a, b):
    """pb_bss/permutation_alignment.py:12-39 for two lists."""
    out = []
    for i in range(max(len(a), len(b))):
        if i < len(a):
            out.append(a[i])
        if i < len(b):
            out.append(b[i])
    return out


def dhtv_alignment_plan(stft_size, segment_start, segment_width,
                        segment_shift, main_iterations, sub_iterations):
    """pb_bss/permutation_alignment.py:204-293.  List of [iters, start, end]."""
    F = stft_size // 2 + 1
    if segment_start + segment_width > F:
        raise ValueError('segment_start + segment_width must be smaller '
                         'than stft_size // 2 + 1')
    lower = [[sub_iterations, s, s + segment_width]
             for s in range(segment_start + segment_shift,
                            F - segment_width, segment_shift)]
    higher = [[sub_iterations, s, s + segment_width]
              for s in range(segment_start - segment_shift, 0,
                             -segment_shift)]
    first = [main_iterations, segment_start, segment_start + segment_width]
    if lower:
        lower[-1][-1] = F
    else:
        first[-1] = F
    if higher:
        higher[-1][1] = 0
    else:
        first[1] = 0
    return [first] + _interleave(lower, higher)


def dhtv_plan_from_stft_size(stft_size):
    """pb_bss/permutation_alignment.py:164-184."""
    start = {512: 70, 1024: 100}[stft_size]
    return dhtv_alignment_plan(stft_size, start, 100, 20, 20, 2)


def greedy_mapping_from_score_matrix(score, return_margin=False):
    """score (K, K) [reference, mask] -> reverse permutation (K,).

    pb_bss/permutation_alignment.py:525-553: K times take the first argmax of
    the row-major flattened matrix, then blank its row and column.

    return_margin: also return the smallest gap, over the K rounds, between the
    chosen entry and the largest entry still in play in its row or column (inf
    if there was none).  0 means an exact tie decided by the scan order.  Only
    these runner-ups matter: if a near-equal entry in another row and column
    were taken first, the chosen one would still be taken next (greedy matching
    is fixed by the order of entries that share a row or column).
    """
    score = np.array(score, dtype=np.float64)
    K = score.shape[-1]
    out = np.zeros(K, dtype=np.int64)
    margin = np.inf
    for _ in range(K):
        flat = score.reshape(-1)
        n = np.argmax(flat)
        i, j = np.unravel_index(n, score.shape)
        if return_margin:
            rest = np.concatenate([np.delete(score[i], j), np.delete(score[:, j], i)])
            rest = rest[rest > -np.inf]
            if rest.size:
                margin = min(margin, score[i, j] - rest.max())
        score[i, :] = -np.inf
        score[:, j] = -np.inf
        out[i] = j
    return (out, margin) if return_margin else out


def _vector_norm(a):
    """pb_bss/permutation_alignment.py:358-377."""
    n = np.linalg.norm(a, axis=-1, keepdims=True)
    return a / np.maximum(n, np.finfo(n.dtype).tiny)


def _relative_margin(gap, score):
    """A decision margin in units of the largest |score| of its matrix."""
    scale = np.max(np.abs(score))
    if scale > 0:
        return gap / scale
    return np.inf if gap > 0 else 0.0


def dhtv_calculate_mapping(mask, plan, similarity_metric='cos', algorithm='greedy', return_margin=False):
    """mask (K, F, T) -> mapping (K, F) int.

    pb_bss/permutation_alignment.py:295-355.  For 'cos' the features and the
    centroid are L2-normalised over time and scored by the inner product
    (_ScoreMatrix.multiply, :158-162); 'multiply' and 'euclidean' score the raw
    masks.  The assignment is _mapping_from_score_matrix(algorithm).

    return_margin: also return the smallest decision margin of every
    assignment made (see greedy_ / optimal_mapping_from_score_matrix), relative
    to the largest |score| of its bin's score matrix.
    """
    K, F, _ = mask.shape
    cos = similarity_metric == 'cos'
    metric = 'multiply' if cos else similarity_metric
    assign = {'greedy': greedy_mapping_from_score_matrix, 'optimal': optimal_mapping_from_score_matrix}[algorithm]
    features = _vector_norm(mask) if cos else np.array(mask, dtype=np.float64)
    mapping = np.repeat(np.arange(K)[:, None], F, axis=1)
    margin = np.inf
    for iterations, start, end in plan:
        for _ in range(iterations):
            centroid = np.mean(features[:, start:end, :], axis=1)
            if cos:
                centroid = _vector_norm(centroid)
            nothing_changed = True
            for f in range(start, end):
                score = score_matrix(features[:, f:f + 1, :], centroid[:, None, :], metric)[0]
                perm, gap = assign(score, return_margin=True)
                margin = min(margin, _relative_margin(gap, score))
                if not (perm == np.arange(K)).all():
                    nothing_changed = False
                    features[:, f, :] = features[perm, f, :]
                    mapping[:, f] = mapping[perm, f]
            if nothing_changed:
                break
    return (mapping, margin) if return_margin else mapping


def score_matrix(mask, reference_mask, similarity_metric):
    """(K, F, T) x (K, F, T) -> (F, k_ref, K_mask), pb_bss/permutation_alignment.py:380-420."""
    if similarity_metric == 'cos':
        mask, reference_mask = _vector_norm(mask), _vector_norm(reference_mask)
    if similarity_metric in ('cos', 'multiply'):
        return np.einsum('KFT,kFT->FkK', mask, reference_mask)
    if similarity_metric == 'euclidean':
        d = np.sqrt(np.sum(np.abs(mask[None] - reference_mask[:, None]) ** 2, axis=-1))  # (k, K, F)
        return -np.moveaxis(d, -1, 0)
    raise ValueError(similarity_metric)


_PERMUTATIONS = {}


def _permutations(K):
    """itertools.permutations(range(K)) as a (K!, K) index array, in that order."""
    if K not in _PERMUTATIONS:
        import itertools
        _PERMUTATIONS[K] = np.array(list(itertools.permutations(range(K))), dtype=np.intp).reshape(-1, K)
    return _PERMUTATIONS[K]


def optimal_mapping_from_score_matrix(score, return_margin=False):
    """score (K, K) -> first best of itertools.permutations (pb_bss/permutation_alignment.py:556-585).

    Every permutation's score is summed left to right, one class at a time, as
    the reference's sum() does; np.argmax returns the first maximum, which is
    the reference's strict '>'.  return_margin: also return the gap between the
    best and the second-best permutation sum (inf for K = 1).
    """
    score = np.asarray(score)
    K = score.shape[-1]
    perms = _permutations(K)
    sums = score[0, perms[:, 0]]
    for k in range(1, K):
        sums = sums + score[k, perms[:, k]]
    best = int(np.argmax(sums))
    out = perms[best].astype(np.int64)
    if not return_margin:
        return out
    margin = np.inf if len(sums) == 1 else float(sums[best] - np.delete(sums, best).max())
    return out, margin


def mapping_from_score_matrix(scores, algorithm, return_margin=False):
    """scores (F, K, K) -> mapping (K, F), pb_bss/permutation_alignment.py:458-590.

    return_margin: also return the smallest decision margin over the bins,
    each relative to the largest |score| of its bin."""
    if not np.all(np.isfinite(scores)):
        raise ValueError('score matrix is infeasible')
    fn = {'greedy': greedy_mapping_from_score_matrix, 'optimal': optimal_mapping_from_score_matrix}[algorithm]
    res = [fn(sc, return_margin=True) for sc in scores]
    mapping = np.stack([r[0] for r in res], axis=1) if res else np.zeros((scores.shape[-1], 0), np.int64)
    if not return_margin:
        return mapping
    return mapping, min((_relative_margin(r[1], sc) for r, sc in zip(res, scores)), default=np.inf)


def greedy_permutation_alignment(mask, similarity_metric='euclidean', return_margin=False):
    """GreedyPermutationAlignment.calculate_mapping, pb_bss/permutation_alignment.py:612-714
    (the pairwise assignment is always 'greedy', :703)."""
    K, F, _ = mask.shape
    pair, margin = mapping_from_score_matrix(score_matrix(mask[:, 1:], mask[:, :-1], similarity_metric), 'greedy',
                                             return_margin=True)
    mapping = np.concatenate([np.arange(K)[:, None], pair], axis=1)
    for f in range(1, F):
        mapping[:, f] = mapping[mapping[:, f - 1], f]
    return (mapping, margin) if return_margin else mapping


def oracle_permutation_alignment(mask, reference_mask, similarity_metric='euclidean', algorithm='optimal',
                                 return_margin=False):
    """OraclePermutationAlignment.calculate_mapping, pb_bss/permutation_alignment.py:723-786."""
    return mapping_from_score_matrix(score_matrix(mask, reference_mask, similarity_metric), algorithm,
                                     return_margin=return_margin)


def apply_mapping(mask, mapping):
    """pb_bss/permutation_alignment.py:54-104."""
    K, F = mapping.shape
    return mask[mapping, range(F)]


# --------------------------------------------------------------------------
# beamforming
# --------------------------------------------------------------------------
def power_spectral_density(observation, mask=None, normalize=True):
    """observation (..., D, T); mask None, (..., T) or (..., K, T).

    pb_bss/extraction/beamformer.py:59-160 for the default dim arguments.
    """
    if mask is None:
        psd = np.einsum('...dt,...et->...de', observation, observation.conj())
        return psd / observation.shape[-1]
    mask = np.array(mask, dtype=np.float64)
    if normalize:
        mask = mask / np.maximum(np.sum(mask, axis=-1, keepdims=True), 1e-10)
    if mask.ndim + 1 == observation.ndim:
        return np.einsum('...dt,...et->...de',
                         mask[..., None, :] * observation, observation.conj())
    return np.einsum('...kt,...dt,...et->...kde', mask, observation,
                     observation.conj())


def pca_vector(target_psd):
    """pb_bss/extraction/beamformer.py:197-224 with scaling=None."""
    return principal_component(target_psd)[0]


def mvdr_vector(atf_vector, noise_psd):
    """pb_bss/extraction/beamformer.py:230-260."""
    while atf_vector.ndim > noise_psd.ndim - 1:
        noise_psd = noise_psd[None]
    noise_psd = 0.5 * (noise_psd + np.conj(noise_psd.swapaxes(-1, -2)))
    num = np.linalg.solve(noise_psd, atf_vector[..., None])[..., 0]
    den = np.einsum('...d,...d->...', atf_vector.conj(), num)
    return num / den[..., None]


def gev_vector(target_psd, noise_psd):
    """Top generalised eigenvector per matrix pair (LAPACK zhegvd semantics).

    pb_bss/extraction/beamformer.py:367-411 (``scipy.linalg.eigh(a, b)`` loop);
    pb_bss/extraction/cythonized/get_gev_vector.pyx:124-150 calls the same
    LAPACK routine (ITYPE=1, JOBZ='V', UPLO='L') and is bit-identical
    (SURVEY.md section 8c).
    """
    D = target_psd.shape[-1]
    shape = target_psd.shape
    a = target_psd.reshape(-1, D, D)
    b = noise_psd.reshape(-1, D, D)
    out = np.empty((a.shape[0], D), dtype=np.complex128)
    for f in range(a.shape[0]):
        lam, vec = scipy.linalg.eigh(a[f], b[f])
        out[f] = vec[:, np.argmax(lam)]
    return out.reshape(shape[:-1])


def mvdr_vector_souden(target_psd, noise_psd, ref_channel=None):
    """pb_bss/extraction/beamformer.py:601-698 (regular matrices: np.linalg.solve,
    pb_bss/math/solve.py:95-97)."""
    phi = np.linalg.solve(noise_psd, target_psd)
    lam = np.trace(phi, axis1=-1, axis2=-2)[..., None, None]
    eps = np.finfo(lam.real.dtype).tiny
    mat = phi / np.maximum(lam.real, eps)
    if ref_channel is None:
        snr = np.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), target_psd,
                        mat) / np.maximum(
            np.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), noise_psd,
                      mat), eps)
        ref_channel = int(np.argmax(snr.real))
    return mat[..., ref_channel], ref_channel


def blind_analytic_normalization(vector, noise_psd):
    """pb_bss/extraction/beamformer.py:459-488."""
    nom = np.sqrt(np.einsum('...a,...ab,...bc,...c->...', vector.conj(),
                            noise_psd, noise_psd, vector))
    den = np.einsum('...a,...ab,...b->...', vector.conj(), noise_psd, vector)
    den = np.sqrt(den * den.conj())
    norm = np.divide(nom, den, out=np.zeros_like(nom), where=den != 0)
    return vector * np.abs(norm[..., None])


def apply_beamforming_vector(vector, mix):
    """pb_bss/extraction/beamformer.py:572-583."""
    return np.einsum('...a,...at->...t', vector.conj(), mix)
