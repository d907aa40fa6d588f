"""pb_bss/distribution/mixture_model_utils.py on the device: the public building blocks (log_pdf_to_affiliation,
its inline-permutation-alignment variant, estimate_mixture_weight, apply_inline_permutation_alignment), and the EM
plumbing the mixture-model trainers share: the fit preamble, the weight layouts between the public models and the
kernels, models to NumPy, and the EM loop whose bins couple in every iteration (frequency-tied mixture weights, inline
permutation alignment) for cACGMM, CWMM and CBMM."""
import copy
import ctypes
import dataclasses
import math
from operator import xor

import numpy as np
import torch
from numpy.lib.array_utils import normalize_axis_tuple

from .. import _device, _lib, _nd
from .gaussian import _dev
from .utils import _ProbabilisticModel, _unit_norm

MAX_INLINE_PA_K = 6  # pbb_log_pdf_to_affiliation enumerates the K! pairings of every bin


def check_initialization(initialization, num_classes):
    assert xor(initialization is None, num_classes is None), (
        'Incompatible input combination. '
        'Exactly one of the two inputs has to be None: '
        f'{initialization is None} xor {num_classes is None}')


def flatten_obs(y):
    *independent, N, D = y.shape
    F = int(np.prod(independent)) if independent else 1
    return tuple(independent), F, N, D


def weight_mode(weight_constant_axis, ndim):
    """Maps ``weight_constant_axis`` (mixture_model_utils.py:133-203) onto the
    modes the kernels implement; ``ndim`` is the affiliation rank.
    WEIGHT_TIME: (-1,); WEIGHT_CONST: -2; WEIGHT_TIED_TIME: (-3,) and
    WEIGHT_TIED: (-3, -1) (frequency-tied, only for a single independent dim)."""
    if isinstance(weight_constant_axis, list):
        weight_constant_axis = tuple(weight_constant_axis)
    if isinstance(weight_constant_axis, int):
        ax = weight_constant_axis % ndim - ndim
        if ax == -2:
            return _lib.WEIGHT_CONST  # constant 1/K, shape (K, 1)
        axes = (ax,)
    else:
        axes = tuple(sorted(a % ndim - ndim for a in weight_constant_axis))
    if axes == (-1,):
        return _lib.WEIGHT_TIME
    if ndim >= 3 and axes == (-3,):
        return _lib.WEIGHT_TIED_TIME
    if ndim >= 3 and axes == (-3, -1):
        return _lib.WEIGHT_TIED
    raise NotImplementedError(
        f'weight_constant_axis={weight_constant_axis!r}: supported on the '
        'device are (-1,), -2, (-3,) and (-3, -1) (the last independent dim, the bins, tied).')


def status_check(status, what):
    """Reads a cACGMM / CWMM status word now (synchronises the stream) or at the end of the enclosing
    ``_device.deferred_status()`` block."""
    def on_error(s):
        # the reference asserts finiteness at cacg.py:127,326,333
        raise AssertionError(f'{what}: non-finite covariance / eigenvalues in bin {s - 1}')
    _device.check_status(status, on_error)


def initial_affiliation(initialization, num_classes, lead, N):
    """The reference's random initialisation from NumPy's global stream (gmm.py:71-76, vmfmm.py:80-85), or the given
    one broadcast to the leading dims -> (B, K, N) device."""
    if initialization is None:
        initialization = np.random.uniform(size=(*lead, num_classes, N))
        initialization /= np.einsum('...kn->...n', initialization)[..., None, :]
    aff = _dev(initialization)
    K = aff.shape[-2]
    return aff.expand(lead + (K, N)).reshape(math.prod(lead), K, N).contiguous()


def saliency_bn(saliency, lead, N):
    return None if saliency is None else _dev(saliency).expand(lead + (N,)).reshape(math.prod(lead), N).contiguous()


def masked_affiliation(aff, sal):
    return aff if sal is None else (aff * sal[:, None, :]).contiguous()


def class_weight(masked):
    """Per-row class weights of masked affiliations (B, K, N) (gcacgmm.py:286-291): the sum over N divided by its
    sum over the classes -> (B, K).  The sums are non-negative, so that divisor is their L1 norm; with eps = 0 a row
    without weight stays 0 / 0 = NaN, as in the reference."""
    return _unit_norm(_nd.axis_sum(masked, (2,), False), ord=1, axis=-1, eps=0.)


def tied_weight(affiliation, sal, mode, saliency_form):
    """The frequency-tied weight of (F, K, T) affiliations (estimate_mixture_weight, mixture_model_utils.py:187-203)
    -> (1, K, T) for WEIGHT_TIED_TIME, (1, K, 1) for WEIGHT_TIED, float64: the mean over the bins (and frames), or,
    with saliency_form, the sum of affiliation * saliency L1-normalised over the classes.  sal: (F, T) or None."""
    axes = (0,) if mode == _lib.WEIGHT_TIED_TIME else (0, 2)
    weight = _nd.axis_sum(affiliation, axes, True, multiplier=None if sal is None else sal[:, None, :],
                          divide_by_count=not saliency_form, out_dtype=torch.float64)
    if saliency_form:
        weight = _unit_norm(weight, ord=1, axis=-2, eps=1e-10, eps_style='where')
    return weight


def weight_to_device(weight, independent, F, K, N):
    """A model's weight -> (device weight, mode) for the predict kernels: (..., K, 1) -> (F, K) WEIGHT_TIME; the
    time-varying weight (..., K, T) of weight_constant_axis=(-3,), shared by every bin -> (K, T) WEIGHT_TIED_TIME."""
    w = _device.to_device(weight, torch.float64)
    if w.shape[-1] == 1:
        return w[..., 0].expand(*independent, K).reshape(F, K).contiguous(), _lib.WEIGHT_TIME
    assert all(int(n) == 1 for n in w.shape[:-2]), (tuple(w.shape), independent)
    # the reference broadcasts the weight against the (..., K, N) log pdf, which fails for T != N
    if w.shape[-1] != N:
        raise ValueError(f'time-varying weight has {w.shape[-1]} frames, the observation {N}')
    return w.reshape(K, N).contiguous(), _lib.WEIGHT_TIED_TIME


def weight_to_host(mode, w, independent, K, like_numpy):
    """The per-bin weight (F, K) of a fit -> the reference's (..., K, 1), or (K, 1) of 1/K for WEIGHT_CONST."""
    if mode == _lib.WEIGHT_CONST:
        weight = np.full([K, 1], 1 / K)  # mixture_model_utils.py:180-183
        return weight if like_numpy else _device.to_device(weight)
    return _device.to_host(w.reshape(*independent, K, 1), like_numpy)


def _walk(models, leaf):
    """A copy of ``models[0]`` whose every field is ``leaf`` of that field of all ``models``; fields that are models
    themselves are walked the same way.  No constructor runs, so nothing is recomputed."""
    out = copy.copy(models[0])
    for f in dataclasses.fields(out):
        values = [getattr(m, f.name) for m in models]
        setattr(out, f.name, _walk(values, leaf) if isinstance(values[0], _ProbabilisticModel) else leaf(values))
    return out


def model_to_host(model):
    """The model with every tensor, also those of its sub-models, as a NumPy array; other fields stay as they are."""
    return _walk([model], lambda v: _device.to_host(v[0], True) if _device.is_tensor(v[0]) else v[0])


# trailing dims of the trainers' array arguments; the dims in front of them are the leading independent dims
_TRAILING_DIMS = {'y': 3, 'initialization': 3, 'saliency': 2, 'source_activity_mask': 3}


def fit_tied_leading(fit, lead, **kwargs):
    """Frequency-tied weights with more than one independent dim, e.g. y (B, F, T, D): the weights are tied over the
    last independent dim (the bins) only, the reference's mean over axis -3 keeps the leading indices apart
    (mixture_model_utils.py:187).  So every index of ``lead`` is its own ``fit(**kwargs)``, with the array arguments
    picked at that index (singleton dims broadcast), and the models are stacked to (*lead, ...)."""
    def pick(name, x, idx):
        nlead = x.ndim - _TRAILING_DIMS[name] if name in _TRAILING_DIMS and x is not None else 0
        if nlead <= 0:
            return x
        return x[tuple(i if x.shape[d] != 1 else 0 for d, i in enumerate(idx[len(lead) - nlead:]))]

    def stack(values):
        x = torch.stack(values) if _device.is_tensor(values[0]) else np.stack(values)
        return x.reshape(*lead, *values[0].shape)
    models = [fit(**{k: pick(k, v, idx) for k, v in kwargs.items()}) for idx in np.ndindex(*lead)]
    return _walk(models, stack)


def coupled_fit(yd, affiliation, model, iterations, weight_constant_axis, sal, aligner, predict, m_step,
                saliency_form, total_bins=None, bin_group=None):
    """EM whose bins couple in every iteration: frequency-tied mixture weights (``weight_constant_axis`` (-3,) /
    (-3, -1), mixture_model_utils.py:187-190) and / or the inline permutation alignment
    (mixture_model_utils.py:264-306); with per-bin weights (the cACGMM fit with a graph) the model is the M-step's.  The loop is the reference's (cacgmm.py:252-278, cwmm.py:152-184,
    cbmm.py:186-203); every step runs on the device and the status words are read once, after the last iteration.

    yd: (F, N, D) device observation; affiliation: initial (F, K, N) device affiliations, or ``model`` to start from;
    sal: (F, N) device saliency or None.  ``predict(model)`` -> (affiliation (F, K, N), quadratic form or None);
    ``m_step(affiliation, quadratic_form)`` -> model with per-bin weights, which then get the tied weight.
    saliency_form: the tied weight is the sum of affiliation * saliency L1-normalised over the classes (tied_weight).
    total_bins, bin_group: ``yd`` holds this rank's slice of ``total_bins`` bins (pb_bss_b200.parallel).
    Returns the model of device tensors."""
    from .. import parallel
    from ..permutation_alignment import apply_mapping
    independent, F, _, _ = flatten_obs(yd)
    mode = weight_mode(weight_constant_axis, len(independent) + 2)
    if aligner is not None:
        message = ('Inline permutation alignment reduces mismatch between frequency independent '
                   'mixtures weights and a frequency independent observation model. Therefore, we '
                   f'require `affiliation.ndim == 3` and a corresponding `weight_constant_axis` '
                   f'({weight_constant_axis}).')
        assert len(independent) == 1 and mode in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED), message
    F_all = F if total_bins is None else int(total_bins)
    lo, hi = parallel.local_bins(F_all, bin_group) if F_all != F else (0, F)
    assert hi - lo == F, ('this rank holds bins', (lo, hi), 'but y has', F)
    if sal is not None and F_all != F:
        raise NotImplementedError('saliency with frequency-tied weights is single-rank only')
    quadratic_form = None
    with _device.deferred_status():
        for _ in range(iterations):
            if model is not None:
                affiliation, quadratic_form = predict(model)
                if aligner is not None:
                    mask_kft = affiliation.permute(1, 0, 2).contiguous()
                    if F_all != F:  # the alignment needs every bin: gather, align replicated, keep the slice
                        every = parallel.all_gather_bins(affiliation.contiguous(), F_all, bin_group)
                        mapping = aligner.calculate_mapping(every.permute(1, 0, 2).contiguous())[:, lo:hi].contiguous()
                    else:
                        mapping = aligner.calculate_mapping(mask_kft)
                    affiliation = apply_mapping(mask_kft, mapping).permute(1, 0, 2).contiguous()
                    if quadratic_form is not None:
                        quadratic_form = apply_mapping(quadratic_form.permute(1, 0, 2).contiguous(),
                                                       mapping).permute(1, 0, 2).contiguous()
            model = m_step(affiliation, quadratic_form)
            if mode not in (_lib.WEIGHT_TIED_TIME, _lib.WEIGHT_TIED):
                continue  # per-bin weights (the cACGMM fit with a graph): the M-step's own
            weight = tied_weight(affiliation, sal, mode, saliency_form)
            if F_all != F:  # sum over the other ranks' bins
                weight = parallel.mean_over_all_bins(weight, F, F_all, bin_group)
            model.weight = weight
    return model


# ---- the public building blocks (mixture_model_utils.py:7-306) -------------------------------------------------------

def log_pdf_to_affiliation(weight, log_pdf, source_activity_mask=None, affiliation_eps=0.):
    """The posterior of a mixture model from its log-pdfs (mixture_model_utils.py:7-55), on the device.

    log_pdf (..., K, N) float32 / float64 (other dtypes are taken as float64), any K and leading dims; weight any
    shape that broadcasts to log_pdf; source_activity_mask a bool array of such a shape.  Per column: subtract the
    max over K, exp, times weight, times mask, divide by max(sum over K, tiny of the dtype), clip to
    [eps, 1 - eps] if eps != 0.  Every operand is read in its own strides (pbb_affiliation_nd), the arithmetic is fp64
    and the result, of log_pdf's shape and dtype, is rounded once.  A weight or mask that would broadcast log_pdf to a
    larger shape raises ValueError, as the reference's in-place product does."""
    like = _nd.like_numpy(weight, log_pdf, source_activity_mask)
    lp = _nd.device_view(log_pdf)
    if lp.is_complex():
        raise TypeError(f'log_pdf must be real, got {lp.dtype}')
    nd = lp.dim()
    if nd < 2:
        raise np.exceptions.AxisError(-2, nd)
    w = _nd.device_view(weight).to(torch.float64)
    shapes = [tuple(w.shape), tuple(lp.shape)]
    m = None
    if source_activity_mask is not None:
        m = _nd.device_view(source_activity_mask, floating=False)
        shapes.append(tuple(m.shape))
    np.broadcast_shapes(*shapes)  # ValueError for incompatible shapes, as np.broadcast_arrays

    def check_fits(operand_shape):  # the reference's in-place products raise ValueError here
        bshape = np.broadcast_shapes(operand_shape, tuple(lp.shape))
        if bshape != tuple(lp.shape):
            raise ValueError(f'non-broadcastable output operand with shape {tuple(lp.shape)} doesn\'t match the '
                             f'broadcast shape {bshape}')
    check_fits(tuple(w.shape))  # affiliation *= weight
    if source_activity_mask is not None:
        assert m.dtype == torch.bool, (source_activity_mask.dtype if hasattr(source_activity_mask, 'dtype')
                                       else m.dtype)
        check_fits(tuple(m.shape))  # affiliation *= source_activity_mask
    shape = tuple(lp.shape)
    out = _device.empty(shape, lp.dtype)
    ws = _nd.broadcast_strides(w, shape)
    ms = _nd.broadcast_strides(m, shape) if m is not None else (0,) * nd
    ls, os_ = lp.stride(), out.stride()
    cols = [a for a in range(nd) if a != nd - 2]
    lay = _nd.layout([shape[a] for a in cols], *[[s[a] for a in cols] for s in (ls, ws, ms, os_)])
    cs = (ctypes.c_longlong * 4)(ls[-2], ws[-2], ms[-2], os_[-2])
    if out.numel():
        _device.call('pbb_affiliation_nd', lp, _nd.CODES[lp.dtype], w, m.view(torch.uint8) if m is not None else None,
                     lay, shape[-2], cs, float(affiliation_eps), out)
    return _device.to_host(out, like)


def log_pdf_to_affiliation_for_integration_models_with_inline_pa(weight, spatial_log_pdf, spectral_log_pdf,
                                                                 source_activity_mask=None, affiliation_eps=0.):
    """Inline permutation alignment of the integrated models (mixture_model_utils.py:58-130): per bin the spatial
    classes are re-paired with the spectral ones by the first permutation (itertools order) that maximises the
    auxiliary function, then log_pdf_to_affiliation of the paired sum.  spatial / spectral log-pdfs (F, K, T), weight
    any shape that broadcasts to (F, K, T) (read with zero strides, PBB_WEIGHT_BCAST), the mask (F, K, T).  This is
    pbb_log_pdf_to_affiliation with inline_pa = 1; it enumerates the K! permutations per bin, so K <= 6.  The result
    is float64, as in the reference."""
    like = _nd.like_numpy(weight, spatial_log_pdf, spectral_log_pdf, source_activity_mask)
    a = _device.to_device(spatial_log_pdf, torch.float64)
    b = _device.to_device(spectral_log_pdf, torch.float64)
    F, K, T = a.shape
    if K > MAX_INLINE_PA_K:
        raise NotImplementedError(
            f'log_pdf_to_affiliation_for_integration_models_with_inline_pa: need K <= {MAX_INLINE_PA_K} '
            f'(K! pairings per bin), got K = {K}')
    w = _nd.device_view(weight).to(torch.float64)
    if w.dim() > 3 or np.broadcast_shapes(tuple(w.shape), (F, K, T)) != (F, K, T):
        raise ValueError(f'weight of shape {tuple(w.shape)} does not broadcast to {(F, K, T)}')  # np.broadcast_to
    w3 = w.reshape((1,) * (3 - w.dim()) + tuple(w.shape))
    mode = _lib.WEIGHT_BCAST | sum(bit for bit, n in zip((1, 2, 4), w3.shape) if n != 1)
    w3 = w3.contiguous()
    act = None
    if source_activity_mask is not None:
        act = _device.to_device(source_activity_mask, torch.bool).expand(F, K, T).contiguous().view(torch.uint8)
    out = _device.empty((F, K, T), torch.float64)
    _device.call('pbb_log_pdf_to_affiliation', a, b, 1.0, 1.0, w3, mode, act, float(affiliation_eps), 1, F, K, T, out,
                 None)
    return _device.to_host(out, like)


def _promoted_float(aff_dtype, sal_dtype):
    """The dtype of affiliation * saliency in NumPy (float32 * bool stays float32), float32 or float64."""
    def np_dtype(d):
        return torch.empty(0, dtype=d).numpy().dtype if isinstance(d, torch.dtype) else np.dtype(d)
    return torch.float32 if np.result_type(np_dtype(aff_dtype), np_dtype(sal_dtype)) == np.float32 else torch.float64


def estimate_mixture_weight(affiliation, saliency=None, weight_constant_axis=-1):
    """The mixture weight (mixture_model_utils.py:133-203): an int axis equivalent to -2 gives np.full([K, 1], 1/K)
    (host); otherwise the mean over ``weight_constant_axis`` with keepdims, or, with a saliency (..., N), the sum
    over those axes of affiliation * saliency[..., None, :], L1-normalised over the classes (_unit_norm with ord=1,
    axis=-2, eps=1e-10, eps_style='where').  The sums run on the device in a fixed order (pbb_axis_sum): fp64,
    rounded once to the dtype NumPy returns; they are not NumPy's pairwise sums, so a result may differ from the
    reference by the rounding of a reordered sum (a few ulp times the number of summed elements)."""
    like = _nd.like_numpy(affiliation, saliency)
    if not _device.is_tensor(affiliation):
        affiliation = np.asarray(affiliation)
    ndim = affiliation.ndim
    if isinstance(weight_constant_axis, int) and weight_constant_axis % ndim - ndim == -2:
        K = affiliation.shape[-2]
        weight = np.full([K, 1], 1 / K)
        return weight if like else _device.to_device(weight)
    elif isinstance(weight_constant_axis, list):
        weight_constant_axis = tuple(weight_constant_axis)
    axes = tuple(sorted(normalize_axis_tuple(weight_constant_axis, ndim)))
    x = _nd.device_view(affiliation)
    if saliency is None:
        weight = _nd.axis_sum(x, axes, True, divide_by_count=True)
    else:
        sal_dtype = saliency.dtype if _device.is_tensor(saliency) else np.asarray(saliency).dtype
        s = _nd.device_view(saliency)
        out_dtype = _promoted_float(x.dtype, sal_dtype)
        mul = s.to(torch.float64)[..., None, :]
        nd_all = max(x.dim(), mul.dim())
        ax = tuple(sorted(normalize_axis_tuple(weight_constant_axis, nd_all)))
        total = _nd.axis_sum(x, ax, True, multiplier=mul, out_dtype=out_dtype)
        weight = _unit_norm(total, ord=1, axis=-2, eps=1e-10, eps_style='where')
    return _device.to_host(weight, like)


def apply_inline_permutation_alignment(affiliation, *, quadratic_form=None, weight_constant_axis, aligner):
    """The inline permutation alignment step of the EM loops (mixture_model_utils.py:264-306): the aligner's
    calculate_mapping of the (K, F, T) affiliation, applied to the affiliation and, if given, to the quadratic form.
    affiliation / quadratic_form (F, K, T).  Both aligner steps run on the device."""
    message = (
        f'Inline permutation alignment reduces mismatch between frequency '
        f'independent mixtures weights and a frequency independent '
        f'observation model. Therefore, we require `affiliation.ndim == 3` '
        f'({tuple(affiliation.shape)}) and a corresponding '
        f'`weight_constant_axis` ({weight_constant_axis}).'
    )
    assert affiliation.ndim == 3, message
    assert weight_constant_axis in ((-3,), (-3, -1), -3), message

    def swap(x):
        return x.permute(1, 0, 2) if _device.is_tensor(x) else np.transpose(x, (1, 0, 2))
    affiliation = swap(affiliation)
    mapping = aligner.calculate_mapping(affiliation)
    affiliation = swap(aligner.apply_mapping(affiliation, mapping))
    if quadratic_form is None:
        return affiliation
    quadratic_form = swap(aligner.apply_mapping(swap(quadratic_form), mapping))
    return affiliation, quadratic_form
