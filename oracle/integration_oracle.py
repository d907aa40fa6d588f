"""NumPy restatement of the integrated spatial + spectral mixture models of pb_bss (TEST INFRASTRUCTURE, see
oracle/__init__.py): GCACGMM / GCACGMMTrainer (pb_bss/distribution/gcacgmm.py:38-333) and VMFCACGMM /
VMFCACGMMTrainer (vmfcacgmm.py:34-301).

The cACG pieces are those of oracle/pb_bss_oracle.py, the Gaussian and von Mises-Fisher pieces those of
oracle/embedding_oracle.py.  This module adds the integration logic: the inline pairing of spatial and spectral
classes (mixture_model_utils.py:58-130), the class-weight layouts, the fixed covariance and the spatial / spectral
weights.  Every function names the reference lines it follows.

Parity: PINNED against the live reference, see oracle/make_golden_integration.py and
tests/test_integration_oracle.py.
"""
import itertools

import numpy as np

from . import embedding_oracle as EO
from .pb_bss_oracle import (cacg_covariance, cacg_from_covariance, cacg_log_pdf, log_pdf_to_affiliation,
                            normalize_observation_cacg)


def unsqueeze(weight, axes):
    """pb_bss/utils.py:306-336: the squeezed weight back to a shape that broadcasts against (F, K, T)."""
    weight = np.array(weight)
    ndim = weight.ndim + len(axes)
    if any(not -ndim <= a < ndim for a in axes):      # :326-329, e.g. the scalar 1 / K with axes (-2,)
        raise IndexError(weight.shape, axes)
    axes = sorted(a % ndim for a in axes)
    for a in axes:
        weight = np.expand_dims(weight, a)
    return weight


def class_weight(masked_affiliation, weight_constant_axis):
    """The mixture weight of the integrated M-step (gcacgmm.py:283-291, vmfcacgmm.py:266-274): 1 / K when -2 is one of
    the axes, else the masked affiliations summed over the axes, L1-normalised over the classes, squeezed."""
    K = masked_affiliation.shape[-2]
    if -2 in weight_constant_axis:
        return 1 / K
    weight = np.sum(masked_affiliation, axis=weight_constant_axis, keepdims=True)
    weight /= np.sum(weight, axis=-2, keepdims=True)
    return np.squeeze(weight, axis=weight_constant_axis)


def inline_pa_affiliation(weight, spatial_log_pdf, spectral_log_pdf, affiliation_eps=0.):
    """log_pdf_to_affiliation_for_integration_models_with_inline_pa (mixture_model_utils.py:58-130) without a source
    activity mask.  Per bin, the first of itertools.permutations(range(K)) that maximises
    sum_{k,t} softmax_k(log_pdf) * log_pdf with log_pdf = spatial[perm] + spectral.

    Returns (affiliation (F, K, T), chosen permutation (F, K), margin (F,)): the margin is the gap between the best
    and the second-best auxiliary value over max |auxiliary value| of the bin (inf for K = 1)."""
    F, K, T = spatial_log_pdf.shape
    permutations = np.asarray(list(itertools.permutations(range(K))))
    weight = np.broadcast_to(weight, spatial_log_pdf.shape)
    affiliation = np.zeros((F, K, T), dtype=np.float64)
    chosen = np.zeros((F, K), dtype=np.int64)
    margin = np.full(F, np.inf)
    for f in range(F):
        aux = np.empty(len(permutations))
        for i, permutation in enumerate(permutations):                            # :93-115
            log_pdf = spatial_log_pdf[f, permutation, :] + spectral_log_pdf[f, :, :]
            candidate = log_pdf - np.max(log_pdf, axis=-2, keepdims=True)
            np.exp(candidate, out=candidate)
            candidate /= np.maximum(np.sum(candidate, axis=-2, keepdims=True), np.finfo(np.float64).tiny)
            aux[i] = np.sum(candidate * log_pdf, axis=(-2, -1))
        best = int(np.argmax(aux))                                               # first maximum, like the strict >
        chosen[f] = permutations[best]
        if len(aux) > 1:
            second = np.max(np.delete(aux, best))
            margin[f] = (aux[best] - second) / np.max(np.abs(aux))
        affiliation[f] = log_pdf_to_affiliation(                                 # :117-128
            weight[f], spatial_log_pdf[f, chosen[f], :] + spectral_log_pdf[f], affiliation_eps=affiliation_eps)
    return affiliation, chosen, margin


def _spectral_log_pdf_fkt(spectral, embedding):
    """The spectral model's log pdf of the (F*T, E) embeddings as (F, K, T) (gcacgmm.py:92-97, vmfcacgmm.py:72-77)."""
    F, T, E = embedding.shape
    embedding_ = np.reshape(embedding, (1, F * T, E))
    if 'concentration' in spectral:
        log_pdf = EO.vmf_log_pdf(embedding_, spectral['mean'], spectral['concentration'])
    else:
        log_pdf = EO.gaussian_model_log_pdf(spectral, embedding_)
    K = log_pdf.shape[0]
    return np.transpose(np.reshape(log_pdf, (K, F, T)), (1, 0, 2))


def integrated_e_step(z, embedding, model, affiliation_eps=0., inline_permutation_alignment=False):
    """GCACGMM._predict (gcacgmm.py:70-128) / VMFCACGMM._predict (vmfcacgmm.py:57-97) of unit-norm observations
    z (F, D, T).  Returns (affiliation, quadratic_form, chosen permutation or None, margin or None)."""
    spatial, quadratic_form = cacg_log_pdf(z[..., None, :, :], model['eigenvectors'], model['eigenvalues'])
    spectral = _spectral_log_pdf_fkt(model['spectral'], embedding)
    weight = unsqueeze(model['weight'], model['weight_constant_axis'])
    if inline_permutation_alignment:
        affiliation, chosen, margin = inline_pa_affiliation(
            weight, model['spatial_weight'] * spatial, model['spectral_weight'] * spectral, affiliation_eps)
        return affiliation, quadratic_form, chosen, margin
    affiliation = log_pdf_to_affiliation(
        weight, model['spatial_weight'] * spatial + model['spectral_weight'] * spectral,
        affiliation_eps=affiliation_eps)
    return affiliation, quadratic_form, None, None


def _spectral_fit(embedding, masked_affiliation, spectral, covariance_type, fixed_covariance, min_concentration,
                  max_concentration):
    """GaussianTrainer._fit (gcacgmm.py:293-310, with the fixed covariance) or VonMisesFisherTrainer._fit
    (vmfcacgmm.py:276-285) of the (1, F*T, E) embeddings with the (K, F*T) masked affiliations."""
    F, K, T = masked_affiliation.shape
    embedding_ = np.reshape(embedding, (1, F * T, embedding.shape[-1]))
    masked_ = np.reshape(np.transpose(masked_affiliation, (1, 0, 2)), (K, F * T))   # 'fkt->k,ft'
    if spectral == 'vmf':
        mean, concentration = EO.vmf_fit(embedding_, masked_, min_concentration, max_concentration)
        return dict(mean=mean, concentration=concentration)
    gaussian = EO.gaussian_fit(embedding_, masked_, covariance_type)
    if fixed_covariance is not None:
        assert fixed_covariance.shape == gaussian['covariance'].shape
        gaussian = EO.gaussian_model(gaussian['mean'], fixed_covariance, covariance_type)
    return gaussian


def integrated_fit(y, embedding, initialization, iterations, spectral='gaussian', *, saliency=None, hermitize=True,
                   covariance_norm='eigenvalue', eigenvalue_floor=1e-10, covariance_type='spherical',
                   fixed_covariance=None, min_concentration=1e-10, max_concentration=500, affiliation_eps=1e-10,
                   weight_constant_axis=(-1,), spatial_weight=1., spectral_weight=1.,
                   inline_permutation_alignment=False):
    """GCACGMMTrainer.fit (gcacgmm.py:131-227, spectral='gaussian') or VMFCACGMMTrainer.fit (vmfcacgmm.py:101-199,
    spectral='vmf') from an explicit initialization (F, K, T) -> model dict.  With the inline pairing the dict also
    holds 'min_margin', the smallest relative margin of any bin's choice over all E-steps."""
    z = normalize_observation_cacg(y)                       # (F, D, T); max(norm, tiny) == 'where' for norm > 0
    if saliency is None:
        saliency = np.ones_like(initialization[..., 0, :])
    affiliation = initialization
    quadratic_form = np.ones_like(initialization)
    min_margin = np.inf
    model = None
    for _ in range(iterations):
        if model is not None:
            affiliation, quadratic_form, _, margin = integrated_e_step(
                z, embedding, model, affiliation_eps, inline_permutation_alignment)
            if margin is not None:
                min_margin = min(min_margin, margin.min())
        masked = affiliation * saliency[..., None, :]                              # gcacgmm.py:280-281
        cov = cacg_covariance(z[..., None, :, :], masked, quadratic_form, hermitize)
        eigenvectors, eigenvalues = cacg_from_covariance(cov, eigenvalue_floor, covariance_norm)
        model = dict(
            weight=class_weight(masked, weight_constant_axis), weight_constant_axis=weight_constant_axis,
            spectral=_spectral_fit(embedding, masked, spectral, covariance_type, fixed_covariance, min_concentration,
                                   max_concentration),
            eigenvectors=eigenvectors, eigenvalues=eigenvalues,
            spatial_weight=spatial_weight, spectral_weight=spectral_weight)
    if inline_permutation_alignment:
        model['min_margin'] = min_margin
    return model


def integrated_predict(y, embedding, model):
    """GCACGMM.predict (gcacgmm.py:46-68) / VMFCACGMM.predict (vmfcacgmm.py:44-55): affiliation_eps 0, no pairing."""
    return integrated_e_step(normalize_observation_cacg(y), embedding, model)[0]
