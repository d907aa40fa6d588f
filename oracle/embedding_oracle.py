"""NumPy restatement of the embedding mixture models of pb_bss (TEST INFRASTRUCTURE, see oracle/__init__.py):
Gaussian / GaussianTrainer (pb_bss/distribution/gaussian.py:19-193), GMM / GMMTrainer (gmm.py:16-173),
VonMisesFisher / VonMisesFisherTrainer (von_mises_fisher.py:31-144) and VMFMM / VMFMMTrainer (vmfmm.py:14-172).

Every function names the reference lines it follows; the einsum expressions and LAPACK entry points are those of the
reference (and of sklearn's precision Cholesky helpers it calls).  The posterior and the mixture weights are the
restatements of oracle/pb_bss_oracle.py.

Parity: PINNED against the live reference, see oracle/make_golden_embedding.py and
tests/test_embedding_oracle.py.
"""
import numpy as np
import scipy.linalg
import scipy.special

from .pb_bss_oracle import estimate_mixture_weight, log_pdf_to_affiliation


ILL_DEFINED = ('Fitting the mixture model failed because some components have ill-defined empirical '
               'covariance (for instance caused by singleton or collapsed samples).')


def precision_cholesky_full(covariance):
    """sklearn's _compute_precision_cholesky(cov, 'full') and _compute_log_det_cholesky as
    pb_bss/distribution/gaussian.py:26-34 calls them: cov (..., D, D) -> (U, log_det)."""
    D = covariance.shape[-1]
    c = np.reshape(covariance, (-1, D, D))
    pc = np.empty_like(c)
    for k, ck in enumerate(c):
        try:
            L = scipy.linalg.cholesky(ck, lower=True)
        except scipy.linalg.LinAlgError:
            raise ValueError(ILL_DEFINED)
        pc[k] = scipy.linalg.solve_triangular(L, np.eye(D), lower=True).T
    log_det = np.sum(np.log(pc.reshape(len(c), -1)[:, ::D + 1]), 1)
    return np.reshape(pc, covariance.shape), np.reshape(log_det, covariance.shape[:-2])


def precision_cholesky_diag(covariance):
    """sklearn's _compute_precision_cholesky(cov, 'diag') (gaussian.py:66-71, 103-108)."""
    if np.any(np.less_equal(covariance, 0.0)):
        raise ValueError(ILL_DEFINED)
    return 1. / np.sqrt(covariance)


def gaussian_log_pdf(y, mean, precision_cholesky, log_det):
    """Gaussian.log_pdf (gaussian.py:36-56).  The einsum '...dD,...nD->...nd' contracts the upper-triangular U as U d
    (sklearn's density uses U^T d): the quadratic form is d^T U^T U d, equal to d^T Sigma^-1 d for a diagonal Sigma
    only.  The same expression serves DiagonalGaussian (gaussian.py:73-93), where d runs over the classes."""
    D = mean.shape[-1]
    difference = y - mean[..., None, :]
    white_x = np.einsum('...dD,...nD->...nd', precision_cholesky, difference)
    return (-1 / 2 * D * np.log(2 * np.pi) + log_det[..., None]
            - 1 / 2 * np.einsum('...nd,...nd->...n', white_x, white_x))


def spherical_log_pdf(y, mean, precision_cholesky, log_det):
    """SphericalGaussian.log_pdf (gaussian.py:110-130)."""
    D = mean.shape[-1]
    difference = y - mean[..., None, :]
    white_x = np.einsum('...,...nd->...nd', precision_cholesky, difference)
    return (-1 / 2 * D * np.log(2 * np.pi) + log_det[..., None]
            - 1 / 2 * np.einsum('...nd,...nd->...n', white_x, white_x))


def gaussian_model(mean, covariance, covariance_type):
    """Gaussian / DiagonalGaussian / SphericalGaussian.__post_init__ (gaussian.py:26-34, 66-71, 103-108) as a dict."""
    D = mean.shape[-1]
    if covariance_type == 'full':
        pc, ld = precision_cholesky_full(covariance)
    elif covariance_type == 'diagonal':
        pc = precision_cholesky_diag(covariance)
        ld = np.sum(np.log(np.reshape(pc, (-1, D))), axis=1)
    else:
        pc = precision_cholesky_diag(covariance)
        ld = D * np.log(np.reshape(pc, (-1,)))
    return dict(type=covariance_type, mean=mean, covariance=covariance, precision_cholesky=pc, log_det=ld)


def gaussian_model_log_pdf(model, y):
    f = spherical_log_pdf if model['type'] == 'spherical' else gaussian_log_pdf
    return f(y, model['mean'], model['precision_cholesky'], model['log_det'])


def gaussian_fit(y, saliency, covariance_type):
    """GaussianTrainer._fit (gaussian.py:152-193) -> gaussian_model dict."""
    dimension = y.shape[-1]
    if saliency is None:
        denominator = np.array(y.shape[-2])
        mean = np.einsum('...nd->...d', y)
    else:
        denominator = np.maximum(np.einsum('...n->...', saliency), np.finfo(y.dtype).tiny)
        mean = np.einsum('...n,...nd->...d', saliency, y)
    mean = mean / denominator[..., None]
    difference = y - mean[..., None, :]
    if covariance_type == 'full':
        operation, denominator = '...nd,...nD->...dD', denominator[..., None, None]
    elif covariance_type == 'diagonal':
        operation, denominator = '...nd,...nd->...d', denominator[..., None]
    elif covariance_type == 'spherical':
        operation, denominator = '...nd,...nd->...', denominator * dimension
    else:
        raise ValueError(f"Unknown covariance type '{covariance_type}'.")
    if saliency is None:
        covariance = np.einsum(operation, difference, difference)
    else:
        covariance = np.einsum('...n,' + operation, saliency, difference, difference)
    covariance = covariance / denominator
    return gaussian_model(mean, covariance, covariance_type)


def gmm_predict(x, model):
    """GMM.predict (gmm.py:21-25)."""
    return log_pdf_to_affiliation(model['weight'], gaussian_model_log_pdf(model['gaussian'], x[..., None, :, :]))


def gmm_fit(y, initialization, iterations=100, *, saliency=None, weight_constant_axis=(-1,),
            covariance_type='full', fixed_covariance=None):
    """GMMTrainer.fit / _fit / _m_step (gmm.py:33-173) from an explicit initialization -> dict(weight, gaussian)."""
    if saliency is None:
        saliency = np.ones_like(initialization[..., 0, :])
    affiliation = initialization
    model = None
    for _ in range(iterations):
        if model is not None:
            affiliation = gmm_predict(y, model)
        weight = estimate_mixture_weight(affiliation, saliency, weight_constant_axis)
        gaussian = gaussian_fit(y[..., None, :, :], affiliation * saliency[..., None, :], covariance_type)
        if fixed_covariance is not None:
            assert fixed_covariance.shape == gaussian['covariance'].shape
            gaussian = gaussian_model(gaussian['mean'], fixed_covariance, covariance_type)
        model = dict(weight=weight, gaussian=gaussian)
    return model


def _unit_rows(y):
    return y / np.maximum(np.linalg.norm(y, axis=-1, keepdims=True), np.finfo(y.dtype).tiny)


def vmf_log_norm(concentration, D):
    """VonMisesFisher.log_norm (von_mises_fisher.py:35-45)."""
    return ((D / 2) * np.log(2 * np.pi) + np.log(scipy.special.ive(D / 2 - 1, concentration))
            + (np.abs(concentration) - (D / 2 - 1) * np.log(concentration)))


def vmf_log_pdf(y, mean, concentration):
    """VonMisesFisher.log_pdf (von_mises_fisher.py:65-79)."""
    y = _unit_rows(y)
    result = np.einsum('...d,...d', y, mean[..., None, :])
    result = result * concentration[..., None]
    return result - vmf_log_norm(concentration, mean.shape[-1])[..., None]


def vmf_fit(y, saliency, min_concentration=1e-10, max_concentration=500):
    """VonMisesFisherTrainer._fit (von_mises_fisher.py:122-144) of unit-norm y -> (mean, concentration)."""
    D = y.shape[-1]
    if saliency is None:
        saliency = np.ones(y.shape[:-1])
    r = np.einsum('...n,...nd->...d', saliency, y)                       # Banerjee2005vMF eq. 2.4
    norm = np.linalg.norm(r, axis=-1)
    mean = r / np.maximum(norm, np.finfo(y.dtype).tiny)[..., None]
    r_bar = norm / np.sum(saliency, axis=-1)                             # eq. 2.5
    concentration = (r_bar * D - r_bar ** 3) / (1 - r_bar ** 2)          # eq. 4.4
    return mean, np.clip(concentration, min_concentration, max_concentration)


def vmfmm_predict(y, model):
    """VMFMM.predict (vmfmm.py:19-37)."""
    y = _unit_rows(y)
    return log_pdf_to_affiliation(model['weight'], vmf_log_pdf(y[..., None, :, :], model['mean'],
                                                               model['concentration']))


def vmfmm_fit(y, initialization, iterations=100, saliency=None, weight_constant_axis=(-1,),
              min_concentration=1e-10, max_concentration=500):
    """VMFMMTrainer.fit / _fit / _m_step (vmfmm.py:43-172) from an explicit initialization
    -> dict(weight, mean, concentration)."""
    y = _unit_rows(y)
    if saliency is None:
        saliency = np.ones_like(initialization[..., 0, :])
    affiliation = initialization
    model = None
    for _ in range(iterations):
        if model is not None:
            affiliation = vmfmm_predict(y, model)
        weight = estimate_mixture_weight(affiliation, saliency, weight_constant_axis)
        mean, concentration = vmf_fit(y[..., None, :, :], affiliation * saliency[..., None, :],
                                      min_concentration, max_concentration)
        model = dict(weight=weight, mean=mean, concentration=concentration)
    return model
