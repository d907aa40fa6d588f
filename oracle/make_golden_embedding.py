"""Generate tests/golden/gmm.npz and tests/golden/vmfmm.npz from the UNMODIFIED reference (oracle/ref_shim.py):
the embedding mixture models GMM / Gaussian and VMFMM / von Mises-Fisher.

Run where a reference checkout or oracle/_ref is present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_embedding [OUT_DIR]

Every fixture stores the inputs next to the reference's outputs, so the tests need neither the reference nor this
script.  Inputs are float64 class-dependent clouds with explicit initialisations, 5 EM iterations.
"""
import os
import sys

import numpy as np

from . import ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def _embedding_clouds(rng, lead, N, E, K):
    """Class-dependent float64 embedding clouds (..., N, E) and a normalised initialisation (..., K, N)."""
    centers = rng.randn(*lead, K, E) * 2.0
    labels = rng.randint(0, K, size=(*lead, N))
    idx = np.indices(labels.shape)[:-1]
    y = centers[(*idx, labels)] + rng.randn(*lead, N, E) * rng.uniform(0.5, 1.0, size=E)
    init = rng.uniform(size=(*lead, K, N))
    init /= init.sum(-2, keepdims=True)
    return y, init


def make_embedding(ref, out_dir=OUT):
    """GMM / Gaussian (gmm.py:16-173, gaussian.py:19-193) and VMFMM / von Mises-Fisher (vmfmm.py:14-172,
    von_mises_fisher.py:31-144) over embeddings: covariance types, independent dims, weight layouts, saliency."""
    import pb_bss.distribution.gaussian as RG
    import pb_bss.distribution.gmm as RM
    import pb_bss.distribution.vmfmm as RV
    import pb_bss.distribution.von_mises_fisher as RF
    rng = np.random.RandomState(23)
    N, E, K, it = 300, 5, 3, 5
    y0, init0 = _embedding_clouds(rng, (), N, E, K)
    yb, initb = _embedding_clouds(rng, (3,), N, E, K)
    sal = rng.uniform(0.2, 1.0, size=N)
    sal[rng.uniform(size=N) < 0.1] = 0.0                        # zero-saliency observations
    a = rng.randn(K, E, E)
    fixed = np.einsum('kde,kfe->kdf', a, a) / E + 0.5 * np.eye(E)
    out = dict(y0=y0, init0=init0, yb=yb, initb=initb, saliency=sal, fixed_covariance=fixed, iterations=it)
    cases = {
        'full': (y0, init0, dict()),
        'full_b3': (yb, initb, dict()),
        'diagonal': (y0, init0, dict(covariance_type='diagonal')),
        'spherical': (y0, init0, dict(covariance_type='spherical')),
        'full_fixed': (y0, init0, dict(fixed_covariance=fixed)),
        'full_sal': (y0, init0, dict(saliency=sal)),
        'w_m2': (y0, init0, dict(weight_constant_axis=-2)),
        'w_t2_sal': (yb, initb, dict(weight_constant_axis=(-2,), saliency=np.broadcast_to(sal, (3, N)).copy())),
    }
    for name, (y, init, kw) in cases.items():
        model = RM.GMMTrainer().fit(y, initialization=init, iterations=it, **kw)
        out[f'{name}_weight'] = np.asarray(model.weight)
        out[f'{name}_mean'] = model.gaussian.mean
        out[f'{name}_covariance'] = model.gaussian.covariance
        out[f'{name}_affiliation'] = model.predict(y)
    # Gaussian.log_pdf of a given full model, and single GaussianTrainer.fit calls
    g = RG.Gaussian(mean=out['full_b3_mean'], covariance=out['full_b3_covariance'])
    out['logpdf_y'] = yb[:, None, :40]
    out['logpdf'] = g.log_pdf(yb[:, None, :40])
    for ct in ('full', 'diagonal', 'spherical'):
        fit = RG.GaussianTrainer().fit(yb, saliency=np.broadcast_to(sal, (3, N)).copy(), covariance_type=ct)
        out[f'fit_{ct}_mean'] = fit.mean
        out[f'fit_{ct}_covariance'] = fit.covariance
    fit = RG.GaussianTrainer().fit(y0)
    out['fit_nosal_mean'], out['fit_nosal_covariance'] = fit.mean, fit.covariance
    np.savez_compressed(os.path.join(out_dir, 'gmm.npz'), **out)

    vout = dict(y0=y0, init0=init0, yb=yb[:2], initb=initb[:2], saliency=sal, iterations=it)
    vcases = {
        'vmf': (y0, init0, dict()),
        'vmf_b2_maxc': (yb[:2], initb[:2], dict(max_concentration=3.)),
        'vmf_sal_t2': (y0, init0, dict(saliency=sal, weight_constant_axis=(-2,))),
    }
    for name, (y, init, kw) in vcases.items():
        model = RV.VMFMMTrainer().fit(y, initialization=init, iterations=it, **kw)
        vout[f'{name}_weight'] = np.asarray(model.weight)
        vout[f'{name}_mean'] = model.vmf.mean
        vout[f'{name}_concentration'] = model.vmf.concentration
        vout[f'{name}_affiliation'] = model.predict(y)
    fit = RF.VonMisesFisherTrainer().fit(yb, saliency=np.broadcast_to(sal, (3, N)).copy())
    vout['fit_mean'], vout['fit_concentration'] = fit.mean, fit.concentration
    np.savez_compressed(os.path.join(out_dir, 'vmfmm.npz'), **vout)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    os.makedirs(out, exist_ok=True)
    make_embedding(ref_shim.load(), out)


if __name__ == '__main__':
    main()
