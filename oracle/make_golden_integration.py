"""Generate tests/golden/integration_shapes.npz from the UNMODIFIED reference (oracle/ref_shim.py): GCACGMM and
VMFCACGMM fits (gcacgmm.py:38-333, vmfcacgmm.py:34-301) at the shapes the fixtures of make_golden.make_gcacgmm do
not reach -- K = 1, 2, 4, 6 (the inline pairing at K = 4 and 6), E = 1, 16, 33, 64, D = 2, 6, T = 255, 257, 700 --
with every weight layout, both covariance types, a fixed covariance, affiliation_eps = 0 and a saliency with zero
frames.

Run where a reference checkout or oracle/_ref is present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_integration [OUT_DIR]

The fixture stores the reference's outputs ('<case>_<output>') and, to keep it small, only a fingerprint of each
seeded input ('<problem>_fingerprint_<input>'): the tests regenerate the inputs with ``problem_inputs`` (NumPy's legacy
RandomState streams, stable across versions) and ``fixture_inputs`` checks them against the fingerprints, so the tests
need neither the reference nor a run of this script.  Each inline-pairing case is checked
here to keep every bin's choice clear of a tie (oracle/integration_oracle.py, relative margin > 1e-6), so a device
that sums in another order still picks the same pairing.
"""
import os
import sys

import numpy as np

from . import ref_shim, synth
from . import integration_oracle as IO

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
ITERATIONS = 4

# name -> (F, T, D, E, K)
PROBLEMS = {
    'k1': (3, 255, 2, 1, 1),
    'k2': (3, 257, 6, 33, 2),
    'k4': (3, 257, 2, 16, 4),
    'k6': (2, 700, 6, 64, 6),
}

# name -> (problem, spectral model, keyword arguments of the trainer); 'saliency' / 'fixed_covariance' name inputs
CASES = {
    'k1_spherical': ('k1', 'gaussian', dict()),
    'k2_diagonal_kt': ('k2', 'gaussian', dict(covariance_type='diagonal', weight_constant_axis=(-3,))),
    'k2_spherical_const': ('k2', 'gaussian', dict(weight_constant_axis=(-3, -2, -1))),
    'k2_vmf_k_eps0': ('k2', 'vmf', dict(weight_constant_axis=(-3, -1), affiliation_eps=0.)),
    'k4_spherical_inline': ('k4', 'gaussian', dict(inline_permutation_alignment=True, spectral_weight=0.5)),
    'k4_fixed_k': ('k4', 'gaussian', dict(fixed_covariance='fixed_covariance', weight_constant_axis=(-3, -1))),
    'k4_diagonal_sal': ('k4', 'gaussian', dict(covariance_type='diagonal', saliency='saliency',
                                               spatial_weight=0.7, spectral_weight=1.3)),
    'k4_vmf_kt_inline': ('k4', 'vmf', dict(weight_constant_axis=(-3,), inline_permutation_alignment=True,
                                           max_concentration=50)),
    'k6_spherical_k_inline_eps0': ('k6', 'gaussian', dict(weight_constant_axis=(-3, -1), affiliation_eps=0.,
                                                          inline_permutation_alignment=True)),
    'k6_vmf_inline_sal': ('k6', 'vmf', dict(inline_permutation_alignment=True, saliency='saliency')),
}

# fixture key -> weight_constant_axis with -2 whose scalar weight the reference has to unsqueeze
ERROR_AXES = {'error_axes_m2': (-2,), 'error_axes_m3m2': (-3, -2), 'error_axes_m2m1': (-2, -1)}


def problem_inputs(name):
    """Seeded inputs of one problem: y (F, T, D), class-dependent embedding clouds (F, T, E) and the same scaled to
    unit norm (the von Mises-Fisher M-step fits the embeddings as given, vmfcacgmm.py:280-285), an initialisation
    (F, K, T), a saliency (F, T) with about 10 % zero frames and a spherical fixed covariance (K,)."""
    F, T, D, E, K = PROBLEMS[name]
    seed = sum(PROBLEMS[name])
    y, labels = synth.structured_stft(F, T, D, K, seed=seed)
    rng = np.random.RandomState(seed)
    centers = rng.randn(K, E) * 2.0
    embedding = centers[labels] + 0.7 * rng.randn(F, T, E)
    saliency = rng.uniform(0.3, 1.0, size=(F, T))
    saliency[rng.uniform(size=(F, T)) < 0.1] = 0.
    return dict(y=y, embedding=embedding, unit_embedding=embedding / np.linalg.norm(embedding, axis=-1, keepdims=True),
                init=synth.init_affiliation(F, K, T, seed=seed + 1), saliency=saliency,
                fixed_covariance=rng.uniform(0.5, 2.0, size=K))


def fingerprint(x):
    """Three weighted sums of |x| and of x.real: a regenerated input that differs in any element changes them."""
    a = np.asarray(x).ravel()
    ramp = np.arange(a.size) % 7 + 1.
    return np.array([np.sum(np.abs(a)), np.sum(ramp * np.abs(a)), np.sum(ramp * a.real)])


def fixture_inputs(g, problem):
    """The seeded inputs of ``problem``, checked against the fingerprints stored in the fixture ``g``."""
    d = problem_inputs(problem)
    for k, v in d.items():
        np.testing.assert_allclose(fingerprint(v), g[f'{problem}_fingerprint_{k}'], rtol=1e-13,
                                   err_msg=f'{problem} {k}: regenerated input differs from the fixture')
    return d


def resolve(inputs, kw):
    """The trainer's keyword arguments with the named inputs filled in."""
    return {k: inputs[v] if k in ('saliency', 'fixed_covariance') else v for k, v in kw.items()}


def embedding_of(inputs, spectral):
    return inputs['embedding' if spectral == 'gaussian' else 'unit_embedding']


def make_integration(ref, out_dir=OUT):
    import pb_bss.distribution.gcacgmm as G
    import pb_bss.distribution.vmfcacgmm as V
    out = dict(iterations=ITERATIONS)
    inputs = {name: problem_inputs(name) for name in PROBLEMS}
    for name, d in inputs.items():
        out.update({f'{name}_fingerprint_{k}': fingerprint(v) for k, v in d.items()})
    for name, (problem, spectral, kw) in CASES.items():
        d = inputs[problem]
        kw = resolve(d, kw)
        emb = embedding_of(d, spectral)
        trainer = G.GCACGMMTrainer() if spectral == 'gaussian' else V.VMFCACGMMTrainer()
        model = trainer.fit(d['y'], emb, initialization=d['init'], iterations=ITERATIONS, **kw)
        out[f'{name}_weight'] = np.asarray(model.weight)
        if spectral == 'gaussian':
            out[f'{name}_mean'] = model.gaussian.mean
            out[f'{name}_gcov'] = model.gaussian.covariance
        else:
            out[f'{name}_mean'] = model.vmf.mean
            out[f'{name}_concentration'] = model.vmf.concentration
        out[f'{name}_eigenvalues'] = model.cacg.covariance_eigenvalues
        out[f'{name}_covariance'] = model.cacg.covariance
        out[f'{name}_affiliation'] = model.predict(d['y'], emb)
        assert all(np.isfinite(v).all() for k, v in out.items() if k.startswith(name + '_')), name
        if kw.get('inline_permutation_alignment'):
            o = IO.integrated_fit(d['y'], emb, d['init'], ITERATIONS, spectral, **kw)
            assert o['min_margin'] > 1e-6, (name, o['min_margin'])
    # a constant weight 1 / K that the reference cannot unsqueeze to the axes given (gcacgmm.py:109, utils.py:324-329):
    # the type of the exception of the first E-step, '' if none
    d = inputs['k2']
    for key, axes in ERROR_AXES.items():
        try:
            G.GCACGMMTrainer().fit(d['y'], d['embedding'], initialization=d['init'], iterations=2,
                                   weight_constant_axis=axes)
            out[key] = np.array('')
        except Exception as e:  # noqa: BLE001 -- the type is the fixture
            out[key] = np.array(type(e).__name__)
    np.savez_compressed(os.path.join(out_dir, 'integration_shapes.npz'), **out)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    os.makedirs(out, exist_ok=True)
    make_integration(ref_shim.load(), out)


if __name__ == '__main__':
    main()
