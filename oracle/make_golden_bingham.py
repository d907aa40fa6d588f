"""Generate tests/golden/cbmm*.npz from the UNMODIFIED reference (oracle/ref_shim.py): the complex Bingham
distribution and mixture model (pb_bss/distribution/complex_bingham.py, cbmm.py).

Run where a reference checkout or oracle/_ref is present:

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_bingham [OUT_DIR]

Every fixture stores the inputs next to the reference's outputs, so the tests need neither the reference nor this
script.  The reference is slow (scipy least squares per bin and class), so the problems are small.
"""
import os
import sys

import numpy as np

from . import ref_shim, synth

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def _model(model):
    cb = model.complex_bingham
    return dict(weight=np.asarray(model.weight), V=cb.covariance_eigenvectors, lam=cb.covariance_eigenvalues)


def make_bingham(out_dir=OUT):
    import pb_bss.distribution.cbmm as RC
    import pb_bss.distribution.complex_bingham as RB
    from pb_bss.distribution.mixture_model_utils import log_pdf_to_affiliation
    pa = ref_shim.load().permutation_alignment
    T = RB.ComplexBinghamTrainer
    out = {}
    # known answers of find_eigenvalues_v3 and norm (complex_bingham.py:83-164, :304-425)
    s6 = np.array([5.15996555e-04, 6.28805516e-04, 1.37554184e-03, 1.53621463e-02, 3.74437619e-02, 9.44673748e-01])
    out['known_s2'] = np.array([.9, .1])
    out['known_lam2'] = T.find_eigenvalues_v3(out['known_s2'])
    out['known_s6'] = s6
    out['known_lam6'] = T.find_eigenvalues_v3(s6)
    out['known_lam6_mc500'] = T.find_eigenvalues_v3(s6, max_concentration=500)
    out['known_norm_lam'] = np.array([.8, .92679492, 1.27320508])
    out['known_norm'] = RB.ComplexBingham(None, out['known_norm_lam']).norm()
    # single M-steps from given affiliations, D = 2..6 (cbmm.py:215-237)
    for D in range(2, 7):
        F, N, K = 3, 60, 2
        y = synth.structured_stft(F, N, D, K, seed=30 + D)[0]
        aff = synth.init_affiliation(F, K, N, seed=D)
        z = RB.normalize_observation(y)
        m = RC.CBMMTrainer().fit(y, initialization=aff, iterations=1)
        scat = np.einsum('fkn,fnd,fnD->fkdD', aff, z, z.conj()) / aff.sum(-1)[..., None, None]
        s_eig = np.linalg.eigvalsh((scat + np.swapaxes(scat.conj(), -1, -2)) / 2)
        lp = m.complex_bingham.log_pdf(z[:, None])
        out.update({f'mstep_d{D}_y': y, f'mstep_d{D}_aff': aff, f'mstep_d{D}_scatter_eig': s_eig,
                    f'mstep_d{D}_log_pdf': lp,
                    f'mstep_d{D}_posterior': log_pdf_to_affiliation(m.weight, lp, None, 0),
                    **{f'mstep_d{D}_{k}': v for k, v in _model(m).items()}})
    np.savez_compressed(os.path.join(out_dir, 'cbmm_steps.npz'), **out)

    # predict from a reference model, fits on structured data, options
    fits = {}
    y, _ = synth.structured_stft(4, 100, 4, 2, seed=51)
    init = synth.init_affiliation(4, 2, 100, seed=52)
    fits['y'], fits['init'] = y, init
    for it in (2, 5):
        m = RC.CBMMTrainer().fit(y, initialization=init, iterations=it)
        fits.update({f'fit{it}_{k}': v for k, v in _model(m).items()})
        fits[f'fit{it}_affiliation'] = m.predict(y)
        fits[f'fit{it}_affiliation_eps'] = m.predict(y, affiliation_eps=1e-3)
    sal = np.random.RandomState(53).uniform(0.2, 1.0, size=(4, 100))
    fits['saliency'] = sal
    options = {'sal': dict(saliency=sal), 'mc5': dict(), 'eps': dict(affiliation_eps=1e-2)}
    for name, kw in options.items():
        tr = RC.CBMMTrainer(max_concentration=5.) if name == 'mc5' else RC.CBMMTrainer()
        m = tr.fit(y, initialization=init, iterations=2, **kw)
        fits.update({f'{name}_{k}': v for k, v in _model(m).items()})
        fits[f'{name}_affiliation'] = m.predict(y)
    # a leading batch dim
    yb = np.stack([y[:2], synth.structured_stft(2, 100, 4, 2, seed=54)[0]])
    initb = np.stack([init[:2], init[2:]])
    m = RC.CBMMTrainer().fit(yb, initialization=initb, iterations=2)
    fits['yb'], fits['initb'] = yb, initb
    fits.update({f'batch_{k}': v for k, v in _model(m).items()})
    fits['batch_affiliation'] = m.predict(yb)
    np.savez_compressed(os.path.join(out_dir, 'cbmm_fit.npz'), **fits)

    # frequency-tied weights and the inline permutation alignment (cbmm.py:186-203)
    coupled = {}
    y = synth.structured_stft(65, 40, 3, 2, seed=55)[0]
    init = synth.init_affiliation(65, 2, 40, seed=56)
    coupled['y'], coupled['init'] = y, init
    for name, axis, inline in (('tied_time', (-3,), False), ('tied', (-3, -1), False), ('inline_pa', (-3,), True)):
        al = pa.DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                         main_iterations=5, sub_iterations=2) if inline else None
        m = RC.CBMMTrainer().fit(y, initialization=init, iterations=2, weight_constant_axis=axis,
                                 inline_permutation_aligner=al)
        coupled.update({f'{name}_{k}': v for k, v in _model(m).items()})
        coupled[f'{name}_affiliation'] = m.predict(y)
        if inline:
            coupled['plan'] = np.asarray(al.alignment_plan)
    np.savez_compressed(os.path.join(out_dir, 'cbmm_coupled.npz'), **coupled)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else OUT
    os.makedirs(out, exist_ok=True)
    ref_shim.load()
    make_bingham(out)


if __name__ == '__main__':
    main()
