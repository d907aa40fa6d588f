"""The EM kernels over their whole shape domain against the oracle (oracle/pb_bss_oracle.py, oracle/em_oracle.py).

The entry points accept 1 < D < 35 and 0 < K < 20.  D in {4, 6, 8} x K in {2, 3, 4} run on em_fast_kernel (per
iteration) and the persistent kernels (em_persistent_kernel lean / full / Watson, em_ws_kernel, em_sticky_kernel);
every other shape runs on em_generic_kernel.  Each group records the launches it made (pbb_profile_*) and asserts
which kernel actually ran.

Tolerances are derived from error scales, not flat (DESIGN.md section 3):
- quadratic forms: |dq| <= 16 D u zᴴ|B⁻¹|z (em_oracle.q_error_scale), u the unit roundoff of the stored observation
  (2^-53 for complex128, 2^-24 for complex64: the device normalises in fp64 from the stored values);
- posteriors: |d gamma| <= 2 g max |d lp| from the q and log-det bounds, g = gamma (1 - gamma) at the larger end
  (check_predict);
- single M-steps: eigenvalues and V diag(lambda) Vᴴ to 64 D u (lambda_max = 1);
- fits: the fixed-point tolerances of tests/test_cacgmm_gpu.py (1e-6 / 1e-9), widened by D cond eps where the
  covariances are ill-conditioned (group 4), where both the float64 oracle and the kernels' no-pivot inverse are
  only accurate to cond eps relative.
"""
import os
import sys

import numpy as np
import pytest

from conftest import cos_similarity
from oracle import bingham_oracle as B
from oracle import em_oracle as E
from oracle import pb_bss_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
UNIT = {'complex128': 2.0 ** -53, 'complex64': 2.0 ** -24}
FAST = [(D, K) for D in (4, 6, 8) for K in (2, 3, 4)]
DTYPES = ['complex128', 'complex64']
LEAN_NAMES = {'em_persistent_kernel', 'em_ws_kernel', 'em_sticky_kernel'}


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _recorded_launches(lib):
    """Names of the launches recorded since the last pbb_profile_reset (pbb_profile_dump prints them on fd 2)."""
    import tempfile
    import torch
    torch.cuda.synchronize()
    sys.stderr.flush()
    with tempfile.TemporaryFile(mode='w+') as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            lib.pbb_profile_dump()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        names = [line.split()[1] for line in tmp.read().splitlines() if line.startswith('[pbb]')]
    lib.pbb_profile_reset()
    return names


def last_plan():
    """(kernel, split, variant) of the last persistent fit of this thread (pbb_em_last_plan): kernel 0 em_ws_kernel,
    1 em_sticky_kernel, 2 em_persistent_kernel; variant 0 lean, 1 full with the integer-power softmax, 2 full with the
    log-domain softmax, 3 complex Watson."""
    import ctypes
    from pb_bss_b200 import _lib
    k, s, v = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().pbb_em_last_plan(ctypes.byref(k), ctypes.byref(s), ctypes.byref(v)), 'pbb_em_last_plan')
    return k.value, s.value, v.value


def dispatch(F, T, D, K, lean, streamed):
    """(kernel, split) of pbb_em_dispatch on this GPU's SM count: the plan pbb_cacgmm_fit picks, as long as it picks
    no sticky-bins clusters (which the fit counts on the device)."""
    import ctypes
    import torch
    from pb_bss_b200 import _lib
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    k, s = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().pbb_em_dispatch(F, T, D, K, int(lean), int(streamed), sms, ctypes.byref(k),
                                           ctypes.byref(s)), 'pbb_em_dispatch')
    return k.value, s.value


def device_fit(y, init, iterations, pinned=False, **kw):
    """CACGMMTrainer().fit of NumPy y / init, or (pinned) of pinned host copies of them, which the library streams in
    while it computes; the model with NumPy arrays."""
    import torch
    from pb_bss_b200.distribution import CACGMMTrainer
    from pb_bss_b200.distribution.mixture_model_utils import model_to_host
    if pinned:
        y, init = torch.from_numpy(y).pin_memory(), torch.from_numpy(init).pin_memory()
    return model_to_host(CACGMMTrainer().fit(y, initialization=init, iterations=iterations, **kw))


class Launches:
    """with Launches() as rec: ... -> rec.names, the kernels launched inside the block."""

    def __enter__(self):
        from pb_bss_b200 import _lib
        self.lib = _lib.load()
        self.lib.pbb_profile_reset()
        self.lib.pbb_profile_enable(1)
        self.names = []
        return self

    def __exit__(self, *exc):
        try:
            self.names = _recorded_launches(self.lib)
        finally:
            self.lib.pbb_profile_enable(0)
        return False

    def __contains__(self, name):
        return name in self.names


def _rand_model(F, K, D, seed, lam_min=0.05):
    rng = np.random.default_rng(seed)
    from oracle import linalg_oracle as L
    V = np.stack([np.stack([L.unitary(D, rng) for _ in range(K)]) for _ in range(F)])
    lam = np.sort(rng.uniform(lam_min, 1.0, size=(F, K, D)), axis=-1)
    lam[..., -1] = 1.0
    w = rng.uniform(0.2, 1.0, size=(F, K, 1))
    return dict(weight=w / w.sum(-2, keepdims=True), eigenvectors=V, eigenvalues=lam)


def _device_cacgmm(model):
    from pb_bss_b200.distribution import CACGMM
    from pb_bss_b200.distribution import ComplexAngularCentralGaussian as CACG
    return CACGMM(weight=model['weight'], cacg=CACG(covariance_eigenvectors=model['eigenvectors'],
                                                    covariance_eigenvalues=model['eigenvalues']))


def _noise(F, T, D, seed, cdtype):
    rng = np.random.default_rng(seed)
    y = (rng.standard_normal((F, T, D)) + 1j * rng.standard_normal((F, T, D))) * rng.uniform(0.5, 2, (F, T, 1))
    return y.astype(cdtype)


def _rand_aff(F, K, T, seed):
    a = np.random.default_rng(seed).uniform(0.01, 1.0, size=(F, K, T))
    return a / a.sum(-2, keepdims=True)


def check_predict(y, model, aff, q, cdtype):
    """Device posteriors / quadratic forms against the oracle within the derived bounds."""
    y128 = np.asarray(y).astype(np.complex128)
    D = y128.shape[-1]
    ref_aff, ref_q = O.cacgmm_predict(y128, model, return_quadratic_form=True)
    dq = 16 * D * UNIT[cdtype] * E.q_error_scale(y128, model)
    assert np.all(np.abs(q - ref_q) <= dq + 1e-300), np.max(np.abs(q - ref_q) / dq)
    # gamma (1 - gamma) at either end of the perturbation (1/4 if they straddle 1/2): the first-order bound taken at
    # the oracle's end alone misses a posterior the oracle rounds to exactly 0 or 1
    g = np.maximum(ref_aff * (1 - ref_aff), aff * (1 - aff))
    g = np.where((ref_aff - 0.5) * (aff - 0.5) < 0, 0.25, g)
    dlp = np.max(D * dq / np.maximum(ref_q, O.TINY64), axis=-2, keepdims=True) + 16 * D * EPS
    bound = 2 * g * dlp + 4 * EPS
    err = np.abs(aff - ref_aff)
    assert np.all(err <= bound), (np.max(err / bound), np.unravel_index(np.argmax(err / bound), err.shape))
    return ref_aff, np.broadcast_to(dlp, aff.shape)


def check_model(m, ref, atol, rtol=0.0):
    """cACGMM model against an oracle dict: weights, eigenvalues and the covariances V diag(lambda) Vᴴ."""
    np.testing.assert_allclose(np.asarray(m.weight).reshape(ref['weight'].shape), ref['weight'], rtol=rtol,
                               atol=atol)
    np.testing.assert_allclose(m.cacg.covariance_eigenvalues, ref['eigenvalues'], rtol=rtol, atol=atol)
    np.testing.assert_allclose(m.cacg.covariance, O.cacg_covariance_from_eig(ref['eigenvectors'], ref['eigenvalues']),
                               rtol=rtol, atol=atol)


# ---- 1. generic kernel and update kernels, single steps ---------------------------------------------------------------
GEN_D = [2, 3, 5, 7, 9, 10, 12, 16, 17, 23, 31, 32, 33, 34]
GEN_SHAPES = sorted({(D, K) for D in GEN_D for K in (2, 19)} | {(D, K) for D in (2, 17, 34)
                                                                for K in (1, 2, 5, 16, 17, 19)})


def _t_grid(D):
    return sorted({1, 2, max(D - 1, 1), 127, 128, 129, 300})


@pytest.mark.parametrize('cdtype', DTYPES)
@pytest.mark.parametrize('D,K', GEN_SHAPES)
def test_generic_predict_and_m_step(D, K, cdtype):
    """em_generic_kernel (E and M modes) and cacg_update_kernel at every D, K = 1 .. 19 (the class loop runs several
    times per warp once K exceeds the update CTA's warps, 4 at D = 34), T at the 128-frame chunk edges and T < D
    (singular scatter matrices: every eigenvalue but the largest is floored, as in the reference)."""
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    F = 2
    for T in _t_grid(D):
        y = _noise(F, T, D, seed=T + D, cdtype=cdtype)
        y128 = y.astype(np.complex128)
        model = _rand_model(F, K, D, seed=D * K + T)
        with Launches() as rec:
            aff, q = _device_cacgmm(model).predict(y, return_quadratic_form=True)
            ll = _device_cacgmm(model).log_likelihood(y)
        assert 'em_generic_kernel' in rec and 'em_fast_kernel' not in rec, rec.names
        check_predict(y, model, aff, q, cdtype)
        np.testing.assert_allclose(ll, O.cacgmm_log_likelihood(y128, model), rtol=1e-9,
                                   atol=0 if cdtype == 'complex128' else 16 * D * UNIT[cdtype] * F * T)
        # one M-step from given affiliations and quadratic forms
        a = _rand_aff(F, K, T, seed=T)
        qq = np.random.default_rng(T).uniform(0.1, 10.0, size=(F, K, T))
        with Launches() as rec:
            m = cacgmm_m_step(y, qq, a)
        assert {'em_generic_kernel', 'cacg_update_kernel'} <= set(rec.names), rec.names
        ref = O.cacgmm_m_step(O.normalize_observation_cacg(y128), qq, a)
        check_model(m, ref, atol=64 * D * UNIT[cdtype])
        if T < D:
            assert np.all(m.cacg.covariance_eigenvalues[..., :D - T] == 1e-10)


@pytest.mark.parametrize('D,K,T,I', [(2, 2, 3, 3), (3, 5, 127, 4), (7, 19, 129, 3), (12, 16, 300, 5),
                                     (17, 2, 128, 4), (23, 17, 257, 3), (34, 19, 300, 3), (33, 5, 129, 3)])
def test_generic_fits(D, K, T, I):
    """Short fits on the generic path (per-iteration em_generic_kernel + cacg_update_kernel)."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F = 2
    y, _ = synth.structured_stft(F, T, D, K, seed=D + T)
    init = synth.init_affiliation(F, K, T, seed=K)
    with Launches() as rec:
        m = CACGMMTrainer().fit(y, initialization=init, iterations=I)
    assert 'em_generic_kernel' in rec and not set(rec.names) & (LEAN_NAMES | {'em_fast_kernel'}), rec.names
    ref = O.cacgmm_fit(y, init, I)
    check_model(m, ref, atol=1e-9, rtol=1e-6)
    np.testing.assert_allclose(m.predict(y), O.cacgmm_predict(y, ref), rtol=1e-6, atol=1e-9)


# ---- 2. em_fast_kernel on the per-iteration path -------------------------------------------------------------------
# fits over the T / frames_per_block grids: short utterances make EM amplify rounding (1e-6 relative seen on 31 to
# 128 frames), so these sweeps take 1e-5 relative / 1e-8 absolute; the mutations they guard against are O(1)
FIT_TOL = {'complex128': 1e-8, 'complex64': 1e-3}
FAST_T = [1, 31, 32, 33, 127, 128, 129, 255, 257, 513]
FPB = [32, 64, 96, 128, 160, 256, 1024]


@pytest.mark.parametrize('cdtype', DTYPES)
@pytest.mark.parametrize('D,K', FAST)
def test_fast_kernel_per_iteration(D, K, cdtype):
    """em_fast_kernel's E- and M-modes and multi_kernel fits with frames_per_block 32 .. 1024 (rounded to 32,
    capped at T) and T at the 32-frame and block edges."""
    from pb_bss_b200.distribution import CACGMMTrainer
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    F = 3
    for i, T in enumerate(FAST_T):
        y = synth.structured_stft(F, T, D, K, seed=T)[0].astype(cdtype)
        y128 = y.astype(np.complex128)
        model = _rand_model(F, K, D, seed=T)
        with Launches() as rec:
            aff, q = _device_cacgmm(model).predict(y, return_quadratic_form=True)
        assert rec.names.count('em_fast_kernel') == 1 and 'em_generic_kernel' not in rec, rec.names
        check_predict(y, model, aff, q, cdtype)
        a = _rand_aff(F, K, T, seed=T)
        qq = np.random.default_rng(T).uniform(0.1, 10.0, size=(F, K, T))
        m = cacgmm_m_step(y, qq, a)
        check_model(m, O.cacgmm_m_step(O.normalize_observation_cacg(y128), qq, a), atol=64 * D * UNIT[cdtype])
        init = synth.init_affiliation(F, K, T, seed=i)
        I = 1 if T < D else 3  # EM on fewer frames than channels is ill-posed: one M-step only
        ref = O.cacgmm_fit(y128, init, I)
        tol = FIT_TOL[cdtype]
        for fpb in (FPB[i % len(FPB)], FPB[(i + 3) % len(FPB)]):
            with Launches() as rec:
                m = CACGMMTrainer().fit(y, initialization=init, iterations=I, multi_kernel=True, frames_per_block=fpb)
            assert rec.names.count('em_fast_kernel') == I and not set(rec.names) & LEAN_NAMES, rec.names
            check_model(m, ref, atol=tol, rtol=1e-5)


# ---- 3. persistent kernels -------------------------------------------------------------------------------------------
PERSIST_T = [1, 2, 31, 127, 128, 129, 256, 257, 383, 384, 385, 1000]


def _persist_cases(D):
    # EM on fewer frames than channels is ill-posed: one M-step only there
    return [(T, 1 if T < D else (1, 2, 8)[i % 3]) for i, T in enumerate(PERSIST_T)]


@pytest.mark.parametrize('cdtype', DTYPES)
@pytest.mark.parametrize('variant', ['lean', 'full', 'watson'])
@pytest.mark.parametrize('D,K', FAST)
def test_persistent_kernels_match_oracle(D, K, variant, cdtype):
    """Every persistent instantiation (lean, full with a saliency, complex Watson) against the oracle, T at the
    128-frame ring-stage edges, 1, 2 and 8 iterations."""
    from pb_bss_b200.distribution import CACGMMTrainer, CWMMTrainer
    F = 2
    tol = FIT_TOL[cdtype]
    for T, I in _persist_cases(D):
        y = synth.structured_stft(F, T, D, K, seed=T + 7)[0].astype(cdtype)
        y128 = y.astype(np.complex128)
        init = synth.init_affiliation(F, K, T, seed=T)
        if variant == 'watson':
            with Launches() as rec:
                m = CWMMTrainer().fit(y, initialization=init, iterations=I)
            assert 'em_persistent_kernel_cw' in rec and 'cw_update_kernel' in rec, rec.names
            ref = O.cwmm_fit(y128, init, I)
            np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-6, atol=tol)
            np.testing.assert_allclose(m.complex_watson.concentration, ref['concentration'],
                                       rtol=1e-6 if cdtype == 'complex128' else 1e-2)
            np.testing.assert_allclose(cos_similarity(m.complex_watson.mode, ref['mode']), 1, atol=tol)
            continue
        sal = None
        if variant == 'full':
            sal = np.random.default_rng(T).uniform(0.2, 1.0, size=(F, T))
        with Launches() as rec:
            m = CACGMMTrainer().fit(y, initialization=init, iterations=I, saliency=sal)
        if variant == 'full':
            assert 'em_persistent_kernel_full' in rec, rec.names
        else:
            assert set(rec.names) & LEAN_NAMES and 'em_persistent_kernel_full' not in rec, rec.names
        assert 'cacg_update_kernel' in rec and 'em_fast_kernel' not in rec, rec.names
        ref = O.cacgmm_fit(y128, init, I, saliency=sal)
        check_model(m, ref, atol=tol, rtol=1e-5)


# D = 8, lean: (F, T, K, I, pinned host input, the plan the library picks: kernel, split)
D8_CASES = [
    (4, 128, 3, 5, False, (1, 1)),    # one ring stage: sticky bins, clusters of 1 CTA
    (5, 350, 3, 8, False, (1, 2)),    # three stages: clusters of 2
    (3, 257, 2, 2, False, (1, 2)),
    (2, 385, 4, 1, False, (1, 4)),    # four stages: clusters of 4
    (2, 1000, 2, 8, False, (1, 4)),
    (300, 200, 3, 3, False, (0, 1)),  # more bins than clusters run at once: em_ws_kernel, no frame split
    (2, 2100, 3, 2, False, (0, 4)),   # 17 stages: a part does not fit the ring of a sticky CTA
    (5, 350, 3, 8, True, (0, 2)),     # pinned host input (streamed upload): em_ws_kernel with the frame split
]


def test_d8_plans_match_oracle():
    """D = 8: every plan the library picks for the lean fit -- em_sticky_kernel with clusters of 1, 2 and 4 CTAs,
    em_ws_kernel without and with the frame split -- each against the oracle."""
    for F, T, K, I, pinned, plan in D8_CASES:
        y, _ = synth.structured_stft(F, T, 8, K, seed=T)
        init = synth.init_affiliation(F, K, T, seed=I)
        with Launches() as rec:
            m = device_fit(y, init, I, pinned=pinned)
        ran = 'em_sticky_kernel' if plan[0] == 1 else 'em_ws_kernel'
        assert ran in rec and not set(rec.names) & (LEAN_NAMES - {ran}), (F, T, rec.names)
        assert last_plan() == (*plan, 0), (F, T, last_plan())
        check_model(m, O.cacgmm_fit(y, init, I), atol=1e-9, rtol=1e-6)


# frame lengths among which every persistent shape finds each frame split the library picks at F = 2
SPLIT_T = [129, 200, 257, 300, 385, 500, 1000, 1500, 2100]


@pytest.mark.parametrize('S', [1, 2, 4])
@pytest.mark.parametrize('D,K', FAST)
def test_frame_split_picked_for_every_shape(D, K, S):
    """Every persistent shape, lean and full, at each frame split S the library picks: the first two T of SPLIT_T for
    which pbb_em_dispatch reports S, and the fit must run the plan it reports.  The lean D = 8 fit reads pinned host
    input, so that it runs em_ws_kernel rather than the sticky-bins kernel."""
    F, I = 2, 4
    ts = [T for T in SPLIT_T if dispatch(F, T, D, K, lean=True, streamed=True)[1] == S][:2]
    assert ts, (D, K, S)
    for T in ts:
        y, _ = synth.structured_stft(F, T, D, K, seed=T + S)
        init = synth.init_affiliation(F, K, T, seed=S)
        for sal in (None, np.random.default_rng(T).uniform(0.2, 1.0, size=(F, T))):
            lean = sal is None
            pinned = lean and D == 8
            m = device_fit(y, init, I, pinned=pinned, saliency=sal)
            plan = dispatch(F, T, D, K, lean, pinned)
            assert last_plan()[:2] == plan == (0 if pinned else 2, S), (T, last_plan(), plan)
            check_model(m, O.cacgmm_fit(y, init, I, saliency=sal), atol=1e-9, rtol=1e-6)


# ---- 4. the floor decision of the persistent update ------------------------------------------------------------------
CONDS = [1e4, 1e7, 1e9, 4e9, 1e11, 'rank']
FLOOR_SHAPES = FAST + [(12, 3), (34, 2)]


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('cond', CONDS, ids=str)
@pytest.mark.parametrize('D,K', FLOOR_SHAPES)
def test_floor_decision(D, K, cond, norm):
    """Graded data on both sides of the no-floor bound tr tn tr(A^-1) floor < 0.5 of cacg_update_class (Gauss-Jordan
    without pivoting below it, Jacobi + floor above it), floor 1e-10.  The fitted models must match the oracle to
    the fixed-point tolerance widened by D cond eps, and every eigenvalue the oracle floors must be the floor."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, I = 2, 300, 4
    floor = 1e-10
    if cond == 'rank':
        y, _ = E.graded_stft(F, T, D, K, 1.0, seed=D * K, rank=D - 2)
        c = 1.0 / floor
    else:
        y, _ = E.graded_stft(F, T, D, K, cond, seed=D * K)
        c = min(cond, 1.0 / floor)
    init = synth.init_affiliation(F, K, T, seed=K)
    with Launches() as rec:
        m = CACGMMTrainer().fit(y, initialization=init, iterations=I, covariance_norm=norm, eigenvalue_floor=floor)
    assert ('em_generic_kernel' in rec) == (D not in (4, 6, 8)), rec.names
    ref = O.cacgmm_fit(y, init, I, covariance_norm=norm, eigenvalue_floor=floor)
    tol = 1e-9 + 10 * D * c * EPS
    lam, lam_ref = m.cacg.covariance_eigenvalues, ref['eigenvalues']
    lmax = lam_ref[..., -1:]
    np.testing.assert_allclose(m.weight, ref['weight'], rtol=0, atol=tol)
    assert np.all(np.abs(lam - lam_ref) <= tol * lam_ref + 64 * D * EPS * lmax), np.max(np.abs(lam - lam_ref) / lam_ref)
    cov_ref = O.cacg_covariance_from_eig(ref['eigenvectors'], lam_ref)
    np.testing.assert_allclose(m.cacg.covariance / lmax[..., None], cov_ref / lmax[..., None], rtol=0, atol=tol)
    floored = lam_ref == (floor if norm == 'eigenvalue' else lmax * floor)
    if norm == 'eigenvalue':
        assert np.all(lam[floored] == floor)
    else:
        np.testing.assert_allclose(lam[floored], np.broadcast_to(lmax * floor, lam.shape)[floored], rtol=tol)
    if cond == 'rank':
        assert np.all(floored[..., :2]), lam_ref[..., :3]
    elif cond == 1e11:
        assert np.any(floored[..., 0]), lam_ref[..., :2]


def test_floor_decision_eigenvalues_against_mpmath():
    """One M-step at cond 4e9 and 1e11 against mpmath at 40 digits: the device's eigenvalues (Jacobi) must be within
    D eps lambda_max of the exact ones, floored exactly where the exact ones are below the floor."""
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    D, K, T = 4, 2, 60
    for cond in (4e9, 1e11):
        y, _ = E.graded_stft(1, T, D, K, cond, seed=3)
        a = _rand_aff(1, K, T, seed=1)
        q = np.random.default_rng(2).uniform(0.5, 2.0, size=(1, K, T))
        m = cacgmm_m_step(y, q, a)
        lam_f, lam_raw = E.mp_cacg_m_step(O.normalize_observation_cacg(y)[0], q[0], a[0])
        np.testing.assert_allclose(m.cacg.covariance_eigenvalues[0], lam_f, rtol=0, atol=64 * D * EPS)
        assert np.all((m.cacg.covariance_eigenvalues[0] == 1e-10) == (lam_raw <= 1e-10))


# ---- 5. the softmax switches -----------------------------------------------------------------------------------------
def _switch_floors(D, K):
    lt, ft = E.lean_threshold(D, K), E.fast_threshold(D)
    out = [lt * 1.5, lt / 1.5]
    if ft != lt:
        out += [ft * 1.5, ft / 1.5]
    return out


@pytest.mark.parametrize('D,K', FAST)
def test_softmax_switches(D, K):
    """Floors just inside and just outside lean_ok ((K-1) D (log10(1/floor) + 1) < 290) and softmax_fast_ok
    (2 D log10(1/floor) < 280): the variant and softmax that run (pbb_em_last_plan), and the fitted models against
    the log-domain oracle -- on separated_stft data, whose fitted covariances reach the floor so that the product-form
    softmax runs at the q ratios and log-det spans its proof assumes, and from the extreme user model of extreme_stft
    (log-domain first E-step, then the fast or log-domain softmax)."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T, I = 2, 200, 5
    floors = _switch_floors(D, K)
    assert E.lean_ok(D, K, floors[0]) and not E.lean_ok(D, K, floors[1])
    for floor in floors:
        lean = E.lean_ok(D, K, floor)
        y, xmodel = E.extreme_stft(F, T, D, K, floor, seed=D + K)
        init = synth.init_affiliation(F, K, T, seed=1)
        variant = 0 if lean else (1 if E.softmax_fast_ok(D, floor) else 2)
        with Launches() as rec:
            m = CACGMMTrainer().fit(y, initialization=init, iterations=I, eigenvalue_floor=floor)
        assert ('em_persistent_kernel_full' in rec) != lean, (floor, rec.names)
        assert last_plan()[2] == variant, (floor, last_plan())
        ref = O.cacgmm_fit(y, init, I, eigenvalue_floor=floor)
        c = 1.0 / ref['eigenvalues'].min()
        check_model(m, ref, atol=1e-9 + 100 * D * c * EPS, rtol=1e-6)
        # separated classes: every fitted covariance floors one direction, other classes' frames have q ~ 1/floor
        ys, lab = E.separated_stft(F, T, D, K, seed=D * K)
        init_s = np.where(np.arange(K)[None, :, None] == lab[:, None, :], 0.7, 0.3 / (K - 1))
        m = CACGMMTrainer().fit(ys, initialization=init_s, iterations=I, eigenvalue_floor=floor)
        assert last_plan()[2] == variant, (floor, last_plan())
        ref = O.cacgmm_fit(ys, init_s, I, eigenvalue_floor=floor)
        _, q_s = O.cacgmm_predict(ys, ref, return_quadratic_form=True)
        assert (q_s.max(-2) / q_s.min(-2)).max() > 1e6  # the q ratios the product form has to carry
        np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-6, atol=1e-9)
        # the fitted covariances are conditioned up to 1/floor, where float64 fixes neither the eigenvectors nor
        # q; the device's own model is therefore judged through its E-step, within the derived bounds
        mm = dict(weight=np.asarray(m.weight), eigenvectors=m.cacg.covariance_eigenvectors,
                  eigenvalues=m.cacg.covariance_eigenvalues)
        aff_s, q_s = m.predict(ys, return_quadratic_form=True)
        ref_s, dlp = check_predict(ys, mm, aff_s, q_s, 'complex128')
        tiny = np.finfo(np.float64).tiny
        # where float64 fixes the log posterior to within 1, no posterior may underflow (at floors near 1e-35 the
        # error scale leaves almost no frame determined: the bound of check_predict is all that can be asked there)
        sure = (ref_s >= tiny) & (dlp < 1)
        assert np.all(aff_s[sure] >= tiny), 'a posterior underflowed'
        # the user model at the limits: predict (log-domain) and a warm start (full variant)
        dm = _device_cacgmm(xmodel)
        aff, q = dm.predict(y, return_quadratic_form=True)
        ref_aff, dlp = check_predict(y, xmodel, aff, q, 'complex128')
        normal = (ref_aff >= np.finfo(np.float64).tiny) & (dlp < 1)
        assert np.all(aff[normal] >= np.finfo(np.float64).tiny), 'a posterior underflowed'
        with Launches() as rec:
            mw = CACGMMTrainer().fit(y, initialization=dm, iterations=2, eigenvalue_floor=floor)
        assert 'em_persistent_kernel_full' in rec, rec.names
        assert last_plan()[2] == (1 if E.softmax_fast_ok(D, floor) else 2), last_plan()
        refw = O.cacgmm_fit(y, xmodel, 2, eigenvalue_floor=floor)
        c = 1.0 / refw['eigenvalues'].min()
        check_model(mw, refw, atol=1e-9 + 100 * D * c * EPS, rtol=1e-6)


# ---- 6. CWMM ---------------------------------------------------------------------------------------------------------
def _device_cwmm(weight, mode, kappa):
    from pb_bss_b200.distribution import CWMM, ComplexWatson
    return CWMM(weight=weight, complex_watson=ComplexWatson(mode=mode, concentration=kappa))


@pytest.mark.parametrize('D', [2, 3, 5, 7, 12, 17, 34])
@pytest.mark.parametrize('K', [1, 2, 5, 19])
def test_cwmm_generic(D, K):
    """CWMM predict (em_generic_kernel, model_kind 1) and fits (cw_update_kernel, class loop past the warps) on the
    generic path."""
    from pb_bss_b200.distribution import CWMMTrainer
    F, T = 2, 129
    y, _ = synth.structured_stft(F, T, D, max(K, 2), seed=D)
    rng = np.random.default_rng(D * K)
    mode = rng.standard_normal((F, K, D)) + 1j * rng.standard_normal((F, K, D))
    mode /= np.linalg.norm(mode, axis=-1, keepdims=True)
    kappa = rng.uniform(0.5, 60.0, size=(F, K))
    w = rng.uniform(0.2, 1, size=(F, K, 1))
    w /= w.sum(-2, keepdims=True)
    with Launches() as rec:
        aff = _device_cwmm(w, mode, kappa).predict(y)
    assert 'em_generic_kernel' in rec, rec.names
    ref = O.cwmm_predict(y, dict(weight=w, mode=mode, concentration=kappa))
    np.testing.assert_allclose(aff, ref, rtol=1e-10, atol=1e-13)
    if K == 1:
        return
    init = synth.init_affiliation(F, K, T, seed=K)
    with Launches() as rec:
        m = CWMMTrainer().fit(y, initialization=init, iterations=3)
    assert 'em_generic_kernel' in rec and 'cw_update_kernel' in rec, rec.names
    r = O.cwmm_fit(y, init, 3)
    np.testing.assert_allclose(m.weight, r['weight'], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(m.complex_watson.concentration, r['concentration'], rtol=1e-6)
    np.testing.assert_allclose(cos_similarity(m.complex_watson.mode, r['mode']), 1, atol=1e-9)


KAPPAS = [1e-3, 0.5, 5.0, 8.0, 10.0, 15.0, 19.999, 20.0, 20.001, 35.0, 100.0, 250.0, 499.0, 500.0]


@pytest.mark.parametrize('D', [2, 3, 4, 5, 8, 12, 17, 34])
def test_watson_normaliser_against_mpmath(D):
    """cw_log_norm (series below kappa = 20, Mardia's closed form above) through the posteriors of CWMM.predict: class
    0 has the tested concentration, class 1 kappa = 1, both the same mode; the weights put the posteriors near 1/2,
    where d gamma = gamma (1 - gamma) d log c.  The reference posteriors use the mpmath normaliser."""
    F, T = len(KAPPAS), 64
    rng = np.random.default_rng(D)
    m0 = rng.standard_normal(D) + 1j * rng.standard_normal(D)
    m0 /= np.linalg.norm(m0)
    mode = np.broadcast_to(m0, (F, 2, D)).copy()
    kappa = np.stack([np.array(KAPPAS), np.ones(F)], axis=1)
    # frames near the mode, so |mᴴz|^2 spans (0, 1] and kappa |mᴴz|^2 stays comparable to the normaliser
    y = m0 + 0.4 * (rng.standard_normal((F, T, D)) + 1j * rng.standard_normal((F, T, D))) / np.sqrt(D)
    z = O.normalize_observation_cw(y)
    r = np.abs(np.einsum('ftd,d->ft', z, m0.conj())) ** 2
    lc = np.stack([E.mp_cw_log_norm(kappa[:, 0], D), E.mp_cw_log_norm(kappa[:, 1], D)], axis=1)
    lp = kappa[:, :, None] * r[:, None, :] - lc[..., None]
    shift = np.median(lp[:, 0] - lp[:, 1], axis=-1)
    w = np.stack([1 / (1 + np.exp(shift)), np.exp(shift) / (1 + np.exp(shift))], axis=1)[..., None]
    ref = O.log_pdf_to_affiliation(w, lp)
    with Launches() as rec:
        aff = _device_cwmm(w, mode, kappa).predict(y)
    assert 'cw_from_model_kernel' in rec, rec.names
    bound = 2 * ref * (1 - ref) * (1e-12 * (1 + np.abs(lc).max(-1)) + 1e-12 * kappa[:, 0])[:, None, None] + 4 * EPS
    err = np.abs(aff - ref)
    assert np.all(err <= bound), [(KAPPAS[i], (err / bound)[i].max()) for i in range(F) if (err > bound)[i].any()]


@pytest.mark.parametrize('D,K', [(4, 3), (4, 4), (6, 2), (6, 3), (8, 2), (8, 4)])
def test_cwmm_persistent_shapes(D, K):
    """The complex Watson persistent kernel at the six shapes the other tests leave out, with concentrations up to
    max_concentration (well-separated data) and down to 20 (a smaller cap)."""
    from pb_bss_b200.distribution import CWMMTrainer
    F, T, I = 3, 300, 6
    y, _ = synth.structured_stft(F, T, D, K, seed=D * K)
    init = synth.init_affiliation(F, K, T, seed=K)
    for mc in (500, 20):
        with Launches() as rec:
            m = CWMMTrainer(max_concentration=mc).fit(y, initialization=init, iterations=I)
        assert 'em_persistent_kernel_cw' in rec, rec.names
        r = O.cwmm_fit(y, init, I, max_concentration=mc)
        np.testing.assert_allclose(m.weight, r['weight'], rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(m.complex_watson.concentration, r['concentration'], rtol=1e-6)
        np.testing.assert_allclose(cos_similarity(m.complex_watson.mode, r['mode']), 1, atol=1e-9)
        np.testing.assert_allclose(m.predict(y), O.cwmm_predict(y, r), rtol=1e-5, atol=1e-8)


# ---- 7. CBMM ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D', [2, 3, 4, 5, 6])
@pytest.mark.parametrize('K', [1, 2, 3, 4, 5, 8, 19])
def test_cbmm_predict_and_m_step(D, K):
    """CBMM predict (model_kind 1 in em_fast_kernel at D in {4, 6} x K in {2, 3, 4}, else em_generic_kernel), with
    and without affiliation_eps, and one M-step (cb_update_kernel, class loop past its warps at K = 8, 19)."""
    from pb_bss_b200.distribution import CBMM, CBMMTrainer, ComplexBingham
    F, T = 2, 257
    y, _ = synth.structured_stft(F, T, D, max(K, 2), seed=D + K)
    init = synth.init_affiliation(F, K, T, seed=K) if K > 1 else np.ones((F, 1, T))
    ref = B.cbmm_m_step(B.normalize_observation_cw(y), init, np.ones((F, T)))
    if K > 1:
        with Launches() as rec:
            m = CBMMTrainer().fit(y, initialization=init, iterations=1)
        assert 'cb_update_kernel' in rec, rec.names
        cb = m.complex_bingham
        np.testing.assert_allclose(cb.covariance_eigenvalues, ref['lam'], rtol=1e-9, atol=1e-12)
        s = np.broadcast_to(np.arange(1, D + 1, dtype=float), ref['lam'].shape)
        np.testing.assert_allclose(B.model_covariance(cb.covariance_eigenvectors, s),
                                   B.model_covariance(ref['V'], s), atol=1e-9)
        np.testing.assert_allclose(m.weight, ref['weight'], rtol=1e-12, atol=1e-15)
    model = CBMM(weight=ref['weight'], complex_bingham=ComplexBingham(ref['V'], ref['lam']))
    fast = D in (4, 6) and K in (2, 3, 4)
    for eps in (0, 1e-3):
        with Launches() as rec:
            aff = model.predict(y, affiliation_eps=eps)
        assert ('em_fast_kernel' if fast else 'em_generic_kernel') in rec, rec.names
        np.testing.assert_allclose(aff, B.cbmm_predict(y, ref, eps), rtol=1e-9, atol=1e-12)


# ---- 8. more than 65535 bins -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('D,K', [(2, 2), (4, 2)])
def test_more_than_65535_bins(D, K):
    """F = 70000 bins take two launches (gridDim.y <= 65535): every bin of the cACGMM, CWMM and CBMM predicts and of
    one cacgmm_m_step against the oracle."""
    from pb_bss_b200.distribution import CBMM, ComplexBingham
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step
    F, T = 70000, 3
    kern = 'em_fast_kernel' if (D, K) == (4, 2) else 'em_generic_kernel'
    y = _noise(F, T, D, seed=1, cdtype=np.complex128)
    model = _rand_model(F, K, D, seed=2)
    with Launches() as rec:
        aff, q = _device_cacgmm(model).predict(y, return_quadratic_form=True)
    assert rec.names.count(kern) == 2, rec.names
    check_predict(y, model, aff, q, 'complex128')
    a, qq = _rand_aff(F, K, T, seed=3), np.random.default_rng(4).uniform(0.1, 10, size=(F, K, T))
    with Launches() as rec:
        m = cacgmm_m_step(y, qq, a)
    assert rec.names.count(kern) == 2, rec.names
    check_model(m, O.cacgmm_m_step(O.normalize_observation_cacg(y), qq, a), atol=64 * D * EPS)
    rng = np.random.default_rng(5)
    mode = rng.standard_normal((F, K, D)) + 1j * rng.standard_normal((F, K, D))
    mode /= np.linalg.norm(mode, axis=-1, keepdims=True)
    kappa = rng.uniform(0.5, 30, size=(F, K))
    w = model['weight']
    with Launches() as rec:
        aff = _device_cwmm(w, mode, kappa).predict(y)
    assert rec.names.count(kern) == 2, rec.names
    np.testing.assert_allclose(aff, O.cwmm_predict(y, dict(weight=w, mode=mode, concentration=kappa)),
                               rtol=1e-10, atol=1e-13)
    # well-separated Bingham eigenvalues (gaps >= 2): the log normaliser is well-conditioned
    lam = -3.0 * np.arange(D - 1, -1, -1) + rng.uniform(0, 1, size=(F, K, D))
    lam[..., -1] = 0
    bm = dict(weight=w, V=model['eigenvectors'], lam=lam)
    with Launches() as rec:
        aff = CBMM(weight=w, complex_bingham=ComplexBingham(bm['V'], lam)).predict(y)
    assert rec.names.count(kern) == 2, rec.names
    np.testing.assert_allclose(aff, B.cbmm_predict(y, bm), rtol=1e-9, atol=1e-12)


# ---- 9. determinism --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('D,K,multi', [(5, 3, False), (17, 19, False), (8, 3, True), (4, 4, True)])
def test_bitwise_reproducible(D, K, multi):
    """Two identical calls give bitwise-equal models and posteriors on the generic and the per-iteration paths."""
    from pb_bss_b200.distribution import CACGMMTrainer
    F, T = 3, 300
    y, _ = synth.structured_stft(F, T, D, K, seed=1)
    init = synth.init_affiliation(F, K, T, seed=2)
    a = CACGMMTrainer().fit(y, initialization=init, iterations=4, multi_kernel=multi)
    b = CACGMMTrainer().fit(y, initialization=init, iterations=4, multi_kernel=multi)
    assert np.array_equal(a.weight, b.weight)
    assert np.array_equal(a.cacg.covariance_eigenvalues, b.cacg.covariance_eigenvalues)
    assert np.array_equal(a.cacg.covariance_eigenvectors, b.cacg.covariance_eigenvectors)
    assert np.array_equal(a.predict(y), b.predict(y))
