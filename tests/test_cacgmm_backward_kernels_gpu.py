"""The cACGMM backward kernels (em_backward.cuh, and launch_em's scatter with signed coefficients) over their shape
domain and branches, against mpmath directional derivatives (oracle/cacgmm_autograd_oracle.py mp_directional) where
F <= 4 and D <= 8, and elsewhere against the float64 restatement, whose closed forms tests/test_cacgmm_autograd_oracle.py
checks against mpmath.  Every comparison is per bin, against a bound from the bin's conditioning:
64 u D (kappa + 1 / gap) per M-step, kappa = lam_max / lam_min of the bin's model and gap the smallest relative gap
between two of its eigenvalues that the backward divides by (tied pairs excluded)."""
import numpy as np
import pytest
import torch

from oracle import cacgmm_autograd_oracle as A
from oracle import synth

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pb_bss_b200.distribution import CACGMM, CACGMMTrainer, ComplexAngularCentralGaussian
    from pb_bss_b200.distribution.cacgmm import cacgmm_m_step

DEV = 'cuda'
U = np.finfo(np.float64).eps
TIE_GAP = 2.0 ** -26   # kTieGap of em_backward.cuh


def _t(a, grad=False, dtype=None):
    t = torch.tensor(np.ascontiguousarray(a), device=DEV, dtype=dtype)
    return t.requires_grad_() if grad else t


def _np(t):
    return t.detach().cpu().numpy()


def _bin_bound(lam, D, steps=1):
    """(F,) 64 u D steps (kappa + 1 / gap) from the device model's eigenvalues lam (F, K, D) (ascending)"""
    lam = _np(lam).reshape(lam.shape[0], -1, D)
    top = lam[..., -1:]
    kappa = (top / lam).max(axis=(-2, -1))
    gaps = np.diff(lam, axis=-1) / top
    gaps = np.where(gaps > TIE_GAP, gaps, np.inf).min(axis=(-2, -1)) if D > 1 else np.full(lam.shape[0], np.inf)
    return 64 * U * D * steps * (kappa + 1 / gaps)


def _per_bin(got, ref, scale):
    """(F,) max |got - ref| over each bin (leading dim) / scale (F,)"""
    return np.abs(got - ref).reshape(got.shape[0], -1).max(-1) / np.maximum(scale, 1e-300)


def _inputs(F, T, D, K, seed, q=False, sal=False):
    y, _ = synth.structured_stft(F, T, D, K, seed=seed)
    init = synth.init_affiliation(F, K, T, seed=seed + 1)
    rng = np.random.RandomState(seed + 2)
    x = dict(y=y, init=init)
    if q:
        x['q'] = rng.uniform(0.5, 2.0, (F, K, T))
    if sal:
        x['saliency'] = rng.uniform(0.1, 1.0, (F, T))
    return x, rng


def _device(x, R, probe=None, iterations=1, mask=None, dtype=None, **kw):
    """grads of sum R * predict(probe) + 0.1 log_likelihood(probe) through the device M-step (iterations = 1, with
    x['q'] as its quadratic form) or the unrolled fit; returns (grads dict of numpy, eigenvalues of the model)"""
    ts = {k: _t(v, True, dtype if k == 'y' else None) for k, v in x.items()}
    if iterations == 1:
        m = cacgmm_m_step(ts['y'], ts.get('q'), ts['init'], saliency=ts.get('saliency'), **kw)
    else:
        m = CACGMMTrainer().fit(ts['y'], initialization=ts['init'], iterations=iterations, saliency=ts.get('saliency'),
                                source_activity_mask=None if mask is None else _t(mask), **kw)
    yp = ts['y'] if probe is None else _t(probe, dtype=dtype)
    loss = (_t(R) * m.predict(yp)).sum() + 0.1 * m.log_likelihood(yp)
    g = torch.autograd.grad(loss, list(ts.values()))
    return {k: _np(v) for k, v in zip(ts, g)}, m


def _restatement(x, R, probe=None, iterations=1, mask=None, dev=DEV, **kw):
    ts = {k: torch.tensor(v, device=dev, requires_grad=True) for k, v in x.items()}
    if iterations == 1:
        m = A.m_step(ts['y'], ts.get('q'), ts['init'], ts.get('saliency'), **kw)
    else:
        m = A.fit(ts['y'], ts['init'], iterations, saliency=ts.get('saliency'),
                  source_activity_mask=None if mask is None else _t(mask), **kw)
    yp = ts['y'] if probe is None else torch.tensor(probe, device=dev)
    loss = (torch.tensor(R, device=dev) * A.predict(yp, m)).sum() + 0.1 * A.log_likelihood(yp, m)
    g = torch.autograd.grad(loss, list(ts.values()))
    return {k: _np(v) for k, v in zip(ts, g)}


def _compare(name, got, ref, bound):
    """per-bin check of every gradient against the bin's largest reference gradient entry (a gradient that is 0 in
    exact arithmetic, such as that of q at T = 1, is judged by the bin's scale, not by its own rounding noise);
    returns the worst err / bound"""
    worst = 0.0
    scale = np.max([np.abs(v).reshape(v.shape[0], -1).max(-1) for v in ref.values()], axis=0)
    for k in ref:
        assert np.all(np.isfinite(got[k])), k
        r = _per_bin(got[k], ref[k], scale) / bound
        worst = max(worst, float(r.max()))
        assert r.max() <= 1, (name, k, int(r.argmax()), float(r.max()))
    print(f'\n{name}: worst per-bin err / bound {worst:.2e}')
    return worst


def _check_mp(name, grads, x, bound, rng, n_dirs=2, **kw):
    """Re <grad, dir> against mpmath along random directions, |err| <= bound sum |grad| |dir|"""
    worst = 0.0
    for _ in range(n_dirs):
        dirs = {k: (rng.standard_normal(v.shape) + 1j * rng.standard_normal(v.shape)) if np.iscomplexobj(v)
                else rng.standard_normal(v.shape) for k, v in x.items()}
        ref = A.mp_directional(x, dirs, **kw)
        got = A.directional(grads, dirs)
        scale = sum(float(np.sum(np.abs(grads[k]) * np.abs(dirs[k]))) for k in dirs)
        r = abs(got - ref) / (bound * scale)
        worst = max(worst, r)
        assert r <= 1, (name, got, ref, scale)
    print(f'\n{name}: worst err / bound against mpmath {worst:.2e}')


# ---- T around the 64-frame tiles, and one long T ---------------------------------------------------------------------
@pytest.mark.parametrize('T', [1, 2, 63, 64, 65, 127, 128, 129])
@pytest.mark.parametrize('D', [4, 5])   # 4: em_fast_kernel, 5: em_generic_kernel
def test_frame_tiles_m_step_against_mpmath(D, T):
    F, K = 2, 2
    x, rng = _inputs(F, T, D, K, seed=T + 10 * D, q=True, sal=True)
    # probe frames of their own: at T = 1 both classes fit the same model, and a loss on y itself would not change
    # with y (its gradient is rounding noise); T < D: a floored model, so a floor that keeps 1 / floor moderate
    probe = rng.standard_normal((F, 7, D)) + 1j * rng.standard_normal((F, 7, D))
    R = rng.standard_normal((F, K, 7))
    floor = 1e-4
    g, m = _device(x, R, probe=probe, eigenvalue_floor=floor)
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    _compare(f'tiles D={D} T={T}', g, _restatement(x, R, probe=probe, eigenvalue_floor=floor), bound)
    if T <= 65:
        _check_mp(f'tiles D={D} T={T}', g, x, bound.max(), rng, R=R, probe=probe, eigenvalue_floor=floor)


@pytest.mark.parametrize('D,K', [(4, 2), (5, 3)])
def test_long_utterance_m_step(D, K):
    F, T = 2, 70000
    x, rng = _inputs(F, T, D, K, seed=3, q=True)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R)
    # sums over T frames: the bound grows with log2 T (pairwise) to T (sequential chunk sums)
    _compare(f'long T={T} D={D} K={K}', g, _restatement(x, R), _bin_bound(m.cacg.covariance_eigenvalues, D) * 64)


def test_predict_backward_against_mpmath():
    F, T, D, K = 2, 65, 5, 3
    x0, rng = _inputs(F, T, D, K, seed=40)
    m0 = CACGMMTrainer().fit(_t(x0['y']), initialization=_t(x0['init']), iterations=3)
    x = dict(y=x0['y'], V=_np(m0.cacg.covariance_eigenvectors), lam=_np(m0.cacg.covariance_eigenvalues),
             w=_np(m0.weight))
    R = rng.standard_normal((F, K, T))
    ts = {k: _t(v, True) for k, v in x.items()}
    mm = CACGMM(weight=ts['w'], cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=ts['V'],
                                                                    covariance_eigenvalues=ts['lam']))
    loss = (_t(R) * mm.predict(ts['y'])).sum() + 0.1 * mm.log_likelihood(ts['y'])
    g = {k: _np(v) for k, v in zip(ts, torch.autograd.grad(loss, list(ts.values())))}
    _check_mp('predict', g, x, _bin_bound(m0.cacg.covariance_eigenvalues, D).max(), rng, iterations=0, R=R)


# ---- D = 2..34 and K = 1..19 through the unrolled fit ----------------------------------------------------------------
SWEEP = ([(D, K) for D in (4, 6, 8) for K in (2, 3, 4)]                           # em_fast_kernel
         + [(5, 3), (7, 3), (8, 5), (2, 2), (3, 3), (9, 3), (12, 3), (16, 3)]     # generic neighbours
         + [(18, 3), (19, 3), (20, 3), (21, 3), (23, 2), (24, 2)]                  # 48 KB shared-memory crossings
         + [(31, 2), (32, 2), (33, 2), (34, 2)]                                    # lane loops wrap, NS & 31
         + [(6, 19), (34, 19)])


@pytest.mark.parametrize('D,K', SWEEP)
def test_fit_gradient_over_the_shape_domain(D, K):
    F, T, it = 2, 70, 2
    x, rng = _inputs(F, T, D, K, seed=D * 31 + K, sal=D % 2 == 0)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R, iterations=it)
    _compare(f'fit D={D} K={K}', g, _restatement(x, R, iterations=it),
             _bin_bound(m.cacg.covariance_eigenvalues, D, it) * 16)


def test_k1_m_step_against_mpmath():
    F, T, D, K = 2, 20, 4, 1
    x, rng = _inputs(F, T, D, K, seed=5, q=True)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R)
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    _compare('K=1', g, _restatement(x, R), bound)
    _check_mp('K=1', g, x, bound.max(), rng, R=R)


# ---- F past launch_em's 65535-bin split ------------------------------------------------------------------------------
def test_65537_bins_match_and_each_bin_is_independent_of_the_others():
    F, T, D, K = 65537, 3, 2, 2
    x, rng = _inputs(F, T, D, K, seed=7, q=True)
    probe = rng.standard_normal((F, 4, D)) + 1j * rng.standard_normal((F, 4, D))
    R = rng.standard_normal((F, K, 4))
    g, m = _device(x, R, probe=probe)
    # (the restatement on the CPU: cuSOLVER's batched eigh takes fewer matrices; 4x: the tail over 65537 bins)
    _compare('F=65537', g, _restatement(x, R, probe=probe, dev='cpu'),
             4 * _bin_bound(m.cacg.covariance_eigenvalues, D))
    g2, _ = _device(x, R, probe=probe)
    for k in g:
        assert np.array_equal(g[k], g2[k]), k                # repeated backward calls: bitwise equal
    pick = [0, 1, 65534, 65535, 65536]
    xs = {k: v[pick] for k, v in x.items()}
    gs, _ = _device(xs, R[pick], probe=probe[pick])
    for k in g:
        assert np.array_equal(g[k][pick], gs[k]), k          # a bin's gradient does not depend on F or other bins


# ---- complex64: z rounded through float2 as the forward rounds it ----------------------------------------------------
@pytest.mark.parametrize('D,K', [(4, 2), (5, 3)])
def test_complex64_gradient_is_that_of_the_rounded_forward(D, K, monkeypatch):
    F, T = 3, 100
    x, rng = _inputs(F, T, D, K, seed=D + K)
    x['y'] = x['y'].astype(np.complex64)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R, dtype=torch.complex64)
    plain = A.normalize
    # the forward's z of a complex64 y: y / |y| rounded to complex64 (the gradient passes the rounding unchanged)
    monkeypatch.setattr(A, 'normalize', lambda y: plain(y).to(torch.complex64).to(torch.complex128)
                        if y.dtype == torch.complex64 else plain(y))
    ts = {k: _t(v, True) for k, v in x.items()}
    mr = A.m_step(ts['y'], None, ts['init'])
    loss = (_t(R) * A.predict(ts['y'], mr)).sum() + 0.1 * A.log_likelihood(ts['y'], mr)
    ref = {k: _np(v) for k, v in zip(ts, torch.autograd.grad(loss, list(ts.values())))}
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D) * 64
    _compare(f'complex64 D={D} K={K} (affiliation)', {'init': g['init']}, {'init': ref['init']}, bound)
    # the y gradient comes back as complex64: its own rounding, 2^-24 per element, dominates
    _compare(f'complex64 D={D} K={K} (y)', {'y': g['y']}, {'y': ref['y']}, np.maximum(bound, 2.0 ** -21))


# ---- options and branches --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('floor', [1e-10, 0.3])   # 0.3: the floor is active in every class
def test_covariance_norms_and_floor_against_mpmath(norm, floor):
    F, T, D, K = 2, 30, 4, 2
    x, rng = _inputs(F, T, D, K, seed=11, q=True, sal=True)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R, covariance_norm=norm, eigenvalue_floor=floor)
    lam = _np(m.cacg.covariance_eigenvalues)
    assert (floor > 0.1) == bool(np.any(lam[..., 0] == lam[..., 1]))
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    _compare(f'norm={norm} floor={floor}', g, _restatement(x, R, covariance_norm=norm, eigenvalue_floor=floor), bound)
    _check_mp(f'norm={norm} floor={floor}', g, x, bound.max(), rng, R=R, covariance_norm=norm, eigenvalue_floor=floor)


def test_saliency_zero_bin_weight_axis_and_tiny_q():
    F, T, D, K = 3, 40, 5, 3
    x, rng = _inputs(F, T, D, K, seed=12, q=True, sal=True)
    x['saliency'][0, ::3] = 0.0      # frames without saliency
    x['q'][1, 0, :3] = 1e-309        # q <= 10 tiny: c = g / (10 tiny), no gradient to q
    x['init'][1, 0, :3] = 1e-300     # (small weights keep the scatter finite)
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R)
    _compare('saliency / tiny q', g, _restatement(x, R), _bin_bound(m.cacg.covariance_eigenvalues, D))
    assert not np.any(g['init'][0, :, ::3]) and not np.any(g['q'][1, 0, :3])
    x2 = {k: v for k, v in x.items() if k != 'saliency'}
    g, m = _device(x2, R, weight_constant_axis=-2)
    _compare('weight axis -2', g, _restatement(x2, R, weight_constant_axis=-2),
             _bin_bound(m.cacg.covariance_eigenvalues, D))


@pytest.mark.parametrize('eps', [0.0, 1e-10, 1e-3])
def test_fit_with_an_all_inactive_frame_and_affiliation_eps(eps):
    F, T, D, K = 2, 50, 4, 3
    x, rng = _inputs(F, T, D, K, seed=13)
    mask = rng.uniform(size=(F, K, T)) > 0.3
    mask[:, :, 7] = False              # den <= tiny: abar = gbar / tiny
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R, iterations=3, mask=mask, affiliation_eps=eps)
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D, 3) * 16
    _compare(f'mask eps={eps}', g, _restatement(x, R, iterations=3, mask=mask, affiliation_eps=eps), bound)
    _check_mp(f'mask eps={eps}', g, x, bound.max(), rng, n_dirs=1, R=R, iterations=3, mask=mask,
              affiliation_eps=eps)


# ---- edges -----------------------------------------------------------------------------------------------------------
def test_zero_frame_passes_no_gradient():
    F, T, D, K = 2, 40, 4, 3
    x, rng = _inputs(F, T, D, K, seed=14, q=True)
    x['y'][:, 5] = 0.0
    R = rng.standard_normal((F, K, T))
    g, m = _device(x, R)
    _compare('zero frame', g, _restatement(x, R), _bin_bound(m.cacg.covariance_eigenvalues, D))
    assert not np.any(g['y'][:, 5])


@pytest.mark.parametrize('rank_from_top', [1, 'D-1'])
@pytest.mark.parametrize('D', [4, 7])
def test_rank_deficient_observations(D, rank_from_top):
    F, T, K = 2, 60, 2
    r = 1 if rank_from_top == 1 else D - 1
    rng = np.random.RandomState(D + r)
    basis = rng.randn(F, r, D) + 1j * rng.randn(F, r, D)
    y = np.einsum('ftr,frd->ftd', rng.randn(F, T, r) + 1j * rng.randn(F, T, r), basis)
    x = dict(y=y, init=synth.init_affiliation(F, K, T, seed=r))
    probe = rng.randn(F, 9, D) + 1j * rng.randn(F, 9, D)
    R = rng.standard_normal((F, K, 9))
    floor = 1e-4
    g, m = _device(x, R, probe=probe, eigenvalue_floor=floor)
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    _compare(f'rank {r} of D={D}', g, _restatement(x, R, probe=probe, eigenvalue_floor=floor), bound)
    _check_mp(f'rank {r} of D={D}', g, x, bound.max(), rng, R=R, probe=probe, eigenvalue_floor=floor)


@pytest.mark.parametrize('norm', ['eigenvalue', 'trace', False])
@pytest.mark.parametrize('D', [3, 5, 8])
def test_exact_unfloored_ties_against_mpmath(norm, D):
    """tied model eigenvalues below the top: the M-step adjoint's tie limit -lam' P / lam^2 (zero before the fix)"""
    w0 = [0.3, 0.3] + [0.5 + 0.1 * d for d in range(D - 2)]
    w1 = [0.2, 0.2] + [0.45] * (D - 3) + [0.8]
    y, init, probe, R = A.tie_data(D, [w0, w1])
    x = dict(y=y, init=init)
    g, m = _device(x, R, probe=probe, covariance_norm=norm)
    lam = _np(m.cacg.covariance_eigenvalues)[0]
    assert lam[0, 0] == lam[0, 1] and lam[1, 0] == lam[1, 1]
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    _compare(f'tie D={D} {norm}', g, _restatement(x, R, probe=probe, covariance_norm=norm), bound)
    _check_mp(f'tie D={D} {norm}', g, x, bound.max(), np.random.RandomState(D), n_dirs=3, R=R, probe=probe,
              covariance_norm=norm)


@pytest.mark.parametrize('gap', [1e-3, 1e-6, 1e-8, 1e-10])
def test_near_ties_against_mpmath(gap):
    """either side of kTieGap: the divided difference loses ~u D / gap, the tie limit is exact for B^-1 consumers"""
    D = 4
    y, init, probe, R = A.tie_data(D, [[0.3, 0.3 * (1 + gap), 0.5, 0.9], [0.7, 0.2, 0.2 * (1 + gap), 0.4]], seed=1)
    x = dict(y=y, init=init)
    g, m = _device(x, R, probe=probe)
    bound = 64 * U * D * (1 / gap + 10)
    _compare(f'near tie {gap:.0e}', g, _restatement(x, R, probe=probe), np.full(1, bound))
    _check_mp(f'near tie {gap:.0e}', g, x, bound, np.random.RandomState(2), R=R, probe=probe)


def test_tied_top_eigenvalue_follows_the_forwards_top_eigenvector():
    D = 4
    y, init, probe, R = A.tie_data(D, [[0.0, 0.4, 0.7, 0.7], [0.5, 0.0, 0.9, 0.9]], seed=3)
    x = dict(y=y, init=init)
    g, m = _device(x, R, probe=probe, eigenvalue_floor=1e-3)
    _check_mp('top tie', g, x, _bin_bound(m.cacg.covariance_eigenvalues, D).max(), np.random.RandomState(4), n_dirs=3,
              R=R, probe=probe, eigenvalue_floor=1e-3, top=_np(m.cacg.covariance_eigenvectors))


def test_predict_with_subnormal_weights_takes_the_tiny_denominator_branch():
    """weights of 1e-310: den = sum_k a_k <= tiny, so gamma = a / tiny is not normalised and its adjoint is
    abar = gbar / tiny (no - sum_j gbar_j gamma_j term); T = 3 keeps the weight gradient, ~T R / tiny, finite"""
    F, T, D, K = 2, 3, 4, 3
    x0, rng = _inputs(F, 60, D, K, seed=41)
    m0 = CACGMMTrainer().fit(_t(x0['y']), initialization=_t(x0['init']), iterations=2)
    x = dict(y=x0['y'][:, :T], V=_np(m0.cacg.covariance_eigenvectors), lam=_np(m0.cacg.covariance_eigenvalues),
             w=np.full(_np(m0.weight).shape, 1e-310))
    R = 0.1 * rng.standard_normal((F, K, T))
    ts = {k: _t(v, True) for k, v in x.items()}
    mm = CACGMM(weight=ts['w'], cacg=ComplexAngularCentralGaussian(covariance_eigenvectors=ts['V'],
                                                                    covariance_eigenvalues=ts['lam']))
    aff = mm.predict(ts['y'])
    assert 0 < _np(aff).sum(-2).max() < 1          # den <= tiny, and the affiliations are not renormalised
    g = torch.autograd.grad((_t(R) * aff).sum(), list(ts.values()))
    tr = {k: _t(v, True) for k, v in x.items()}
    ref = torch.autograd.grad((_t(R) * A.predict(tr['y'], A.from_eig(tr['V'], tr['lam'], tr['w']))).sum(),
                              list(tr.values()))
    _compare('subnormal weights', {k: _np(v) for k, v in zip(ts, g)}, {k: _np(v) for k, v in zip(tr, ref)},
             _bin_bound(m0.cacg.covariance_eigenvalues, D))


def test_dead_class_passes_no_gradient():
    """a class with S_k <= tiny: affiliations exactly 0 in bin 0 (C_k = 0, every eigenvalue floored) and 1e-310 in
    bin 1 (C_k = D Psi_k / tiny, an ordinary covariance); its affiliations and quadratic forms get exactly 0"""
    F, T, D, K = 2, 20, 4, 3
    x, rng = _inputs(F, T, D, K, seed=15, q=True)
    x['init'][0, 2] = 0.0
    x['init'][1, 2] = 1e-310
    probe = rng.standard_normal((F, 6, D)) + 1j * rng.standard_normal((F, 6, D))
    R = rng.standard_normal((F, K, 6))
    g, m = _device(x, R, probe=probe)
    for k, v in g.items():
        assert np.all(np.isfinite(v)), k
    assert not np.any(g['init'][:, 2]) and not np.any(g['q'][:, 2])
    bound = _bin_bound(m.cacg.covariance_eigenvalues, D)
    # bin 1's dead class is a subnormal scatter, rounded to 2^-1074 absolute by both implementations in their own order
    sub = 2.0 ** -1074 / (1e-310 / x['q'][1, 2].max())
    bound[1] *= (U + sub) / U
    _compare('dead class', g, _restatement(x, R, probe=probe), bound)


def test_floored_and_unfloored_eigenvalue_at_the_kink():
    """lam_1 = floor exactly (floored) and lam_2 one ulp pair above it (unfloored): the pair sits at the floor's kink,
    within the rounding of mu, and contributes 0 in the kernel and the restatement alike.  z = e_d and weights summing
    to 2 keep every value exact."""
    D = 4
    w = np.array([0.125, 0.25, 0.25 + 2.0 ** -52, 1.375 - 2.0 ** -52])
    floor = w[1] / w[3]
    y = np.eye(D, dtype=np.complex128)[None]
    init = np.stack([w, np.array([0.5, 0.2, 0.9, 0.4])])[None]
    rng = np.random.RandomState(16)
    probe = rng.standard_normal((1, 6, D)) + 1j * rng.standard_normal((1, 6, D))
    R = rng.standard_normal((1, 2, 6))
    x = dict(y=y, init=init)
    g, m = _device(x, R, probe=probe, eigenvalue_floor=floor)
    lam = _np(m.cacg.covariance_eigenvalues)[0, 0]
    assert lam[1] == floor and lam[2] > floor
    _compare('kink', g, _restatement(x, R, probe=probe, eigenvalue_floor=floor),
             _bin_bound(m.cacg.covariance_eigenvalues, D))
