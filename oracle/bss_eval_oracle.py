"""NumPy restatement of BSS Eval v3 as pb_bss.evaluation.mir_eval_sources computes it (mir_eval.separation's
bss_eval_sources for E = K estimates, pb_bss's _bss_eval_sources_and_noise for E = K + 1), from the definition in
Vincent, Gribonval and Fevotte, IEEE TASLP 14(4), 2006.  Test infrastructure only: the checker of
pb_bss_b200.evaluation.mir_eval_sources.

For references s_1..s_K and an estimate x, all of T samples, zero-padded to T' = T + L - 1 (L = 512):
  - P_R(x), the orthogonal projection of x onto span{s_i delayed by tau : i in R, 0 <= tau < L}, solves G c = d with
    G[(i,t1),(j,t2)] = r_ij[t1 - t2], d[(i,t)] = r_(i,x)[t] and r_ab[d] = sum_u a[u] b[u + d] (computed by FFT,
    without wrap-around for |d| < L), and is sum_i s_i * c_i, the first T' samples;
  - for reference j: s_filt = P_{j}(x), e_interf = P_all(x) - P_{j}(x), e_artif = x - P_all(x);
  - SDR = 10 log10(|s_filt|^2 / |e_interf + e_artif|^2), SIR = 10 log10(|s_filt|^2 / |e_interf|^2),
    SAR = 10 log10(|s_filt + e_interf|^2 / |e_artif|^2); a zero denominator gives +inf;
  - the sums of squares are taken of the explicit residual signals.
G is solved with np.linalg.solve (LU with partial pivoting), once per item for all estimates.
"""
import itertools

import numpy as np
import scipy.fft

L = 512


def _safe_db(num, den):
    if den == 0:
        return np.inf
    with np.errstate(divide='ignore'):
        return 10 * np.log10(num / den)


def pair_matrices(reference, estimation):
    """sdr, sir, sar (E, K) of every (estimate, reference) pair of one item: reference (K, T), estimation (E, T)."""
    reference = np.asarray(reference, dtype=np.float64)
    estimation = np.asarray(estimation, dtype=np.float64)
    K, T = reference.shape
    E = estimation.shape[0]
    Tp = T + L - 1
    nfft = scipy.fft.next_fast_len(Tp, real=True)
    Fr = scipy.fft.rfft(reference, nfft)
    Fe = scipy.fft.rfft(estimation, nfft)
    rr = scipy.fft.irfft(np.conj(Fr)[:, None] * Fr[None], nfft)      # rr[i, j, m] = r_ij[m] (mod nfft)
    re = scipy.fft.irfft(np.conj(Fr)[:, None] * Fe[None], nfft)[..., :L]
    lag = np.arange(L)
    G = rr[:, :, (lag[:, None] - lag[None, :]) % nfft].transpose(0, 2, 1, 3).reshape(K * L, K * L)
    D = re.transpose(0, 2, 1).reshape(K * L, E)
    c_all = np.linalg.solve(G, D).reshape(K, L, E)
    c_one = np.stack([np.linalg.solve(G[j * L:(j + 1) * L, j * L:(j + 1) * L], D[j * L:(j + 1) * L])
                      for j in range(K)])                              # (K, L, E)

    def project(i, c):  # s_i * c for the E filters c (L, E): (E, T')
        return scipy.fft.irfft(Fr[i][None] * scipy.fft.rfft(c.T, nfft), nfft)[:, :Tp]

    x = np.zeros((E, Tp))
    x[:, :T] = estimation
    p_all = sum(project(i, c_all[i]) for i in range(K))
    sdr, sir, sar = (np.empty((E, K)) for _ in range(3))
    for j in range(K):
        p_j = project(j, c_one[j])
        for e in range(E):
            s_filt, e_interf, e_artif = p_j[e], p_all[e] - p_j[e], x[e] - p_all[e]
            sdr[e, j] = _safe_db(np.sum(s_filt ** 2), np.sum((e_interf + e_artif) ** 2))
            sir[e, j] = _safe_db(np.sum(s_filt ** 2), np.sum(e_interf ** 2))
            sar[e, j] = _safe_db(np.sum((s_filt + e_interf) ** 2), np.sum(e_artif ** 2))
    return sdr, sir, sar


def select(sdr, sir, sar, compute_permutation=True):
    """The first maximiser of the mean SIR over itertools.permutations(range(E), K), with np.mean / np.argmax
    semantics; without permutation the pairs (k, k)."""
    E, K = sir.shape
    dum = np.arange(K)
    if not compute_permutation:
        return sdr[dum, dum], sir[dum, dum], sar[dum, dum], None
    perms = list(itertools.permutations(range(E), K))
    with np.errstate(invalid='ignore'):   # inf - inf: a NaN mean, which np.argmax picks first
        mean_sir = np.array([np.mean(sir[list(p), dum]) for p in perms])
    best = np.asarray(perms[int(np.argmax(mean_sir))])
    return sdr[best, dum], sir[best, dum], sar[best, dum], best


def bss_eval_2d(reference, estimation, compute_permutation=True):
    K, E = reference.shape[0], estimation.shape[0]
    for name, v in (('reference', reference), ('estimation', estimation)):
        if np.any(np.all(v == 0, axis=-1)):
            raise ValueError(f'an all-zero {name} signal')
    if E == K + 1 and not compute_permutation:
        raise NotImplementedError(compute_permutation, 'with K + 1')
    if E not in (K, K + 1):
        raise ValueError(f'Shapes do not fit: {reference.shape} vs. {estimation.shape}')
    return select(*pair_matrices(reference, estimation), compute_permutation=compute_permutation)


def mir_eval_sources(reference, estimation, return_dict=False, compute_permutation=True):
    """The reference's interface: (K, T) or (K, ..., T) in; sdr, sir, sar[, selection] of shape (K, ...) out."""
    reference, estimation = np.asarray(reference), np.asarray(estimation)
    if reference.ndim < 2:
        raise ValueError(f'Strange input shape: {reference.shape}')
    assert reference.shape[1:] == estimation.shape[1:], (reference.shape, estimation.shape)
    K, T = reference.shape[0], reference.shape[-1]
    middle = reference.shape[1:-1]
    r = reference.reshape(K, -1, T)
    x = estimation.reshape(estimation.shape[0], -1, T)
    res = [bss_eval_2d(r[:, m], x[:, m], compute_permutation) for m in range(r.shape[1])]
    out = [np.stack([v[i] for v in res], axis=-1).reshape(K, *middle) for i in range(3)]
    if compute_permutation:
        out.append(np.stack([v[3] for v in res], axis=-1).reshape(K, *middle).astype(np.int64))
    if return_dict:
        return dict(zip(('sdr', 'sir', 'sar', 'selection'), out))
    return tuple(out)
