"""References for the stage-by-stage checks of BSS Eval's kernels (tests/test_bss_eval_kernels_gpu.py), checked on the
CPU by tests/test_bss_eval_kernels_oracle.py.  Test infrastructure only.

- The device's shape choices (csrc/api_bss_eval.cu: bss_shape, the correlation's NS, the sums width, bss_layout with
  its 256-byte alignment), so that a one-group call's workspace can be read stage by stage: R (the reduced lag
  correlations), G and Gb (the in-place LU factors of [G | D] and of the diagonal blocks [G_jj | D_j], the solution c
  in the right-hand columns after the back substitution) and the per-tile energies.
- Exact lag correlations of integer signals (|x| <= 2^10: every product and partial sum is an integer below 2^42, so
  the device's result is exact in any order), by float64 FFTs of 1024-sample blocks rounded to integers.
- Long-double references (np.longdouble, 64-bit mantissa): the lag correlations, the residual D - G c of a solve
  rebuilt from the device's own R, and the tile energies of P_all x_e and P_j x_e from the device's own c.
- The error bounds the GPU file holds the device to (u = 2^-53; see its docstring) and a host restatement of the
  permutation scan (itertools order, np.mean, np.argmax).
"""
import itertools

import numpy as np
import scipy.fft
import scipy.signal
from numpy.lib.stride_tricks import sliding_window_view

L = 512                # PBB_BSS_EVAL_FILTER
CHUNK = 128            # kCorrChunk: samples staged per step of bss_corr_kernel, and the part span's granule
MAX_PARTS = 64         # kCorrParts
TILE = 128             # kProjTile: output samples per CTA of bss_project_kernel
RHS_PAD = 16           # kRhsPad: row stride of an augmented matrix is n + 16
U = 2.0 ** -53
LD = np.longdouble


# ---- the device's shape choices -------------------------------------------------------------------------------------
def bss_shape(T, K, E):
    """dict of bss_shape: span and parts of the correlation (at most 64 parts of whole 128-sample chunks, a function
    of T only), the 128-sample projection tiles of T + L - 1, N = K L and S = K + E"""
    span = -(-T // MAX_PARTS)
    span = -(-span // CHUNK) * CHUNK
    return dict(T=T, K=K, E=E, S=K + E, N=K * L, span=span, parts=-(-T // span), tiles=-(-(T + L - 1) // TILE))


def corr_ns(K, E):
    """NS of bss_corr_kernel<NS>: 8-column n-tiles of the K + E signals"""
    return -(-(K + E) // 8)


def sums_width(E):
    """8 NS of bss_project_kernel<NS>: one n-tile of estimates, two for E = 9"""
    return 16 if E > 8 else 8


def _align256(b):
    return (b + 255) & ~255


def bss_layout(group, K, E, T):
    """byte offsets of bss_layout: flags (int32 per item), part, R, G, Gb (K > 1), sums; and the total"""
    s = bss_shape(T, K, E)
    S, N = s['S'], s['N']
    out = dict(flags=0)
    out['part'] = _align256(group * 4)
    out['R'] = _align256(out['part'] + group * K * s['parts'] * S * L * 8)
    out['G'] = _align256(out['R'] + group * K * S * L * 8)
    out['Gb'] = _align256(out['G'] + group * N * (N + RHS_PAD) * 8)
    gb = group * K * L * (L + RHS_PAD) * 8 if K > 1 else 0
    out['sums'] = _align256(out['Gb'] + gb)
    out['total'] = out['sums'] + group * s['tiles'] * (K + 1) * 3 * sums_width(E) * 8
    return out


def stages(ws, group, K, E, T, items=None):
    """the stages of the first `items` (default: group) items of a workspace laid out for `group` items, as views
    into ws (a uint8 array): flags (items,), R (items, K, S, L), G (items, N, N + 16), Gb (items, K, L, L + 16) or
    None, sums (items, tiles, K + 1, 3, width)"""
    items = group if items is None else items
    s = bss_shape(T, K, E)
    S, N = s['S'], s['N']
    lay = bss_layout(group, K, E, T)

    def f64(key, shape):
        n = int(np.prod(shape))
        return ws[lay[key]:lay[key] + 8 * n].view(np.float64).reshape(shape)

    out = dict(flags=ws[:4 * items].view(np.int32).copy(), R=f64('R', (items, K, S, L)),
               G=f64('G', (items, N, N + RHS_PAD)),
               Gb=f64('Gb', (items, K, L, L + RHS_PAD)) if K > 1 else None,
               sums=f64('sums', (items, s['tiles'], K + 1, 3, sums_width(E))))
    return out


# ---- lag correlations -------------------------------------------------------------------------------------------------
def exact_int_correlations(refs, sigs):
    """R (K, S, L) with R[a, s, d] = sum_v refs[a, v - d] sigs[s, v], exactly, for integer-valued float64 signals with
    |x| <= 2^10 and T <= 2^22.  Per 512-sample block b: the 1024-sample segment of the reference that block's lags
    reach, against the block, is one circular correlation of 1024 points without wrap-around; the block spectra are
    summed, and one inverse transform gives every lag.  The float64 result is within 1/4 of the integer (checked)."""
    refs, sigs = np.asarray(refs, np.float64), np.asarray(sigs, np.float64)
    K, T = refs.shape
    S = sigs.shape[0]
    assert np.all(np.abs(refs) <= 1024) and np.all(np.abs(sigs) <= 1024) and T <= 1 << 22
    assert np.array_equal(refs, np.round(refs)) and np.array_equal(sigs, np.round(sigs))
    nb = -(-T // L)
    C = np.zeros((L + 1, K, S), np.complex128)
    step = 1024                                          # blocks per pass, to bound the memory
    for b0 in range(0, nb, step):
        b1 = min(nb, b0 + step)
        apad = np.zeros((K, (b1 - b0 + 1) * L))           # refs[(b0 - 1) L ...  b1 L)
        lo = max(0, (b0 - 1) * L)
        hi = min(T, b1 * L)
        apad[:, lo - (b0 - 1) * L:hi - (b0 - 1) * L] = refs[:, lo:hi]
        aseg = sliding_window_view(apad, 2 * L, axis=1)[:, ::L]            # (K, blocks, 1024)
        xblk = np.zeros((S, b1 - b0, 2 * L))
        xs = np.zeros((S, (b1 - b0) * L))
        xs[:, :min(T, b1 * L) - b0 * L] = sigs[:, b0 * L:min(T, b1 * L)]
        xblk[:, :, :L] = xs.reshape(S, b1 - b0, L)
        FA = scipy.fft.rfft(aseg, axis=-1)                 # (K, blocks, 513)
        FX = scipy.fft.rfft(xblk, axis=-1)                 # (S, blocks, 513)
        C += np.matmul(FA.transpose(2, 0, 1), np.conj(FX).transpose(2, 1, 0))
    c = scipy.fft.irfft(C.transpose(1, 2, 0), 2 * L, axis=-1)                 # (K, S, 1024)
    # block b: c[m] = sum_n x_b[n] aseg_b[n + m]; lag d sits at m = 512 - d
    r = c[..., L - np.arange(L)]
    out = np.round(r)
    assert np.abs(r - out).max() < 0.25, np.abs(r - out).max()
    return out


def lag_correlations(refs, sigs, dtype=LD, block=4096):
    """R (K, S, L) with R[a, s, d] = sum_v refs[a, v - d] sigs[s, v], summed in `dtype` (long double by default; pass
    float64 and |signals| for the magnitudes of the terms)"""
    refs, sigs = np.asarray(refs), np.asarray(sigs)
    K, T = refs.shape
    S = sigs.shape[0]
    R = np.zeros((K, S, L), dtype)
    apad = np.concatenate([np.zeros((K, L - 1), dtype), refs.astype(dtype)], axis=1)   # apad[:, j] = refs[:, j - 511]
    for v0 in range(0, T, block):
        v1 = min(T, v0 + block)
        X = sigs[:, v0:v1].astype(dtype)
        for a in range(K):
            A = sliding_window_view(apad[a, v0:v1 + L - 1], v1 - v0)[::-1]        # A[d, v] = refs[a, v0 + v - d]
            R[a] += X @ A.T
    return R


def corr_bound(mag, T):
    """|R - R*| <= u (span + parts) sum |a||b|: one rounding per product along a part's span, one per part of the
    ordered sum (whether m8n8k4 rounds per product or per k-step is not established, so the per-product count is
    taken); mag = lag_correlations(|refs|, |sigs|, float64)"""
    s = bss_shape(T, 1, 1)
    return U * (s['span'] + s['parts']) * mag


def chunked_correlation_model(refs, sigs, T, drop_partial_chunk=False, lag_shift=0, skip_last_part=False):
    """float64 model of bss_corr_kernel + bss_corr_reduce_kernel: per part, the 128-sample chunks in order (each
    chunk's products summed in float64), then the parts in order; the mutations are defects the bound must reject"""
    s = bss_shape(T, 1, 1)
    K, S = refs.shape[0], sigs.shape[0]
    apad = np.concatenate([np.zeros((K, L - 1 + abs(lag_shift))), refs], axis=1)
    off = L - 1 + abs(lag_shift) - lag_shift
    parts = []
    for p in range(s['parts'] - (1 if skip_last_part else 0)):
        acc = np.zeros((K, S, L))
        for v0 in range(p * s['span'], min(T, (p + 1) * s['span']), CHUNK):
            v1 = min(T, v0 + CHUNK)
            if drop_partial_chunk and v1 - v0 < CHUNK:
                continue
            for a in range(K):
                A = sliding_window_view(apad[a, v0 + off - (L - 1):v1 + off], v1 - v0)[::-1]
                acc[a] += sigs[:, v0:v1] @ A.T
        parts.append(acc)
    R = np.zeros((K, S, L))
    for p in parts:
        R += p
    return R


# ---- the augmented systems --------------------------------------------------------------------------------------------
def assemble(R, K, E, block=None):
    """[G | D] of bss_assemble_kernel from R (K, S, L), exact copies of R's entries: G (N, N), D (N, E); or, with
    block = j, the diagonal block G_jj (L, L) and D_j (L, E)"""
    t = np.arange(L)
    dlt = t[:, None] - t[None, :]

    def blk(i, j):
        return np.where(dlt >= 0, R[i, j][np.abs(dlt)], R[j, i][np.abs(dlt)])

    if block is not None:
        return blk(block, block), R[block, K:K + E].T.copy()
    G = np.block([[blk(i, j) for j in range(K)] for i in range(K)])
    D = np.concatenate([R[i, K:K + E].T for i in range(K)], axis=0)
    return G, D


def solve_check(A, D, F):
    """A (n, n), D (n, E): the system; F (n, n + E + ...): the device's in-place factors with c in columns n .. n + E.
    Returns (err, bound, max |l|, growth): per column e, err = ||D - A c||_inf in long double and
    bound = 3 n u || |L| (|U| |c|) ||_inf (Higham, Thm. 9.4: (A + dA) c = D with |dA| <= gamma_3n |L||U|; the infinity
    norm does not depend on the row order, which the device does not store), the largest stored |l| below the diagonal
    and the growth factor max|U| / max|A|."""
    n, E = D.shape
    Fn = F[:, :n]
    c = F[:, n:n + E]
    Lo = np.tril(Fn, -1)
    Up = np.triu(Fn)
    mag = (np.abs(Lo) @ (np.abs(Up) @ np.abs(c))) + np.abs(Up) @ np.abs(c)      # |L| |U| |c| with the unit diagonal
    bound = 3 * n * U * np.abs(mag).max(axis=0)
    cl = c.astype(LD)
    err = np.zeros(E)
    for r0 in range(0, n, 512):
        res = D[r0:r0 + 512].astype(LD) - A[r0:r0 + 512].astype(LD) @ cl
        err = np.maximum(err, np.abs(res).max(axis=0).astype(np.float64))
    return err, bound, float(np.abs(Lo).max()) if n > 1 else 0.0, float(np.abs(Up).max() / np.abs(A).max())


# ---- projections ------------------------------------------------------------------------------------------------------
def _tile_toeplitz(s, t0, t1):
    """(t1 - t0, L) with [t - t0, tau] = s[t - tau] (zero outside 0 <= t - tau < T)"""
    T = s.shape[-1]
    if t1 <= t0:
        return np.zeros((0, L), s.dtype)
    pad = np.zeros(t1 - t0 + L - 1, s.dtype)
    lo, hi = max(0, t0 - (L - 1)), min(T, t1)
    if hi > lo:
        pad[lo - (t0 - (L - 1)):hi - (t0 - (L - 1))] = s[lo:hi]
    return sliding_window_view(pad, L)[:, ::-1]


def tile_energies(sig, K, E, T, c_all, c_one, tiles):
    """Long-double energies of the listed tiles and their bounds.  sig (S, T); c_all (K, L, E) from G's right-hand
    columns, c_one (K, L, E) from the blocks' (c_all again at K = 1, where the device takes P_1 = P_all).
    Returns ref, bound, each (len(tiles), K + 1, 3, E) in the slots of bss_project_kernel: slot j < K: sum P_j^2,
    sum (x - P_j)^2, sum (P_all - P_j)^2; slot K: sum P_all^2, sum (x - P_all)^2, 0.

    Per sample, |P_all - P*_all| <= d_all = u (K L + 1) sum_i sum_tau |c_i,tau| |s_i[t - tau]| (and with L for P_j);
    the differences add one rounding of their value.  A tile's energy of d then errs by at most
    sum_t (2 |d_t| delta_t + delta_t^2) plus the rounding of the tile's own fixed-order sum, 16 u sum_t (|d_t| + delta_t)^2
    (a square, an fma, three shuffle levels and eight warps: 13 roundings deep)."""
    Tp = T + L - 1
    ref = np.zeros((len(tiles), K + 1, 3, E), LD)
    bound = np.zeros((len(tiles), K + 1, 3, E))
    ca, co = c_all.astype(LD), c_one.astype(LD)
    for n, k in enumerate(tiles):
        t0, t1 = k * TILE, min(Tp, (k + 1) * TILE)
        x = np.zeros((t1 - t0, E))
        if t0 < T:
            x[:min(T, t1) - t0] = sig[K:, t0:min(T, t1)].T
        Ss = [_tile_toeplitz(sig[i], t0, t1) for i in range(K)]
        p_all = sum(Ss[i].astype(LD) @ ca[i] for i in range(K))
        m_all = sum(np.abs(Ss[i]) @ np.abs(c_all[i]) for i in range(K))
        d_all = U * (K * L + 1) * m_all
        xl = x.astype(LD)

        def energy(d, delta):
            a = np.abs(d).astype(np.float64)
            return (d * d).sum(axis=0), (2 * a * delta + delta ** 2).sum(axis=0) + 16 * U * ((a + delta) ** 2).sum(axis=0)

        def diff(a, b, delta):
            d = a - b
            return d, delta + U * (np.abs(d).astype(np.float64) + delta)

        for j in range(K):
            if K == 1:
                p_j, d_j = p_all, d_all
            else:
                p_j = Ss[j].astype(LD) @ co[j]
                d_j = U * (L + 1) * (np.abs(Ss[j]) @ np.abs(c_one[j]))
            vals = [(p_j, d_j), diff(xl, p_j, d_j)]
            vals.append((p_all - p_j, np.zeros_like(d_j)) if K == 1 else diff(p_all, p_j, d_all + d_j))
            for q, (d, delta) in enumerate(vals):
                ref[n, j, q], bound[n, j, q] = energy(d, delta)
        for q, (d, delta) in enumerate([(p_all, d_all), diff(xl, p_all, d_all)]):
            ref[n, K, q], bound[n, K, q] = energy(d, delta)
    return ref, bound


def solutions(G, Gb, K, E):
    """c_all (K, L, E) and c_one (K, L, E) from a workspace item's G and Gb"""
    N = K * L
    c_all = G[:, N:N + E].reshape(K, L, E)
    c_one = c_all if K == 1 else Gb[:, :, L:L + E]
    return c_all, c_one


def projection_model(sig, K, E, T, c_all, c_one, tiles, drop_tail=False, tap_shift=0, own_block_from_all=False):
    """float64 model of the tile energies (each P as one float64 product per tile); the mutations are defects the bound
    must reject: the L - 1 samples past T dropped, a tap off by one, P_j taken from c_all's block j"""
    Tp = T if drop_tail else T + L - 1
    out = np.zeros((len(tiles), K + 1, 3, E))
    for n, k in enumerate(tiles):
        t0, t1 = k * TILE, max(k * TILE, min(Tp, (k + 1) * TILE))
        x = np.zeros((t1 - t0, E))
        if t0 < T:
            x[:min(T, t1) - t0] = sig[K:, t0:min(T, t1)].T
        Ss = [_tile_toeplitz(sig[i], t0 - tap_shift, t1 - tap_shift) for i in range(K)]
        p_all = sum(Ss[i] @ c_all[i] for i in range(K))
        for j in range(K):
            cj = c_all[j] if own_block_from_all or K == 1 else c_one[j]
            p_j = p_all if K == 1 else Ss[j] @ cj
            for q, d in enumerate((p_j, x - p_j, p_all - p_j)):
                out[n, j, q] = (d * d).sum(axis=0)
        for q, d in enumerate((p_all, x - p_all)):
            out[n, K, q] = (d * d).sum(axis=0)
    return out


# ---- ratios and the permutation ---------------------------------------------------------------------------------------
def safe_db(num, den):
    """mir_eval's _safe_db, elementwise: +inf where den == 0"""
    num, den = np.broadcast_arrays(np.asarray(num, np.float64), np.asarray(den, np.float64))
    with np.errstate(divide='ignore', invalid='ignore'):
        v = 10 * np.log10(num / den)
    return np.where(den == 0, np.inf, v)


def tile_totals(sums):
    """(K + 1, 3, width) of bss_ratio_kernel: the tiles of (tiles, K + 1, 3, width) added in order"""
    return np.cumsum(sums, axis=0)[-1]


def pairs_from_totals(tot, K, E):
    """sdr, sir, sar (E, K) from the tile totals"""
    j = np.arange(K)
    e = np.arange(E)[:, None]
    sdr = safe_db(tot[j, 0][:, :E].T, tot[j, 1][:, :E].T)
    sir = safe_db(tot[j, 0][:, :E].T, tot[j, 2][:, :E].T)
    sar = safe_db(np.broadcast_to(tot[K, 0][e], (E, K)), np.broadcast_to(tot[K, 1][e], (E, K)))
    return sdr, sir, sar


def permutations(E, K):
    """(E! / (E - K)!, K): itertools.permutations(range(E), K) in its order"""
    return np.array(list(itertools.permutations(range(E), K)), np.int64).reshape(-1, K)


def np_mean_rows(v):
    """np.mean of each row of v (n, K), in numpy's order: sequential below 8 values, pairwise at 8"""
    K = v.shape[1]
    if K < 8:
        s = np.zeros(v.shape[0])
        for k in range(K):
            s = s + v[:, k]
    else:
        s = ((v[:, 0] + v[:, 1]) + (v[:, 2] + v[:, 3])) + ((v[:, 4] + v[:, 5]) + (v[:, 6] + v[:, 7]))
    return s / K


def first_argmax(m):
    """np.argmax: the first NaN if there is one, else the first maximum"""
    nan = np.flatnonzero(np.isnan(m))
    if nan.size:
        return int(nan[0])
    return int(np.flatnonzero(m == m.max())[0])


def select(sir):
    """the selection of bss_ratio_kernel for a pair matrix sir (E, K): (rank, permutation)"""
    E, K = sir.shape
    perms = permutations(E, K)
    with np.errstate(invalid='ignore'):
        means = np_mean_rows(sir[perms, np.arange(K)])
    r = first_argmax(means)
    return r, perms[r]


# ---- signals ----------------------------------------------------------------------------------------------------------
def white(rng, K, E, T):
    s = rng.standard_normal((K, T))
    mix = rng.standard_normal((E, K))
    return s, mix @ s + 0.3 * rng.standard_normal((E, T))


def ar_coloured(rng, K, E, T):
    """AR(2) sources with poles near the unit circle, estimates mixing them with white noise"""
    s = np.stack([scipy.signal.lfilter([1], [1, -1.8 + 0.05 * k, 0.9], rng.standard_normal(T)) for k in range(K)])
    mix = np.eye(E, K) + 0.1 * rng.standard_normal((E, K))
    return s, mix @ s + 0.1 * rng.standard_normal((E, T))


def pivoting(rng, K, E, T):
    """references at scales from 1e-3 to 1e3, strongly correlated with each other (a shared coloured component plus a
    small own part), so that the pivot of most of the first block's columns comes from a lower block"""
    base = scipy.signal.lfilter([1], [1, -1.5, 0.7], rng.standard_normal(T))
    scales = np.logspace(-3, 3, K) if K > 1 else np.ones(1)
    s = np.stack([sc * (base + 0.05 * rng.standard_normal(T)) for sc in scales])
    est = np.stack([s[e % K] / scales[e % K] + 0.2 * rng.standard_normal(T) for e in range(E)])
    return s, est


def integers(rng, K, E, T):
    return rng.integers(-1024, 1025, (K, T)).astype(np.float64), rng.integers(-1024, 1025, (E, T)).astype(np.float64)
