"""Seeded synthetic inputs shared by tests, the golden generator and bench.py's
CPU-baseline leg (TEST INFRASTRUCTURE, see oracle/__init__.py).

Shapes and seeds follow SURVEY.md section 8(d).
"""
import numpy as np


def noise_stft(F, T, D, seed=0, dtype=np.complex128):
    """Throughput input: iid complex Gaussian STFT (F, T, D)."""
    rng = np.random.RandomState(seed)
    y = rng.randn(F, T, D) + 1j * rng.randn(F, T, D)
    return y.astype(dtype)


def init_affiliation(F, K, T, seed=7):
    """Explicit EM initialisation (F, K, T), normalised over K."""
    a = np.random.RandomState(seed).uniform(size=(F, K, T))
    return a / a.sum(-2, keepdims=True)


def structured_stft(F, T, D, K, seed=0, dtype=np.complex128):
    """Parity input: per bin a K-class cACG mixture with rank-1-plus-sigma*I
    covariances (sigma 0.05 for sources, 1.0 for the last, noise-like class).
    Returns (y (F, T, D), labels (F, T))."""
    weights = {2: [0.6, 0.4], 3: [0.4, 0.35, 0.25], 4: [0.3, 0.3, 0.2, 0.2]}
    w = np.asarray(weights.get(K, np.full(K, 1 / K)))
    y = np.zeros((F, T, D), dtype=np.complex128)
    labels = np.zeros((F, T), dtype=np.int64)
    for f in range(F):
        rng = np.random.RandomState(seed * 100003 + f)
        lab = rng.choice(K, size=T, p=w)
        for k in range(K):
            a = rng.randn(D) + 1j * rng.randn(D)
            a /= np.linalg.norm(a)
            sigma = 1.0 if k == K - 1 else 0.05
            cov = np.outer(a, a.conj()) + sigma * np.eye(D)
            chol = np.linalg.cholesky(cov)
            n = int(np.sum(lab == k))
            x = (rng.randn(n, D) + 1j * rng.randn(n, D)) / np.sqrt(2)
            y[f, lab == k] = x @ chol.T
        # arbitrary per-frame scale: the models are scale invariant
        y[f] *= rng.uniform(0.5, 2.0, size=(T, 1))
        labels[f] = lab
    return y.astype(dtype), labels


def permuted_mask(K, F, T, seed=0, noise=0.35):
    """Permutation-alignment input: well-separated class masks proto**4 + noise
    (normalised over K), each bin's classes shuffled.  Returns (mask, clean,
    perm) with mask = clean[perm, range(F)], all (K, F, ...)."""
    rng = np.random.RandomState(seed)
    proto = rng.uniform(size=(K, 1, T)) ** 4
    clean = proto + noise * rng.uniform(size=(K, F, T))
    clean /= clean.sum(0, keepdims=True)
    perm = np.stack([rng.permutation(K) for _ in range(F)], axis=1)
    return clean[perm, np.arange(F)], clean, perm


def pos_def_hermitian(*shape, seed=0):
    """Random Hermitian positive definite matrices (..., D, D)."""
    rng = np.random.RandomState(seed)
    D = shape[-1]
    a = rng.randn(*shape[:-2], D, 2 * D) + 1j * rng.randn(*shape[:-2], D, 2 * D)
    return a @ a.conj().swapaxes(-1, -2) / (2 * D)
