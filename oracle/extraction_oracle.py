"""NumPy restatement of the multi-source beamformers and vector post-processing of pb_bss/extraction/beamformer.py
(LCMV, WMWF, MERL MVDR, reference channel, condition_covariance, the post-filters, phase_correction and the
time-varying application).  Written from the equations, bin by bin where that is clearer; it checks the fixtures of
oracle/make_golden_extraction.py on the CPU and the device results in the GPU tests.
"""
import numpy as np


def stable_solve(A, B):
    """np.linalg.solve per matrix; an exactly singular matrix gets the minimum-norm least-squares solution."""
    lead = np.broadcast_shapes(A.shape[:-2], B.shape[:-2])
    A = np.broadcast_to(A, lead + A.shape[-2:])
    B = np.broadcast_to(B, lead + B.shape[-2:])
    X = np.empty(lead + (A.shape[-1], B.shape[-1]), dtype=np.result_type(A, B, np.complex128))
    for idx in np.ndindex(*lead):
        try:
            X[idx] = np.linalg.solve(A[idx], B[idx])
        except np.linalg.LinAlgError:
            X[idx] = np.linalg.lstsq(A[idx], B[idx], rcond=None)[0]
    return X


def lcmv_vector(atf, response, noise):
    """w_f = Phi_f^-1 H_f (H_f^H Phi_f^-1 H_f)^-1 r with r rounded to complex64; atf (K, F, D), noise (F, D, D).
    If the K x K system of any bin is exactly singular, the reference solves bin by bin into a complex64 array, so
    then y of every bin is rounded to complex64."""
    K, F, D = atf.shape
    r = np.asarray(response).astype(np.complex64).astype(np.complex128)
    H = np.transpose(atf, (1, 2, 0))                       # (F, D, K)
    X = stable_solve(noise, H)                             # Phi^-1 H
    G = np.conj(np.transpose(H, (0, 2, 1))) @ X            # (F, K, K)
    y = stable_solve(G, np.broadcast_to(r[:, None], (F, K, 1)))[..., 0]
    if any(np.linalg.matrix_rank(G[f], tol=0) < K for f in range(F)):
        y = y.astype(np.complex64).astype(np.complex128)
    return np.einsum('fdk,fk->fd', X, y)


def wmwf_filter(target, noise, distortion_weight=1.):
    phi = stable_solve(noise, target)
    lam = np.einsum('...dd->...', phi)[..., None, None]
    if isinstance(distortion_weight, str):
        return phi / np.sqrt(target[..., :1, :1] * lam)
    return phi / (distortion_weight + lam)


def optimal_reference_channel(w_mat, target, noise, eps=None):
    if eps is None:
        eps = np.finfo(w_mat.dtype).tiny
    num = np.zeros(w_mat.shape[-1], dtype=np.complex128)
    den = np.zeros(w_mat.shape[-1], dtype=np.complex128)
    for f in range(w_mat.shape[0]):
        for R in range(w_mat.shape[-1]):
            w = w_mat[f, :, R]
            num[R] += w.conj() @ target[f] @ w
            den[R] += w.conj() @ noise[f] @ w
    snr = num / np.maximum(den, eps)
    assert np.all(np.isfinite(snr)), snr
    return int(np.argmax(snr.real))


def wmwf_vector(target, noise, reference_channel=None, channel_selection_vector=None, distortion_weight=1.):
    filt = wmwf_filter(target, noise, distortion_weight)
    if channel_selection_vector is not None:
        return (filt * np.asarray(channel_selection_vector)[..., None, :]).sum(-1)
    if reference_channel is None:
        reference_channel = optimal_reference_channel(filt, target, noise)
    return filt[..., reference_channel]


def mvdr_vector_merl(target, noise):
    """(G / trace G)[..., 0] with G = N^-1 T (the reference's summed SNR always selects channel 0)."""
    G = np.linalg.solve(noise, target)
    return G[..., :, 0] / np.einsum('...dd->...', G)[..., None]


def condition_covariance(x, gamma):
    D = x.shape[-1]
    tr = np.einsum('...dd->...', x)
    return (x + gamma * tr[..., None, None] / D * np.eye(D)) / (1 + gamma)


def distortionless_normalization(vector, atf, noise):
    out = np.empty_like(vector, dtype=np.complex128)
    for f in range(vector.shape[0]):
        u = noise[f] @ vector[f]
        out[f] = u * (vector[f].conj() @ atf[f]) / (vector[f].conj() @ u)
    return out


def mvdr_snr_postfilter(vector, target, noise):
    q = lambda M: np.einsum('fa,fab,fb->f', vector.conj(), M, vector)  # noqa: E731
    return (q(target) / q(noise))[:, None]


def zero_degree_normalization(vector, reference_channel):
    ph = np.angle(vector[..., reference_channel])
    return vector * (np.cos(ph) - 1j * np.sin(ph))[..., None]


def phase_correction(vector):
    """Bin f >= 1 times the running product, along axis 0 of the whole array, of the unit phase factors of
    <w_f, w_{f-1}>: over the bins for (F, D), over the leading axis for (K, F, D)."""
    v = np.array(vector, dtype=np.complex128)
    inner = np.sum(v[..., 1:, :].conj() * v[..., :-1, :], axis=-1)
    e = np.exp(1j * np.angle(inner))
    p = np.empty_like(e)
    p[0] = e[0]
    for i in range(1, e.shape[0]):
        p[i] = p[i - 1] * e[i]
    out = v.copy()
    out[..., 1:, :] = v[..., 1:, :] * p[..., None]
    return out


def apply_online_beamforming_vector(vector, mix):
    """out[..., f, t] = sum_d conj(vector[t, f, d]) mix[..., f, d, t]."""
    return np.sum(np.moveaxis(vector, 0, -1).conj() * mix, axis=-2)
