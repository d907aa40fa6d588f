"""Pure-torch restatement of the six differentiable forwards of pb_bss_b200 (framing + torch.fft, torch.linalg.solve,
einsums), so that torch's own autograd gives the reference gradients of the device backward passes.  Runs on CPU or
CUDA tensors in float64 / complex128.  Test infrastructure only, like the rest of oracle/.

Closed forms of the gradients (PyTorch's convention grad z = dL/dRe z + i dL/dIm z) are restated next to the forwards
for the CPU tests that check them against autograd."""
import math

import numpy as np
import scipy.signal
import torch

from . import fft_oracle as FO
from . import linalg_oracle as LO
from . import transform_oracle as TO


def _windows(size, shift, window_length, window, symmetric_window, device):
    wa = TO.analysis_window(size, window, window_length, symmetric_window)
    ws = TO.synthesis_window(wa, shift)
    return torch.from_numpy(wa).to(device), torch.from_numpy(ws).to(device)


def stft(x, size=1024, shift=256, window=scipy.signal.windows.blackman, window_length=None, fading=True, pad=True,
         symmetric_window=False):
    """nara_wpe stft over the last axis of a real tensor: (..., n) -> (..., T, size // 2 + 1)."""
    wl = window_length or size
    wa, _ = _windows(size, shift, window_length, window, symmetric_window, x.device)
    n = x.shape[-1]
    T = TO.num_frames(n, size, shift, window_length, fading, pad)
    off = wl - shift if fading else 0
    total = max(T - 1, 0) * shift + wl
    keep = min(n, total - off)
    padded = torch.nn.functional.pad(x[..., :keep].to(torch.float64), (off, total - off - keep))
    idx = (torch.arange(T, device=x.device)[:, None] * shift + torch.arange(wl, device=x.device)[None, :])
    frames = padded[..., idx] * wa
    return torch.fft.rfft(frames, n=size, dim=-1)


def istft(X, size=1024, shift=256, window=scipy.signal.windows.blackman, fading=True, window_length=None,
          symmetric_window=False):
    """nara_wpe istft: (..., T, size // 2 + 1) -> (..., T shift + wl - shift [- 2 (wl - shift)])."""
    wl = window_length or size
    _, ws = _windows(size, shift, window_length, window, symmetric_window, X.device)
    T = X.shape[-2]
    frames = torch.fft.irfft(X, n=size, dim=-1)[..., :wl] * ws
    full = T * shift + wl - shift
    idx = (torch.arange(T, device=X.device)[:, None] * shift + torch.arange(wl, device=X.device)[None, :]).reshape(-1)
    out = torch.zeros(X.shape[:-2] + (full,), dtype=torch.float64, device=X.device)
    out = out.index_add(-1, idx, frames.reshape(X.shape[:-2] + (T * wl,)))
    if fading:
        out = out[..., wl - shift:full - (wl - shift)]
    return out


def power_spectral_density(observation, mask=None, normalize=True):
    """observation (..., D, T); mask None, (..., T) or (..., K, T) -> (..., D, D) or (..., K, D, D)."""
    y = observation.to(torch.complex128)
    if mask is None:
        return torch.einsum('...dt,...et->...de', y, y.conj()) / y.shape[-1]
    m = mask.to(torch.float64)
    if normalize:
        m = m / torch.clamp(m.sum(-1, keepdim=True), min=1e-10)
    if m.dim() + 1 == y.dim():
        return torch.einsum('...t,...dt,...et->...de', m.to(y.dtype), y, y.conj())
    return torch.einsum('...kt,...dt,...et->...kde', m.to(y.dtype), y, y.conj())


def mvdr_vector_souden(target_psd, noise_psd, ref_channel=None, eps=None):
    """(w, ref_channel): w = mat[..., ref], mat = solve(noise, target) / max(Re tr, eps); the SNR rule picks ref."""
    phi = torch.linalg.solve(noise_psd, target_psd)
    lam = torch.diagonal(phi, dim1=-2, dim2=-1).sum(-1).real[..., None, None]
    eps = np.finfo(np.float64).tiny if eps is None else eps
    mat = phi / torch.clamp(lam, min=eps)
    if ref_channel is None:
        with torch.no_grad():
            num = torch.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), target_psd, mat)
            den = torch.einsum('...FdR,...FdD,...FDR->...R', mat.conj(), noise_psd, mat)
            snr = num / torch.clamp(den.real, min=eps)
            ref_channel = int(torch.argmax(snr.real))
    return mat[..., ref_channel], ref_channel


def apply_beamforming_vector(vector, mix):
    """sum_a conj(vector[..., a]) mix[..., a, t]."""
    return torch.einsum('...a,...at->...t', vector.conj(), mix.to(torch.complex128))


def si_sdr(reference, estimation):
    """10 log10(|alpha r|^2 / |e - alpha r|^2), alpha = <r, e> / <r, r>, over the last axis after broadcasting."""
    e, r = torch.broadcast_tensors(estimation, reference)
    alpha = (r * e).sum(-1, keepdim=True) / (r * r).sum(-1, keepdim=True)
    p = alpha * r
    q = e - p
    return 10 * torch.log10((p * p).sum(-1) / (q * q).sum(-1))


# ---- closed forms of the gradients (restated from include/pbb.h) ----------------------------------------------------

def si_sdr_grad(reference, estimation, grad):
    """(grad r, grad e) of si_sdr for 1-D reference / estimation and a scalar incoming gradient."""
    alpha = (reference @ estimation) / (reference @ reference)
    p = alpha * reference
    q = estimation - p
    P, Q = p @ p, q @ q
    c = 20 / math.log(10) * grad
    return c * alpha * (1 / P + 1 / Q) * q, c * (p / P - q / Q)


def psd_grad(observation, mask, grad_psd, normalize=True):
    """(grad y, grad mask) of power_spectral_density for observation (F, D, T), mask (F, K, T), grad_psd (F, K, D, D)."""
    y = observation.to(torch.complex128)
    S = mask.sum(-1)
    if normalize:
        w = mask / torch.clamp(S, min=1e-10)[..., None]
    else:
        w = mask
    H = grad_psd + grad_psd.conj().transpose(-1, -2)
    gy = torch.einsum('fkt,fkde,fet->fdt', w.to(y.dtype), H, y)
    quad = torch.einsum('fdt,fkde,fet->fkt', y.conj(), grad_psd, y).real
    if not normalize:
        return gy, quad
    phi = power_spectral_density(y, mask, normalize=True)
    c = (grad_psd.conj() * phi).sum((-1, -2)).real
    active = S > 1e-10
    gm = torch.where(active[..., None], (quad - c[..., None]) / S[..., None], quad / 1e-10)
    return gy, gm


def souden_grad(target_psd, noise_psd, ref_channel, grad_w, eps=None):
    """(grad target, grad noise) of mvdr_vector_souden with a fixed reference channel."""
    eps = np.finfo(np.float64).tiny if eps is None else eps
    phi = torch.linalg.solve(noise_psd, target_psd)
    lam = torch.diagonal(phi, dim1=-2, dim2=-1).sum(-1).real
    D = phi.shape[-1]
    e_r = torch.zeros(D, dtype=phi.dtype)
    e_r[ref_channel] = 1
    outer = grad_w[..., :, None] * e_r
    c = (grad_w.conj() * phi[..., :, ref_channel]).sum(-1).real
    eye = torch.eye(D, dtype=phi.dtype)
    gphi = torch.where((lam > eps)[..., None, None], outer / lam[..., None, None] - (c / lam ** 2)[..., None, None] * eye,
                       outer / eps)
    gx = torch.linalg.solve(noise_psd.conj().transpose(-1, -2), gphi)
    gn = -gx @ phi.conj().transpose(-1, -2)
    return gx, gn


# ---- long-double reference gradients and the bounds the device backward passes are held to --------------------------
# u = 2^-53.  The references evaluate the closed forms above in np.longdouble (64-bit mantissa on x86) from the float64
# inputs the device reads; the bounds are first-order rounding-error bounds of the device's order of operations, with
# gamma(n) = n u / (1 - n u) and a factor for complex products.  Each *_ratio function returns error / bound per
# element, bin or sample (<= 1 passes; 0 / inf where the bound is 0, for an exact-zero result).
LD, CLD = np.longdouble, np.clongdouble
U = 2.0 ** -53
U32 = 2.0 ** -24
C_G = 4.0  # complex products and sums (sqrt 2 gamma per product) and a factor 2 of headroom


def gamma(n):
    return n * U / (1 - n * U)


def _ratio(err, bound):
    err, bound = np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err == 0, 0.0, np.inf))


def _err(got, ref):
    return np.abs(np.asarray(got).astype(CLD if np.iscomplexobj(got) or np.iscomplexobj(ref) else LD) - ref)


def _rounded(bound, ref, dtype):
    """bound plus the final rounding of the gradient to dtype (complex64 / float32 gradients are cast from fp64)."""
    if dtype in (np.float32, np.complex64):
        return bound + 2 * U32 * np.abs(ref).astype(np.float64)
    return bound


# ---- stft: grad x_s = sum_t w_a[s' - t shift] Re sum_{k <= size/2} G_tk e^{+2 pi i jk / size}, s' = s + offset ------
def _halved(G, size):
    """G^ (inner bins halved, exact): size irfft(G^)_j = Re sum_{k=0}^{size/2} G_k e^{+2 pi i jk / size}, the imaginary
    parts at DC and Nyquist dropping out as e^{2 pi i jk / size} is real there."""
    Gh = np.array(G, dtype=np.complex128, copy=True)
    Gh[..., 1:size // 2] *= 0.5
    return Gh


def stft_grad_parts(G, n, size, shift, window_length=None, fading=True):
    """(grad x*, scale) of stft for the incoming gradient G (..., T, size // 2 + 1) and a signal of n samples: the
    transpose in long double, frames overlap-added in increasing t and cropped to the signal (samples no frame covers
    get 0), and the per-sample scale of the inverse bound, sum_t |w_a[s' - t shift]| rms(size irfft G^_t).  Error of a
    correct kernel: |grad x_s - grad x*_s| <= C_I u log2(size) scale_s (fft_oracle.inverse_ratio): the device runs
    istft_frames_kernel's inverse body on G^ with exact power-of-two scalings, so the istft bound carries over; a
    sample covered only by all-zero G frames has scale 0 and must be exactly 0."""
    wl = window_length or size
    wa = TO.analysis_window(size, window_length=wl)
    G = np.asarray(G)
    y = np.fft.irfft(_halved(G, size).astype(CLD), n=size, axis=-1) * size
    rms = np.sqrt(np.mean(np.square(y), axis=-1, keepdims=True))
    x = FO._overlap_add(y[..., :wl] * wa.astype(LD), shift)
    scale = FO._overlap_add((rms * np.abs(wa)).astype(np.float64), shift)
    return _crop(x, n, wl - shift if fading else 0), _crop(scale, n, wl - shift if fading else 0)


def _crop(full, n, offset):
    out = np.zeros(full.shape[:-1] + (n,), dtype=full.dtype)
    m = max(min(n, full.shape[-1] - offset), 0)
    out[..., :m] = full[..., offset:offset + m]
    return out


def model_stft_grad(G, n, size, shift, window_length=None, fading=True):
    """stft_backward_kernel + overlap_add_kernel's arithmetic in float64: fft_oracle's inverse model on G^, times size
    (exact), the analysis window, the overlap-add in increasing t and the crop."""
    wl = window_length or size
    G = np.asarray(G, dtype=np.complex128)
    lead, T = G.shape[:-2], G.shape[-2]
    y = FO.model_irfft(_halved(G, size).reshape(-1, size // 2 + 1), size) * size
    x = FO._overlap_add((TO.analysis_window(size, window_length=wl) * y[:, :wl]).reshape(lead + (T, wl)), shift)
    return _crop(x, n, wl - shift if fading else 0)


# ---- istft: grad X_tk = c_k rfft(w_s g_t)_k, c_k = 2 / size (1 / size at DC and Nyquist) --------------------------
def _grad_frames(g, T, shift, wl, crop):
    """(..., T, wl): g_t[j] = g[t shift + j - crop], 0 outside the output."""
    g = np.asarray(g, dtype=np.float64)
    full = np.zeros(g.shape[:-1] + (T * shift + wl - shift,))
    full[..., crop:crop + g.shape[-1]] = g
    return full[..., np.arange(T)[:, None] * shift + np.arange(wl)[None, :]]


def _c(size):
    c = np.full(size // 2 + 1, 2.0 / size)
    c[0] = c[-1] = 1.0 / size
    return c


def istft_grad(g, T, size, shift, window_length=None, fading=True):
    """grad X* (..., T, size // 2 + 1) of istft for the incoming gradient g (..., n_out), in long double.  Error of a
    correct kernel, per frame: the forward bound ||gX_t - gX*_t|| <= C_F u log2(size) ||gX*_t|| (fft_oracle.
    forward_ratio; the scale c_k is a power of two); an all-zero frame exactly zero."""
    wl = window_length or size
    ws = TO.synthesis_window(TO.analysis_window(size, window_length=wl), shift)
    fr = _grad_frames(g, T, shift, wl, wl - shift if fading else 0)
    return np.fft.rfft(fr.astype(LD) * ws.astype(LD), n=size, axis=-1) * _c(size).astype(LD)


def model_istft_grad(g, T, size, shift, window_length=None, fading=True):
    """istft_backward_kernel's arithmetic in float64: fft_oracle's forward model on the synthesis-windowed gradient
    frames, then the power-of-two scaling."""
    wl = window_length or size
    ws = TO.synthesis_window(TO.analysis_window(size, window_length=wl), shift)
    fr = _grad_frames(g, T, shift, wl, wl - shift if fading else 0)
    lead = fr.shape[:-2]
    f = np.zeros((int(np.prod(lead, dtype=np.int64)) * T, size))
    f[:, :wl] = fr.reshape(-1, wl) * ws
    return (FO.model_rfft(f, size) * _c(size)).reshape(lead + (T, size // 2 + 1))


# ---- PSD ------------------------------------------------------------------------------------------------------------
def psd_grad_ld(observation, mask, grad_psd, normalize=True):
    """(grad y*, grad mask*, bound y, bound mask) of power_spectral_density for observation (F, D, T), mask (F, K, T)
    or None (w = 1 / T, K = 1) and grad_psd (F, K, D, D): psd_grad's closed forms in long double, Phi formed exactly
    from y and the mask.  grad mask* is None without a mask.

    Bounds, elementwise (the device: H = G + G^H; u = H y_t in j order; grad y_t += w_kt u over k; q = Re(y^H u);
    S = sum_t m by 32 strided lanes and a butterfly; Re<G, Phi> over D^2 terms with the device's forward Phi, itself
    within gamma(T) sum_t w |y_d| |y_e| of the exact one):
      |grad y - grad y*|   <= C_G gamma(D + K + T_S + 4) sum_k |w_kt| sum_e |H_kde| |y_et|, T_S = T when S is formed;
      |grad m - grad m*|   <= C_G gamma(D^2 + D + T + 8) (A_q / 2 + A_c) / max(S, 1e-10), with
      A_q = sum_de |y_d| |H_de| |y_e| and A_c = sum_de |G_de| sum_t |w_t| |y_dt| |y_et|: the absolute sizes of the
      two terms whose difference Re(y^H G y) - Re<G, Phi> cancels; without normalize (or once the clamp is active)
      A_c drops out and the divisor is 1 (1e-10)."""
    y = np.asarray(observation).astype(np.complex128).astype(CLD)
    F, D, T = y.shape
    G = np.asarray(grad_psd).astype(CLD)
    H = G + np.conj(np.swapaxes(G, -1, -2))
    aH = np.abs(G) + np.abs(np.swapaxes(G, -1, -2))
    ay = np.abs(y)
    if mask is None:
        w = np.full((F, 1, T), LD(1) / T)
        S = None
    else:
        m = np.asarray(mask, dtype=np.float64).astype(LD)
        S = m.sum(-1)
        w = m / np.maximum(S, LD(1e-10))[..., None] if normalize else m
    K = w.shape[1]
    gy = np.einsum('fkt,fkde,fet->fdt', w.astype(CLD), H, y, optimize=True)
    n_y = D + K + 4 + (T if mask is not None and normalize else 0)
    by = C_G * gamma(n_y) * np.einsum('fkt,fkde,fet->fdt', np.abs(w), aH, ay, optimize=True).astype(np.float64)
    if mask is None:
        return gy, None, by, None
    q = np.einsum('fdt,fkde,fet->fkt', np.conj(y), G, y, optimize=True).real
    aq = np.einsum('fdt,fkde,fet->fkt', ay, aH, ay, optimize=True) / 2
    if not normalize:
        return gy, q, by, (C_G * gamma(D * D + D + 8) * aq).astype(np.float64)
    phi = np.einsum('fkt,fdt,fet->fkde', w.astype(CLD), y, np.conj(y), optimize=True)
    c = (np.conj(G) * phi).sum((-1, -2)).real
    ac = np.einsum('fkde,fkt,fdt,fet->fk', np.abs(G), np.abs(w), ay, ay, optimize=True)
    active = S > 1e-10
    gm = np.where(active[..., None], (q - c[..., None]) / np.where(active, S, 1)[..., None], q / LD(1e-10))
    bm = np.where(active[..., None], (aq + ac[..., None]) / np.where(active, S, 1)[..., None], aq / LD(1e-10))
    return gy, gm, by, (C_G * gamma(D * D + D + T + 8) * bm).astype(np.float64)


# ---- Souden MVDR ----------------------------------------------------------------------------------------------------
C_SOUDEN = 8.0


def souden_grad_ref(target_psd, noise_psd, ref_channel, grad_w, eps=None, high_precision=False):
    """(grad target*, grad noise*, bound target, bound noise) per bin for target, noise (n, D, D) and grad_w (n, D).

    Phi = N^-1 X, lambda = Re tr Phi; grad Phi = g e_r^T / lambda - (Re(g^H Phi_r) / lambda^2) I (lambda > eps),
    g e_r^T / eps otherwise, in long double from Phi; then grad X = N^-H grad Phi and grad N = -grad X Phi^H.  The two
    solves are mpmath's lu_solve at linalg_oracle.DPS digits (high_precision; graded or ill-conditioned N) or
    float64 LAPACK (the wide D sweep, where kappa(N) is small and its own error is inside the bound).

    Bound, normwise per bin (Frobenius): the device's Phi carries the forward solve's error, about u D kappa(N) ||Phi||,
    which reaches grad Phi relative to its absolute size |grad Phi| = |g| e_r^T / lambda + (|g|^T |Phi_r| / lambda^2) I;
    the backward solve adds u D kappa(N) relative.  So
      ||grad X - grad X*|| <= C u D kappa(N) ||N^-1||_2 || |grad Phi| ||,   ||grad N - grad N*|| <= that times ||Phi||."""
    eps = np.finfo(np.float64).tiny if eps is None else eps
    X = np.asarray(target_psd, dtype=np.complex128)
    N = np.asarray(noise_psd, dtype=np.complex128)
    g = np.asarray(grad_w, dtype=np.complex128)
    n, D = X.shape[0], X.shape[-1]
    solve = (lambda a, b: LO.mp_solve(a, b).reshape(b.shape)) if high_precision else np.linalg.solve
    gX = np.empty((n, D, D), dtype=np.complex128)
    gN = np.empty((n, D, D), dtype=np.complex128)
    bX = np.empty(n)
    bN = np.empty(n)
    for m in range(n):
        phi = solve(N[m], X[m]).astype(CLD)
        lam = np.trace(phi).real
        gm = g[m].astype(CLD)
        gphi = np.zeros((D, D), dtype=CLD)
        aphi = np.zeros((D, D), dtype=LD)
        if lam > eps:
            gphi[:, ref_channel] = gm / lam
            c = (np.conj(gm) * phi[:, ref_channel]).sum().real
            gphi -= c / lam ** 2 * np.eye(D)
            aphi[:, ref_channel] = np.abs(gm) / lam
            aphi += (np.abs(gm) * np.abs(phi[:, ref_channel])).sum() / lam ** 2 * np.eye(D)
        else:
            gphi[:, ref_channel] = gm / LD(eps)
            aphi[:, ref_channel] = np.abs(gm) / LD(eps)
        gx = solve(np.conj(N[m]).T, gphi.astype(np.complex128)).astype(CLD)
        gX[m] = gx
        gN[m] = -(gx @ np.conj(phi).T)
        sv = np.linalg.svd(N[m], compute_uv=False)
        kappa, ninv = sv[0] / sv[-1], 1 / sv[-1]
        bX[m] = C_SOUDEN * U * D * kappa * ninv * float(np.sqrt((aphi.astype(np.float64) ** 2).sum()))
        bN[m] = bX[m] * float(np.linalg.norm(phi.astype(np.complex128)))
    return gX, gN, bX, bN


def souden_ratio(gX, gN, ref):
    """Per-bin normwise error / bound of (grad target, grad noise) against souden_grad_ref's output."""
    gXr, gNr, bX, bN = ref
    eX = np.sqrt((_err(gX, gXr) ** 2).sum((-1, -2))).astype(np.float64)
    eN = np.sqrt((_err(gN, gNr) ** 2).sum((-1, -2))).astype(np.float64)
    return np.maximum(_ratio(eX, bX), _ratio(eN, bN))


# ---- apply_beamforming_vector ---------------------------------------------------------------------------------------
def apply_grad_ld(vector, mix, grad_out):
    """(grad vector*, grad mix*, bound vector, bound mix) for vector (B, F, D), one mix (F, D, T) shared by the B
    beamformers (B = 1: the plain path) and grad_out (B, F, T), in long double:
      grad w[b,f,a] = sum_t Y[f,a,t] conj(g[b,f,t]),  |error| <= C_G gamma(T) sum_t |Y| |g|;
      grad Y[f,a,t] = sum_b w[b,f,a] g[b,f,t],        |error| <= C_G gamma(B) sum_b |w| |g|
    (gamma(max(., 2)): a single complex product still rounds)."""
    w = np.asarray(vector).astype(np.complex128).astype(CLD)
    Y = np.asarray(mix).astype(np.complex128).astype(CLD)
    g = np.asarray(grad_out).astype(np.complex128).astype(CLD)
    B, T = w.shape[0], Y.shape[-1]
    gw = np.einsum('fat,bft->bfa', Y, np.conj(g))
    gY = np.einsum('bfa,bft->fat', w, g)
    bw = C_G * gamma(max(T, 2)) * np.einsum('fat,bft->bfa', np.abs(Y), np.abs(g)).astype(np.float64)
    bY = C_G * gamma(max(B, 2)) * np.einsum('bfa,bft->fat', np.abs(w), np.abs(g)).astype(np.float64)
    return gw, gY, bw, bY


# ---- SI-SDR ---------------------------------------------------------------------------------------------------------
C_SI_SDR = 4.0


def si_sdr_grad_ld(reference, estimation, grad):
    """(grad r*, grad e*, bound r, bound e) of si_sdr for rows reference, estimation (rows, n) (already broadcast)
    and the incoming gradients grad (rows,): si_sdr_grad's closed form in long double, per element.

    Derivation.  s = 10 log10(P / Q) with alpha = <r, e> / <r, r>, p = alpha r, q = e - p, P = |p|^2, Q = |q|^2, so
    with c = 20 / ln 10:  ds/de = c (p / P - q / Q),  ds/dr = c alpha (1 / P + 1 / Q) q  (the alpha-terms cancel as
    <p, q> = 0 at the exact alpha).  The device forms alpha from chunked sums, p = alpha r and q = e - p rounded
    elementwise, P and Q from chunked sums, then coef = (c g / P, c g / Q).  To first order in u:
      d alpha  <= gamma(n + 2) (sum |r| |e| / <r, r> + |alpha|)              (conditioning of alpha)
      d p_i    <= d alpha |r_i| + u |p_i|,   d q_i <= d p_i + u |q_i|
      d P      <= 2 sum |p| d p + gamma(n) P,   d Q <= 2 sum |q| d q + gamma(n) Q
    and the gradients, each term by its own absolute size (p / P - q / Q cancels where e is close to alpha r):
      |d grad e_i| <= c |g| (d p_i / P + |p_i| d P / P^2 + d q_i / Q + |q_i| d Q / Q^2 + 4 u (|p_i| / P + |q_i| / Q))
      |d grad r_i| <= c |g| (|q_i| (d alpha (1/P + 1/Q) + |alpha| (d P / P^2 + d Q / Q^2 + 4 u (1/P + 1/Q)))
                             + |alpha| (1/P + 1/Q) d q_i).
    The bound is C_SI_SDR times that.  Non-finite rows (P or Q zero, alpha undefined) get an inf bound."""
    r = np.asarray(reference, dtype=np.float64).astype(LD)
    e = np.asarray(estimation, dtype=np.float64).astype(LD)
    g = np.asarray(grad, dtype=np.float64).astype(LD)[:, None]
    n = r.shape[-1]
    with np.errstate(all='ignore'):
        rr = (r * r).sum(-1, keepdims=True)
        alpha = (r * e).sum(-1, keepdims=True) / rr
        p = alpha * r
        q = e - p
        P = (p * p).sum(-1, keepdims=True)
        Q = (q * q).sum(-1, keepdims=True)
        c = LD(20) / np.log(LD(10)) * g
        ge = c * (p / P - q / Q)
        gr = c * alpha * (1 / P + 1 / Q) * q
        ap, aq, ar = np.abs(p), np.abs(q), np.abs(r)
        da = gamma(n + 2) * ((ar * np.abs(e)).sum(-1, keepdims=True) / rr + np.abs(alpha))
        dp = da * ar + U * ap
        dq = dp + U * aq
        dP = 2 * (ap * dp).sum(-1, keepdims=True) + gamma(n) * P
        dQ = 2 * (aq * dq).sum(-1, keepdims=True) + gamma(n) * Q
        ag, aa = np.abs(c), np.abs(alpha)
        be = ag * (dp / P + ap * dP / P ** 2 + dq / Q + aq * dQ / Q ** 2 + 4 * U * (ap / P + aq / Q))
        br = ag * (aq * (da * (1 / P + 1 / Q) + aa * (dP / P ** 2 + dQ / Q ** 2 + 4 * U * (1 / P + 1 / Q)))
                   + aa * (1 / P + 1 / Q) * dq)
    bad = ~(np.isfinite(P) & np.isfinite(Q) & (P > 0) & (Q > 0) & np.isfinite(alpha))
    be = np.where(bad, np.inf, C_SI_SDR * be).astype(np.float64)
    br = np.where(bad, np.inf, C_SI_SDR * br).astype(np.float64)
    return gr, ge, br, be


def reduce_rows(grad, bound, own_index, own_rows):
    """A broadcast operand's gradient: the rows that read own row u summed in increasing row order, their bounds
    summed plus gamma(rows) times the summed absolute values."""
    grad, bound = np.asarray(grad), np.asarray(bound)
    out = np.zeros((own_rows,) + grad.shape[1:], dtype=grad.dtype)
    b = np.zeros((own_rows,) + grad.shape[1:])
    a = np.zeros((own_rows,) + grad.shape[1:])
    for row, u in enumerate(own_index):
        out[u] += grad[row]
        b[u] += bound[row]
        a[u] += np.abs(grad[row]).astype(np.float64)
    counts = np.bincount(np.asarray(own_index), minlength=own_rows).reshape((own_rows,) + (1,) * (grad.ndim - 1))
    return out, b + gamma(np.maximum(counts, 1)) * a
