"""Mask-based beamforming on the device, signatures of pb_bss/extraction/beamformer.py.

Shapes follow the reference (beamformer.py:1-12): X (F, D, T), mask (F, K, T),
PSD (F, K, D, D); leading dims are independent.  numpy in -> numpy out, CUDA
tensors in -> CUDA tensors out.  Small matrices are complex128 on the device.

get_power_spectral_density_matrix, get_mvdr_vector_souden, get_gev_vector,
get_pca_vector (every scaling), get_pca (return_all_vecs=False), get_mvdr_vector,
blind_analytic_normalization and apply_beamforming_vector are differentiable for
CUDA tensors that require grad: their backward passes are the device kernels of
pbb_*_backward (fp64, gradients in the input's dtype, double backward raises).

An eigenvector (GEV, PCA) is defined only up to a per-bin phase, which the
device's Jacobi solver picks by its rotation sequence.  Its backward holds that
phase fixed to first order, Im(w^H B dw) = 0, the convention torch.linalg.eigh's
backward assumes.  For a loss that does not change under w -> e^{i theta} w per
bin (w w^H, BAN's output power, a rank-1 estimate) the gradient is exact; for a
phase-dependent loss such as gev+ban -> apply -> istft -> SI-SDR it is the
gradient with each bin's phase held fixed.

The other functions (get_pca(return_all_vecs=True), LCMV, WMWF, MERL and the
vector post-processing) return outputs without a graph.
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _device, _lib
from .linalg import eigh

__all__ = [
    'get_power_spectral_density_matrix',
    'get_pca_vector',
    'get_mvdr_vector',
    'get_mvdr_vector_souden',
    'get_gev_vector',
    'blind_analytic_normalization',
    'apply_beamforming_vector',
    'get_pca',
    'get_mvdr_vector_merl',
    'get_lcmv_vector',
    'get_lcmv_vector_souden',
    'get_wmwf_vector',
    'get_optimal_reference_channel',
    'condition_covariance',
    'distortionless_normalization',
    'mvdr_snr_postfilter',
    'zero_degree_normalization',
    'phase_correction',
    'apply_online_beamforming_vector',
]


def _flat(t, inner):
    """(..., *inner dims) -> (n, *inner dims) contiguous; returns (flat, leading shape)."""
    lead = tuple(t.shape[:t.dim() - inner])
    n = int(np.prod(lead)) if lead else 1
    return t.reshape(n, *t.shape[t.dim() - inner:]).contiguous(), lead


def get_power_spectral_density_matrix(observation, mask=None, sensor_dim=-2,
                                      source_dim=-2, time_dim=-1,
                                      normalize=True):
    """Mask-weighted spatial covariance, beamformer.py:59-160.

    observation: (..., sensors, frames) by default; mask: None, (..., frames)
    or (..., sources, frames).  Returns (..., sensors, sensors) or
    (..., sources, sensors, sensors)."""
    like_numpy = not _device.is_tensor(observation)
    obs = _device.to_device(observation)
    _device.complex_dtype_code(obs)
    nd = obs.dim()
    sensor_dim, source_dim, time_dim = (d % nd - nd for d in (sensor_dim, source_dim, time_dim))
    order = [i for i in range(-nd, 0) if i not in (sensor_dim, time_dim)] + [sensor_dim, time_dim]
    obs = obs.permute(*[i % nd for i in order])
    obs, lead = _flat(obs, 2)
    F, D, T = obs.shape
    single = False
    if mask is None:
        m, K = None, 1
        single = True
    else:
        m = _device.to_device(mask)
        m = m.to(torch.float64)
        if m.dim() + 1 == nd:
            m = m.unsqueeze(-2)
            single = True
        else:
            morder = [i for i in range(-nd, 0) if i not in (source_dim, time_dim)] + [source_dim, time_dim]
            m = m.permute(*[i % nd for i in morder])
        K = m.shape[-2]
        m = m.expand(*lead, K, T).reshape(F, K, T).contiguous()
    psd = _Psd.apply(obs, m, K, bool(normalize))
    if single:
        out = psd.reshape(*lead, D, D)
    else:
        out = psd.reshape(*lead, K, D, D)
        if source_dim < -2:
            # PSD shape (sources, ..., sensors, sensors), beamformer.py:156-158
            out = out.movedim(-3, source_dim % nd)
    return _device.to_host(out.contiguous(), like_numpy)


class _Psd(torch.autograd.Function):
    """observation (F, D, T) complex64 / complex128, mask (F, K, T) float64 or None -> PSD (F, K, D, D) by
    pbb_power_spectral_density; backward pbb_power_spectral_density_backward."""

    @staticmethod
    def forward(ctx, obs, m, K, normalize):
        F, D, T = obs.shape
        code = _device.complex_dtype_code(obs)
        lib = _lib.load()
        psd = _device.empty((F, K, D, D), torch.complex128)
        nbytes = lib.pbb_psd_workspace_bytes(F, T, D, K)
        ws = _device.workspace(nbytes)
        _device.call('pbb_power_spectral_density', obs, code, F, D, T, m, K, int(normalize), psd, ws, nbytes)
        ctx.save_for_backward(obs, m, psd)
        ctx.args = (code, K, normalize)
        return psd

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        obs, m, psd = ctx.saved_tensors
        code, K, normalize = ctx.args
        F, D, T = obs.shape
        need_y, need_m = ctx.needs_input_grad[:2]
        gy = _device.empty((F, D, T), torch.complex128) if need_y else None
        gm = _device.empty((F, K, T), torch.float64) if need_m else None
        if need_y or need_m:
            g = grad.to(torch.complex128).contiguous()
            _device.call('pbb_power_spectral_density_backward', obs, code, F, D, T, m, K, int(normalize), psd, g, gy,
                         gm)
        return None if gy is None else gy.to(obs.dtype), gm, None, None


def _top_eig(psd):
    """(eigenvalue (...), eigenvector (..., D)) of the largest eigenvalue of psd (..., D, D) complex128 on the device,
    through _TopEig."""
    D = psd.shape[-1]
    af, lead = _flat(psd, 2)
    val, vec = _TopEig.apply(af)
    return val.reshape(lead), vec.reshape(*lead, D)


class _TopEig(torch.autograd.Function):
    """a (n, D, D) complex128 -> (the largest eigenvalue (n), its eigenvector (n, D)) of the Hermitian part: the last
    column of pbb_heig_batched; backward pbb_eigenvector_backward without a second matrix (B = I), the phase held
    fixed (include/pbb.h)."""

    @staticmethod
    def forward(ctx, af):
        n, D = af.shape[0], af.shape[-1]
        w = _device.empty((n, D), torch.float64)
        v = _device.empty((n, D, D), torch.complex128)
        status = _status()
        _device.call('pbb_heig_batched', af, n, D, w, v, status)

        def on_error(s):
            raise np.linalg.LinAlgError(f'eigh: non-finite input or no convergence in matrix {s - 1}')
        _device.check_status(status, on_error)
        val, vec = w[:, -1].contiguous(), v[:, :, -1].contiguous()
        ctx.save_for_backward(af, vec)
        return val, vec

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_val, grad_vec):
        af, vec = ctx.saved_tensors
        n, D = vec.shape
        gv = grad_vec.to(torch.complex128).contiguous()
        gl = grad_val.to(torch.float64).contiguous()
        ga = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_eigenvector_backward', af, None, vec, gv, gl, n, D, ga, None)
        return ga


def get_pca_vector(target_psd_matrix, scaling=None):
    """Principal eigenvector of the target PSD, beamformer.py:197-224.  Differentiable for CUDA tensors with respect to
    the target PSD, with the eigenvector's arbitrary per-bin phase held fixed (_TopEig); the scalings are torch ops on
    the eigenvalue and eigenvector."""
    like_numpy = not _device.is_tensor(target_psd_matrix)
    psd = _device.to_device(target_psd_matrix, torch.complex128)
    val, vec = _top_eig(psd)
    if scaling is None:
        pass
    elif scaling == 'trace':
        tr = torch.diagonal(psd, dim1=-2, dim2=-1).sum(-1)
        vec = vec * (torch.sqrt(tr) / torch.linalg.vector_norm(vec, dim=-1))[..., None]
    elif scaling == 'eigenvalue':
        vec = vec * (val / torch.linalg.vector_norm(vec, dim=-1))[..., None]
    else:
        raise ValueError(scaling)
    return _device.to_host(vec.contiguous(), like_numpy)


def get_mvdr_vector(atf_vector, noise_psd_matrix):
    """w = N^-1 a / (a^H N^-1 a), beamformer.py:230-260.
    atf_vector (..., bins, sensors), noise_psd_matrix (bins, sensors, sensors)."""
    assert noise_psd_matrix is not None
    like_numpy = not _device.is_tensor(atf_vector)
    atf = _device.to_device(atf_vector, torch.complex128)
    noise = _device.to_device(noise_psd_matrix, torch.complex128)
    while atf.dim() > noise.dim() - 1:
        noise = noise.unsqueeze(0)
    D = atf.shape[-1]
    lead = torch.broadcast_shapes(atf.shape[:-1], noise.shape[:-2])
    atf_f = atf.expand(*lead, D).reshape(-1, D).contiguous()
    noise_f = noise.expand(*lead, D, D).reshape(-1, D, D).contiguous()
    w = _Mvdr.apply(atf_f, noise_f)
    return _device.to_host(w.reshape(*lead, D), like_numpy)


class _Mvdr(torch.autograd.Function):
    """atf (n, D), noise (n, D, D) complex128 -> w (n, D) by pbb_mvdr; backward pbb_mvdr_backward (a singular noise
    matrix, the forward's minimum-norm branch, gives NaN gradients in its bin)."""

    @staticmethod
    def forward(ctx, atf_f, noise_f):
        n, D = atf_f.shape
        w = _device.empty((n, D), torch.complex128)
        scratch = _device.empty((n, D), torch.complex128)
        status = _status()
        _device.call('pbb_mvdr', atf_f, noise_f, n, D, w, scratch, status)
        # a singular noise PSD matrix takes the reference's np.linalg.lstsq fallback (beamformer.py:251-256) on the
        # device (minimum-norm solution); the status word is only set where that fallback does not exist (D > 40)
        def on_error(s):
            raise np.linalg.LinAlgError(
                f'get_mvdr_vector: singular noise PSD matrix {s - 1} (D > 40: no lstsq fallback)')
        _device.check_status(status, on_error)
        ctx.save_for_backward(atf_f, noise_f, scratch, w)
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        atf_f, noise_f, x, w = ctx.saved_tensors
        n, D = atf_f.shape
        g = grad.to(torch.complex128).contiguous()
        ga = _device.empty((n, D), torch.complex128)
        gn = _device.empty((n, D, D), torch.complex128)
        scratch = _device.empty((n, D), torch.complex128)
        _device.call('pbb_mvdr_backward', atf_f, noise_f, x, w, g, n, D, ga, gn, scratch)
        return ga, gn


def get_gev_vector(target_psd_matrix, noise_psd_matrix, force_cython=False,
                   use_eig=False):
    """Generalised-eigenvalue beamformer, beamformer.py:292-364: eigenvector of
    the largest eigenvalue of (target, noise), LAPACK ``zhegvd`` normalisation.
    ``force_cython`` is accepted for signature parity (there is only the device
    path here); ``use_eig`` (non-Hermitian ``zggev``) is not implemented."""
    assert noise_psd_matrix is not None
    if use_eig:
        raise NotImplementedError('use_eig=True (general eig) is outside the hot path (SURVEY.md section 2)')
    like_numpy = not _device.is_tensor(target_psd_matrix)
    a = _device.to_device(target_psd_matrix, torch.complex128)
    b = _device.to_device(noise_psd_matrix, torch.complex128)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert a.shape[-1] == a.shape[-2], a.shape
    D = a.shape[-1]
    af, lead = _flat(a, 2)
    bf, _ = _flat(b, 2)
    w = _Gev.apply(af, bf)
    return _device.to_host(w.reshape(*lead, D), like_numpy)


class _Gev(torch.autograd.Function):
    """target, noise (n, D, D) complex128 -> the top generalised eigenvector w (n, D), w^H noise w = 1, by
    pbb_gev_batched; backward pbb_eigenvector_backward with the phase held fixed (include/pbb.h)."""

    @staticmethod
    def forward(ctx, af, bf):
        n, D = af.shape[0], af.shape[-1]
        w = _device.empty((n, D), torch.complex128)
        status = _status()
        _device.call('pbb_gev_batched', af, bf, n, D, w, status)

        def on_error(s):
            # get_gev_vector.pyx:130-147 / beamformer.py:398-408
            raise ValueError(f'Error for frequency {s - 1}: noise PSD not positive definite or non-finite input')
        _device.check_status(status, on_error)
        ctx.save_for_backward(af, bf, w)
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        af, bf, w = ctx.saved_tensors
        n, D = w.shape
        g = grad.to(torch.complex128).contiguous()
        ga = _device.empty((n, D, D), torch.complex128)
        gb = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_eigenvector_backward', af, bf, w, g, None, n, D, ga, gb)
        return ga, gb


def get_mvdr_vector_souden(target_psd_matrix, noise_psd_matrix, ref_channel=None,
                           eps=None, return_ref_channel=False):
    """Souden MVDR, beamformer.py:627-698 (+ get_optimal_reference_channel :601-624)."""
    assert noise_psd_matrix is not None
    like_numpy = not _device.is_tensor(target_psd_matrix)
    if isinstance(target_psd_matrix, (list, tuple)):
        target_psd_matrix = np.asarray(target_psd_matrix)
    if isinstance(noise_psd_matrix, (list, tuple)):
        noise_psd_matrix = np.asarray(noise_psd_matrix)
    # real PSD matrices give a real vector in the reference (NumPy keeps the dtype); the device path is complex
    real_in = like_numpy and not np.iscomplexobj(target_psd_matrix) and not np.iscomplexobj(noise_psd_matrix)
    t = _device.to_device(np.asarray(target_psd_matrix) if isinstance(target_psd_matrix, (list, tuple))
                          else target_psd_matrix, torch.complex128)
    nz = _device.to_device(np.asarray(noise_psd_matrix) if isinstance(noise_psd_matrix, (list, tuple))
                           else noise_psd_matrix, torch.complex128)
    D = t.shape[-1]
    tf, lead = _flat(t, 2)
    nf, _ = _flat(nz.expand_as(t), 2)
    n = tf.shape[0]
    if eps is None:
        eps = np.finfo(np.float64).tiny
    chosen = {}
    w = _Souden.apply(tf, nf, ref_channel, float(eps), len(lead), chosen)
    ref_channel = chosen['ref_channel']
    beamformer = _device.to_host(w.reshape(*lead, D), like_numpy)
    if real_in:
        beamformer = np.ascontiguousarray(beamformer.real)
    return (beamformer, ref_channel) if return_ref_channel else beamformer


class _Souden(torch.autograd.Function):
    """target, noise (n, D, D) complex128 -> w = mat[:, ref_channel] (n, D) by pbb_solve_batched + pbb_souden, the
    reference channel given or chosen by the SNR rule (written to chosen['ref_channel']; a constant of the backward,
    pbb_souden_backward)."""

    @staticmethod
    def forward(ctx, tf, nf, ref_channel, eps, lead_dims, chosen):
        n, D = tf.shape[0], tf.shape[-1]
        phi = _device.empty((n, D, D), torch.complex128)
        status = _device.empty((1,), torch.int32)
        status.zero_()
        _device.call('pbb_solve_batched', nf, tf, n, D, D, 0, phi, status)
        # stable_solve (math/solve.py:95-114): singular systems get the minimum-norm (lstsq) solution on the device
        def on_error(s):
            raise np.linalg.LinAlgError(
                f'get_mvdr_vector_souden: singular noise PSD matrix {s - 1} (D > 40: no lstsq fallback)')
        _device.check_status(status, on_error)
        mat = _device.empty((n, D, D), torch.complex128)
        num = _device.empty((n, D), torch.complex128)
        den = _device.empty((n, D), torch.complex128)
        nsum = _device.empty((D,), torch.complex128)
        dsum = _device.empty((D,), torch.complex128)
        _device.call('pbb_souden', phi, tf, nf, n, D, eps, mat, num, den, nsum, dsum)
        if ref_channel is None:
            if lead_dims != 1:
                raise ValueError(
                    'Estimating the ref_channel expects currently that the input '
                    'has 3 ndims (frequency x sensors x sensors). '
                    'Considering an independent dim in the SNR estimate is not unique.')
            ns, ds = nsum.cpu().numpy(), dsum.cpu().numpy()
            snr = ns / np.maximum(ds, eps)
            assert np.all(np.isfinite(snr)), snr
            ref_channel = int(np.argmax(snr.real))
        assert np.isscalar(ref_channel), ref_channel
        chosen['ref_channel'] = ref_channel
        ctx.save_for_backward(phi, nf)
        ctx.args = (int(ref_channel) % D, eps)
        return mat[..., ref_channel].contiguous()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        phi, nf = ctx.saved_tensors
        ref, eps = ctx.args
        n, D = phi.shape[0], phi.shape[-1]
        g = grad.to(torch.complex128).contiguous()
        gt = _device.empty((n, D, D), torch.complex128)
        gn = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_souden_backward', phi, nf, g, n, D, ref, eps, gt, gn)
        return gt, gn, None, None, None, None


def blind_analytic_normalization(vector, noise_psd_matrix):
    """beamformer.py:459-488."""
    like_numpy = not _device.is_tensor(vector)
    v = _device.to_device(vector, torch.complex128)
    nz = _device.to_device(noise_psd_matrix, torch.complex128)
    D = v.shape[-1]
    lead = torch.broadcast_shapes(v.shape[:-1], nz.shape[:-2])
    vf = v.expand(*lead, D).reshape(-1, D).contiguous()
    nf = nz.expand(*lead, D, D).reshape(-1, D, D).contiguous()
    out = _Ban.apply(vf, nf)
    return _device.to_host(out.reshape(*lead, D), like_numpy)


class _Ban(torch.autograd.Function):
    """vector (n, D), noise (n, D, D) complex128 -> the normalised vector (n, D) by pbb_blind_analytic_normalization;
    backward pbb_blind_analytic_normalization_backward."""

    @staticmethod
    def forward(ctx, vf, nf):
        n, D = vf.shape
        out = _device.empty((n, D), torch.complex128)
        _device.call('pbb_blind_analytic_normalization', vf, nf, n, D, out)
        ctx.save_for_backward(vf, nf)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        vf, nf = ctx.saved_tensors
        n, D = vf.shape
        g = grad.to(torch.complex128).contiguous()
        gv = _device.empty((n, D), torch.complex128)
        gn = _device.empty((n, D, D), torch.complex128)
        _device.call('pbb_blind_analytic_normalization_backward', vf, nf, g, n, D, gv, gn)
        return gv, gn


def apply_beamforming_vector(vector, mix):
    """out[..., t] = sum_a conj(vector[..., a]) mix[..., a, t], beamformer.py:572-583."""
    like_numpy = not _device.is_tensor(mix)
    v = _device.to_device(vector, torch.complex128)
    y = _device.to_device(mix)
    _device.complex_dtype_code(y)
    assert v.shape[-1] < 30, (v.shape, y.shape)
    D, T = y.shape[-2], y.shape[-1]
    lead = tuple(torch.broadcast_shapes(v.shape[:-1], y.shape[:-2]))
    ye = y.expand(*lead, D, T)
    # leading dims over which the mix is only broadcast (K beamformers applied to ONE STFT): the kernel reads the one
    # mix for every index instead of a materialised copy per index
    bdims = [i for i in range(len(lead)) if lead[i] > 1 and ye.stride(i) == 0]
    if bdims:
        nb = len(bdims)
        others = [i for i in range(len(lead)) if i not in bdims]
        bshape, oshape = [lead[i] for i in bdims], [lead[i] for i in others]
        B, F = int(np.prod(bshape)), int(np.prod(oshape)) if others else 1
        ve = v.expand(*lead, D).permute(*bdims, *others, len(lead)).reshape(B, F, D).contiguous()
        ysmall = ye[tuple(0 if i in bdims else slice(None) for i in range(len(lead)))].reshape(F, D, T).contiguous()
        out = _Apply.apply(ve, ysmall, True)
        out = out.reshape(*bshape, *oshape, T)
        if bdims != list(range(nb)):
            out = out.permute(*np.argsort(bdims + others).tolist(), len(lead)).contiguous()
        return _device.to_host(out, like_numpy)
    vf = v.expand(*lead, D).reshape(-1, D).contiguous()
    yf = ye.reshape(-1, D, T).contiguous()
    out = _Apply.apply(vf, yf, False)
    return _device.to_host(out.reshape(*lead, T), like_numpy)


class _Apply(torch.autograd.Function):
    """vector (F, D) complex128, mix (F, D, T) complex64 / complex128 -> (F, T) by pbb_apply_beamforming_vector, or
    (shared) vector (B, F, D) and one mix (F, D, T) -> (B, F, T) by pbb_apply_beamforming_vector_shared; backward
    pbb_apply_beamforming_vector[_shared]_backward."""

    @staticmethod
    def forward(ctx, v, y, shared):
        code = _device.complex_dtype_code(y)
        F, D, T = y.shape
        if shared:
            B = v.shape[0]
            out = _device.empty((B, F, T), torch.complex128)
            _device.call('pbb_apply_beamforming_vector_shared', v, y, code, B, F, D, T, out)
        else:
            out = _device.empty((F, T), torch.complex128)
            _device.call('pbb_apply_beamforming_vector', v, y, code, F, D, T, out)
        ctx.save_for_backward(v, y)
        ctx.args = (code, shared)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        v, y = ctx.saved_tensors
        code, shared = ctx.args
        F, D, T = y.shape
        need_v, need_y = ctx.needs_input_grad[:2]
        gv = _device.empty(v.shape, torch.complex128) if need_v else None
        gy = _device.empty((F, D, T), torch.complex128) if need_y else None
        if need_v or need_y:
            g = grad.to(torch.complex128).contiguous()
            if shared:
                _device.call('pbb_apply_beamforming_vector_shared_backward', v, y, code, v.shape[0], F, D, T, g, gv, gy)
            else:
                _device.call('pbb_apply_beamforming_vector_backward', v, y, code, F, D, T, g, gv, gy)
        return gv, None if gy is None else gy.to(y.dtype), None


def _status():
    s = _device.empty((1,), torch.int32)
    s.zero_()
    return s


def _tiny(*arrays):
    """np.finfo(dtype).tiny of the dtype the reference computes in (float32's tiny for complex64 inputs)."""
    def np_dtype(a):
        if _device.is_tensor(a):
            return np.dtype(str(a.dtype).replace('torch.', ''))
        return np.asarray(a).dtype
    return np.finfo(np.result_type(*[np_dtype(a) for a in arrays])).tiny


def get_pca(target_psd_matrix, return_all_vecs=False):
    """All principal components and eigenvalues, beamformer.py:163-194: (eigenvectors, eigenvalues) with
    return_all_vecs, else the eigenvector of the largest eigenvalue (..., D) and that eigenvalue (...).  Without
    return_all_vecs a tensor input is differentiable in both outputs (_TopEig, the eigenvector's phase held fixed);
    return_all_vecs=True returns outputs without a graph."""
    if not return_all_vecs and _device.is_tensor(target_psd_matrix):
        val, vec = _top_eig(_device.to_device(target_psd_matrix, torch.complex128))
        return vec, val
    w, v = eigh(target_psd_matrix)
    if return_all_vecs:
        return v, w
    vec, val = v[..., -1], w[..., -1]
    if _device.is_tensor(vec):
        vec, val = vec.contiguous(), val.contiguous()
    return vec, val


def get_optimal_reference_channel(w_mat, target_psd_matrix, noise_psd_matrix, eps=None):
    """Reference channel of the largest summed SNR, beamformer.py:601-624.  w_mat, target, noise (F, D, D).
    The per-bin quadratic forms and their sums over the bins run on the device; the D sums come to the host for the
    division by max(den, eps) (NumPy's complex maximum), the finiteness assertion and the argmax."""
    if np.ndim(w_mat) != 3:
        raise ValueError(
            'Estimating the ref_channel expects currently that the input '
            'has 3 ndims (frequency x sensors x sensors). '
            'Considering an independent dim in the SNR estimate is not '
            'unique.')
    if eps is None:
        eps = _tiny(w_mat)
    w = _device.to_device(w_mat, torch.complex128)
    n, D, _ = w.shape
    t = _device.to_device(target_psd_matrix, torch.complex128).expand(n, D, D).contiguous()
    nz = _device.to_device(noise_psd_matrix, torch.complex128).expand(n, D, D).contiguous()
    num = _device.empty((n, D), torch.complex128)
    den = _device.empty((n, D), torch.complex128)
    nsum = _device.empty((D,), torch.complex128)
    dsum = _device.empty((D,), torch.complex128)
    _device.call('pbb_reference_channel_snr', w, t, nz, n, D, num, den, nsum, dsum)
    ns, ds = nsum.cpu().numpy(), dsum.cpu().numpy()
    snr = ns / np.maximum(ds, eps)
    assert np.all(np.isfinite(snr)), snr
    return int(np.argmax(snr.real))


def get_mvdr_vector_merl(target_psd_matrix, noise_psd_matrix):
    """MVDR variant of MERL TR2016-072, beamformer.py:263-289.  target, noise (F, D, D) -> (F, D).

    G = solve(noise, target) with np.linalg.solve (an exactly singular noise matrix raises
    np.linalg.LinAlgError, there is no lstsq fallback), h = G / trace(G).  The reference then picks the channel of
    the largest post-SNR, but its np.sum over the per-channel einsum output sums the channels as well, so the SNR is
    a scalar and the argmax is always 0: the result is h[..., 0], the WMWF filter with distortion_weight = 0 at
    channel 0.  This is reproduced, and no SNR is computed."""
    like_numpy = not _device.is_tensor(target_psd_matrix)
    t = _device.to_device(target_psd_matrix, torch.complex128)
    nz = _device.to_device(noise_psd_matrix, torch.complex128)
    if t.dim() != 3 or nz.dim() != 3:
        raise ValueError('einstein sum subscripts string contains too many subscripts for operand 1: '
                         f'target {tuple(t.shape)} and noise {tuple(nz.shape)} must be (bins, sensors, sensors)')
    if t.shape != nz.shape or t.shape[-1] != t.shape[-2]:
        raise ValueError(f'shape mismatch: target {tuple(t.shape)}, noise {tuple(nz.shape)}')
    n, D, _ = t.shape
    w = _device.empty((n, D), torch.complex128)
    scratch = _device.empty((n, D, D), torch.complex128)
    status = _status()
    _device.call('pbb_mvdr_merl', t, nz, n, D, w, scratch, status)

    def on_error(s):
        raise np.linalg.LinAlgError(f'Singular matrix (get_mvdr_vector_merl: noise PSD matrix of bin {s - 1})')
    _device.check_status(status, on_error)
    return _device.to_host(w, like_numpy)


def get_lcmv_vector(atf_vectors, response_vector, noise_psd_matrix):
    """LCMV beamformer, beamformer.py:414-456.  atf_vectors (K, F, D), response_vector (K,), noise_psd_matrix
    (F, D, D) -> (F, D).  Like the reference the response is rounded to complex64, so H^H w meets
    float32(response), and both solves have stable_solve semantics (an exactly singular system takes its
    minimum-norm solution)."""
    like_numpy = not _device.is_tensor(atf_vectors)
    a = _device.to_device(atf_vectors, torch.complex128)
    if a.dim() != 3:
        raise ValueError(f'not enough values to unpack (expected 3, got {a.dim()})' if a.dim() < 3
                         else f'too many values to unpack (expected 3, got {a.dim()})')
    K, F, D = a.shape
    nz = _device.to_device(noise_psd_matrix, torch.complex128)
    assert tuple(nz.shape) == (F, D, D), nz.shape
    r = _device.to_device(response_vector if _device.is_tensor(response_vector) else np.asarray(response_vector),
                          torch.complex128).reshape(-1)
    if r.numel() != K:
        raise ValueError(f'response_vector has {r.numel()} entries for {K} ATF vectors')
    w = _device.empty((F, D), torch.complex128)
    scratch = _device.empty((F * (2 * D * K + K * K + 2 * K) + 1,), torch.complex128)
    status = _status()
    _device.call('pbb_lcmv', a, r, nz, K, F, D, w, scratch, status)

    def on_error(s):
        raise np.linalg.LinAlgError(f'get_lcmv_vector: singular system in bin {s - 1} (D or K > 40: no lstsq fallback)')
    _device.check_status(status, on_error)
    return _device.to_host(w, like_numpy)


def get_lcmv_vector_souden(target_psd_matrix, interference_psd_matrix, noise_psd_matrix, ref_channel=None,
                           eps=None, return_ref_channel=False):
    """beamformer.py:756-787: not implemented in the reference either, which raises before computing anything."""
    raise NotImplementedError(
        'This is not yet thoroughly tested. It also misses the response vector,'
        'thus it is unclear, how to select, which speaker to attend to.'
    )


def get_wmwf_vector(target_psd_matrix, noise_psd_matrix, reference_channel=None, channel_selection_vector=None,
                    distortion_weight=1.):
    """Speech distortion weighted multichannel Wiener filter, beamformer.py:701-753.

    phi = stable_solve(noise, target), lambda = trace(phi); the filter is phi / (distortion_weight + lambda) or, with
    distortion_weight='frequency_dependent', phi / sqrt(target[..., 0, 0] * lambda).  Then the channel_selection_vector
    weighted sum over the columns, or column reference_channel (chosen by get_optimal_reference_channel when None)."""
    assert noise_psd_matrix is not None
    like_numpy = not _device.is_tensor(target_psd_matrix)
    t = _device.to_device(target_psd_matrix, torch.complex128)
    nz = _device.to_device(noise_psd_matrix, torch.complex128)
    D = t.shape[-1]
    lead = tuple(torch.broadcast_shapes(t.shape[:-2], nz.shape[:-2]))
    tf = t.expand(*lead, D, D).reshape(-1, D, D).contiguous()
    nf = nz.expand(*lead, D, D).reshape(-1, D, D).contiguous()
    n = tf.shape[0]
    frequency_dependent = isinstance(distortion_weight, str)
    if frequency_dependent and distortion_weight != 'frequency_dependent':
        raise TypeError(f'distortion_weight must be a number or "frequency_dependent", got {distortion_weight!r}')
    mu = 0.0 if frequency_dependent else float(distortion_weight)
    filt = _device.empty((n, D, D), torch.complex128)
    scratch = _device.empty((n, D, D), torch.complex128)
    status = _status()
    _device.call('pbb_wmwf', tf, nf, n, D, int(frequency_dependent), mu, filt, scratch, status)

    def on_error(s):
        raise np.linalg.LinAlgError(f'get_wmwf_vector: singular noise PSD matrix {s - 1} (D > 40: no lstsq fallback)')
    _device.check_status(status, on_error)
    filt = filt.reshape(*lead, D, D)
    if channel_selection_vector is not None:
        sel = _device.to_device(channel_selection_vector, torch.complex128)[..., None, :]
        shape = tuple(torch.broadcast_shapes(filt.shape, sel.shape))
        ff = filt.expand(shape).reshape(-1, D, D).contiguous()
        sf = sel.expand(shape).reshape(-1, D, D).contiguous()
        out = _device.empty((ff.shape[0], D), torch.complex128)
        _device.call('pbb_weighted_channel_sum', ff, sf, ff.shape[0], D, out)
        return _device.to_host(out.reshape(shape[:-1]), like_numpy)
    if reference_channel is None:
        reference_channel = get_optimal_reference_channel(filt, tf.reshape(*lead, D, D), nf.reshape(*lead, D, D),
                                                          eps=_tiny(target_psd_matrix, noise_psd_matrix))
    assert np.isscalar(reference_channel), reference_channel
    return _device.to_host(filt[..., reference_channel].contiguous(), like_numpy)


def condition_covariance(x, gamma):
    """(x + gamma * trace(x) / D * I) / (1 + gamma) with the complex trace, beamformer.py:563-569; x (..., D, D)."""
    like_numpy = not _device.is_tensor(x)
    xd = _device.to_device(x, torch.complex128)
    D = xd.shape[-1]
    xf, lead = _flat(xd, 2)
    out = _device.empty(xf.shape, torch.complex128)
    _device.call('pbb_condition_covariance', xf, xf.shape[0], D, float(gamma), out)
    return _device.to_host(out.reshape(*lead, D, D), like_numpy)


def _bins(name, t, ndim):
    if t.dim() != ndim:
        raise ValueError(f'{name} must have {ndim} dims (the reference einsum subscripts are fixed), '
                         f'got shape {tuple(t.shape)}')
    return t


def distortionless_normalization(vector, atf_vector, noise_psd_matrix):
    """N w w^H a / (w^H N w), beamformer.py:491-499.  vector, atf_vector (F, D), noise_psd_matrix (F, D, D)."""
    like_numpy = not _device.is_tensor(vector)
    v = _bins('vector', _device.to_device(vector, torch.complex128), 2)
    a = _bins('atf_vector', _device.to_device(atf_vector, torch.complex128), 2)
    nz = _bins('noise_psd_matrix', _device.to_device(noise_psd_matrix, torch.complex128), 3)
    F, D = v.shape
    if a.shape != v.shape or tuple(nz.shape) != (F, D, D):
        raise ValueError(f'shape mismatch: {tuple(v.shape)}, {tuple(a.shape)}, {tuple(nz.shape)}')
    out = _device.empty((F, D), torch.complex128)
    _device.call('pbb_distortionless_normalization', v, a, nz, F, D, out)
    return _device.to_host(out, like_numpy)


def mvdr_snr_postfilter(vector, target_psd_matrix, noise_psd_matrix):
    """(w^H T w) / (w^H N w) per bin, beamformer.py:502-509.  vector (F, D), PSDs (F, D, D) -> (F, 1)."""
    like_numpy = not _device.is_tensor(vector)
    v = _bins('vector', _device.to_device(vector, torch.complex128), 2)
    t = _bins('target_psd_matrix', _device.to_device(target_psd_matrix, torch.complex128), 3)
    nz = _bins('noise_psd_matrix', _device.to_device(noise_psd_matrix, torch.complex128), 3)
    F, D = v.shape
    if tuple(t.shape) != (F, D, D) or tuple(nz.shape) != (F, D, D):
        raise ValueError(f'shape mismatch: {tuple(v.shape)}, {tuple(t.shape)}, {tuple(nz.shape)}')
    out = _device.empty((F, 1), torch.complex128)
    _device.call('pbb_mvdr_snr_postfilter', v, t, nz, F, D, out)
    return _device.to_host(out, like_numpy)


def zero_degree_normalization(vector, reference_channel):
    """vector * exp(-1j * angle(vector[..., reference_channel])), beamformer.py:512-514; vector (..., D)."""
    like_numpy = not _device.is_tensor(vector)
    v = _device.to_device(vector, torch.complex128)
    D = v.shape[-1]
    ref = int(reference_channel)
    if not -D <= ref < D:
        raise IndexError(f'index {ref} is out of bounds for axis {v.dim() - 1} with size {D}')
    vf, lead = _flat(v, 1)
    out = _device.empty(vf.shape, torch.complex128)
    _device.call('pbb_zero_degree_normalization', vf, vf.shape[0], D, ref % D, out)
    return _device.to_host(out.reshape(*lead, D), like_numpy)


def phase_correction(vector):
    """Phase correction of consecutive bins, beamformer.py:517-560; vector (..., bins, sensors), not modified.

    Bin f >= 1 is multiplied by the cumulative product of exp(1j * angle(sum_d conj(w_f) w_{f-1})).  The reference
    takes that product along axis 0 of the whole array, and so does this: for an (F, D) input it runs over the bins,
    for a (K, F, D) input over K, for every bin on its own.  Real input raises a TypeError, as NumPy's in-place
    complex multiplication does in the reference."""
    like_numpy = not _device.is_tensor(vector)
    if like_numpy:
        vector = np.asarray(vector)
        complex_in = np.iscomplexobj(vector)
    else:
        complex_in = vector.is_complex()
    if not complex_in:
        raise TypeError(f"Cannot cast ufunc 'multiply' output from dtype('complex128') to the real input's dtype "
                        f"({vector.dtype}) with casting rule 'same_kind'")
    v = _device.to_device(vector, torch.complex128)
    if v.dim() < 2:
        raise IndexError('too many indices for array: phase_correction needs (..., bins, sensors)')
    F, D = v.shape[-2:]
    if v.dim() == 2:
        A, M, scan = 1, 1, 1
    else:
        A, M, scan = v.shape[0], int(np.prod(v.shape[1:-2])), 0
    out = _device.empty(tuple(v.shape), torch.complex128)
    if out.numel() == 0:
        return _device.to_host(out, like_numpy)
    _device.call('pbb_phase_correction', v, A, M, F, D, scan, out)
    return _device.to_host(out, like_numpy)


def apply_online_beamforming_vector(vector, mix):
    """Time-varying beamforming, beamformer.py:586-598: out[..., f, t] = sum_d conj(vector[t, f, d]) mix[..., f, d, t].

    vector (T, F, D); mix (..., F, D, T) complex64 or complex128 -> (..., F, T) complex128.  The leading dims of the
    mix are read in place by one launch that reads the vector once; a mix that is only broadcast over a leading dim
    (stride 0) is not copied either."""
    like_numpy = not _device.is_tensor(mix)
    v = _device.to_device(vector, torch.complex128)
    if v.dim() != 3:
        raise ValueError("axes don't match array: vector must be (frames, bins, sensors)")
    y = _device.to_device(mix)
    code = _device.complex_dtype_code(y)
    T, Fv, D = v.shape
    if y.dim() < 2 or y.shape[-2] != D or y.shape[-1] != T:
        raise ValueError(f'operands could not be broadcast together: vector {tuple(v.shape)}, mix {tuple(y.shape)}')
    lead = tuple(torch.broadcast_shapes((Fv,), y.shape[:-2]))
    F = lead[-1]
    B = int(np.prod(lead[:-1])) if len(lead) > 1 else 1
    ye = y.expand(*lead, D, T).reshape(B, F, D, T)
    if ye.stride(2) != T or ye.stride(3) != 1:
        ye = ye.contiguous()
    out = _device.empty((B, F, T), torch.complex128)
    _device.call('pbb_apply_online_beamforming_vector', v, ye, code, B, F, D, T, Fv * D, D if Fv == F else 0,
                 ye.stride(0), ye.stride(1), out)
    return _device.to_host(out.reshape(*lead, T), like_numpy)
