"""GPU checks of the STOI / ESTOI backward (pb_bss_b200.evaluation.stoi on CUDA tensors that require grad, include/pbb.h
pbb_stoi_backward): gradcheck at 8, 10 and 16 kHz; parity with torch autograd of the restatement
(oracle/stoi_autograd_oracle.py) on the GPU over frame counts around the 30-frame limit and the 64-segment blocks,
silence gaps, active and inactive clipping, a long row, a broadcast reference, float32 input and a group split; the
invariants (bitwise forward, repeatable backward, dtypes, no double backward, no host synchronisation) and the
degenerate rows; and the mask -> iSTFT -> -STOI training chain.

Parity bound: per row, ||g_dev - g_ref|| <= TOL ||g_ref|| (2-norms over the row's samples).  Both sides compute the
same fp64 function in different summation orders (the resampler as one convolution against the polyphase gather,
torch's FFT and reductions against the device's fixed trees), so each intermediate differs by a few ulps of its
operands' magnitudes; the derivative chain is well conditioned away from clip ties and the VAD threshold, which the
inputs avoid, so the gradients differ by O(depth u) relative to their norm.  The largest difference measured on an
H100 is 1.1e-14 (a 48 kHz row with gaps); the 2^20-sample row gives 2.1e-15.  TOL = 1e-11 is about 10^5 u."""
import numpy as np
import pytest
import scipy.signal
import torch

from oracle import stoi_autograd_oracle as A

pytestmark = pytest.mark.gpu

TOL = 1e-11


def signals(rng, n, fs, rows=1, gaps=(), swing=0.9):
    """(rows, n) reference and estimate: coloured noise under a square envelope (amplitudes 1 -/+ swing; segments
    with the clip active and inactive, every frame far above the 40 dB threshold), zero over the fractions `gaps`;
    the estimate adds white noise."""
    t = np.arange(n) / fs
    xs, ys = [], []
    for _ in range(rows):
        env = 1 + swing * np.sign(np.sin(2 * np.pi * 4 * t + rng.uniform(0, 6)))
        x = scipy.signal.lfilter([1.0], [1.0, -1.3, 0.6], rng.standard_normal(n)) * env
        for a, b in gaps:
            x[int(a * n):int(b * n)] = 0.0
        xs.append(x)
        ys.append(x + 0.7 * rng.standard_normal(n))
    return np.array(xs), np.array(ys)


def length_for_stft_frames(M, fs):
    """n whose length at 10 kHz has M + 1 frames (M STFT frames when every frame is kept)."""
    from pb_bss_b200.evaluation import module_stoi as MS
    L = 256 + 128 * M + 1
    up, down = MS.rates(fs)
    n = -(-L * down // up)
    assert A.num_frames(MS.resampled_length(n, fs)) == M + 1
    return n


def cuda(a, dtype=torch.float64, grad=True):
    return torch.tensor(a, dtype=dtype, device='cuda').requires_grad_(grad)


def device_grads(x, y, fs, extended, w):
    from pb_bss_b200.evaluation import stoi
    v = stoi(x, y, fs, extended=extended)
    gx, gy = torch.autograd.grad((v * w).sum(), (x, y))
    return v, gx, gy


def reference_grads(x, y, fs, extended, w):
    xr = x.detach().to(torch.float64).expand(torch.broadcast_shapes(x.shape, y.shape)).requires_grad_()
    yr = y.detach().to(torch.float64).expand(xr.shape).requires_grad_()
    v, K, M = A.stoi(xr.reshape(-1, xr.shape[-1]), yr.reshape(-1, yr.shape[-1]), fs, extended)
    gx = gy = None                  # every row on the 1e-5 path: no graph, zero gradients
    if v.requires_grad:
        gx, gy = torch.autograd.grad((v.reshape(w.shape) * w).sum(), (xr, yr), allow_unused=True)
    gx = torch.zeros_like(xr) if gx is None else gx
    gy = torch.zeros_like(yr) if gy is None else gy
    return v, gx.sum_to_size(x.shape), gy.sum_to_size(y.shape), K, M


def assert_rows_close(got, ref, tol=TOL):
    got = got.detach().to(torch.float64).reshape(-1, got.shape[-1])
    ref = ref.reshape(-1, ref.shape[-1])
    err = torch.linalg.vector_norm(got - ref, dim=-1)
    scale = torch.linalg.vector_norm(ref, dim=-1)
    assert torch.isfinite(err).all(), err
    assert (err <= tol * scale).all(), (err / scale).tolist()


def check_parity(x, y, fs, extended, tol=TOL, lead=None):
    from pb_bss_b200.evaluation import module_stoi as MS
    lead = torch.broadcast_shapes(x.shape, y.shape)[:-1] if lead is None else lead
    w = torch.linspace(0.5, 1.5, int(np.prod(lead)), dtype=torch.float64, device='cuda').reshape(lead)
    v, gx, gy = device_grads(x, y, fs, extended, w)
    vr, rx, ry, K, M = reference_grads(x, y, fs, extended, w)
    assert gx.dtype == x.dtype and gy.dtype == y.dtype
    shape = torch.broadcast_shapes(x.shape, y.shape)
    xo, yo = MS._operands(x.detach(), y.detach(), shape)
    frames = MS._stages(xo, yo, fs)['frames'].cpu().numpy()
    np.testing.assert_array_equal(frames, np.array([K, M]).T)
    torch.testing.assert_close(v.reshape(-1), vr.reshape(-1), rtol=0, atol=1e-12)
    assert_rows_close(gx, rx, tol)
    assert_rows_close(gy, ry, tol)
    return K, M


def clip_states(x, y, fs):
    """(any segment entry clipped, any not clipped) of the restatement's STOI for 1-D x, y."""
    out = A.stoi_row(torch.as_tensor(x, device='cuda'), torch.as_tensor(y, device='cuda'), fs)
    xs = out['x_tob'].unfold(1, 30, 1)
    ys = out['y_tob'].unfold(1, 30, 1)
    c = torch.linalg.vector_norm(xs, dim=-1, keepdim=True) / (torch.linalg.vector_norm(ys, dim=-1, keepdim=True)
                                                               + A.EPS)
    clipped = ys * c >= xs * A.CLIP
    return bool(clipped.any()), bool((~clipped).any())


@pytest.mark.parametrize('extended', [False, True])
@pytest.mark.parametrize('fs', [8000, 10000, 16000])
def test_gradcheck(fs, extended):
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(fs + extended)
    x, y = signals(rng, length_for_stft_frames(33, fs), fs, rows=2)
    xt, yt = cuda(x), cuda(y)
    assert torch.autograd.gradcheck(lambda a, b: stoi(a, b, fs, extended=extended), (xt, yt), fast_mode=True,
                                    nondet_tol=0)


@pytest.mark.parametrize('extended', [False, True])
@pytest.mark.parametrize('M', [29, 30, 31, 93, 94, 95])
def test_parity_frame_counts(M, extended):
    rng = np.random.default_rng(M + 100 * extended)
    x, y = signals(rng, length_for_stft_frames(M, 10000), 10000, rows=2)
    K, Ms = check_parity(cuda(x), cuda(y), 10000, extended)
    assert Ms == [M, M]


@pytest.mark.parametrize('extended', [False, True])
@pytest.mark.parametrize('fs', [8000, 16000, 48000])
def test_parity_gaps_and_clipping(fs, extended):
    rng = np.random.default_rng(fs + 3 * extended)
    n = length_for_stft_frames(200, fs)
    x, y = signals(rng, n, fs, rows=3, gaps=((0.2, 0.3), (0.55, 0.58)))
    K, M = check_parity(cuda(x), cuda(y), fs, extended)
    assert all(k < 201 for k in K) and all(m >= 30 for m in M)    # frames were dropped inside the row
    if not extended:
        assert clip_states(x[0], y[0], fs) == (True, True)


@pytest.mark.parametrize('extended', [False, True])
def test_parity_long_row(extended):
    rng = np.random.default_rng(5)
    x, y = signals(rng, 1 << 20, 10000, gaps=((0.4, 0.41),))
    check_parity(cuda(x), cuda(y), 10000, extended)


@pytest.mark.parametrize('extended', [False, True])
def test_parity_broadcast_reference(extended):
    rng = np.random.default_rng(6)
    x, y = signals(rng, length_for_stft_frames(70, 16000), 16000, rows=4)
    check_parity(cuda(x[:1]), cuda(y), 16000, extended)


@pytest.mark.parametrize('extended', [False, True])
def test_parity_float32(extended):
    rng = np.random.default_rng(7)
    x, y = signals(rng, length_for_stft_frames(70, 16000), 16000, rows=2)
    xt, yt = cuda(x, torch.float32), cuda(y, torch.float32)
    # the device reads the float32 values exactly; only the returned gradient is rounded to float32
    check_parity(xt, yt, 16000, extended, tol=TOL + 2.0 ** -24)


@pytest.mark.parametrize('extended', [False, True])
def test_group_split(monkeypatch, extended):
    from pb_bss_b200.evaluation import module_stoi as MS
    rng = np.random.default_rng(8)
    x, y = signals(rng, length_for_stft_frames(100, 16000), 16000, rows=3)
    w = torch.tensor([0.3, -1.0, 2.0], dtype=torch.float64, device='cuda')
    _, gx, gy = device_grads(cuda(x), cuda(y), 16000, extended, w)
    per_row = MS._lib.load().pbb_stoi_backward_workspace_bytes(1, x.shape[1], 5, 8, int(extended))
    monkeypatch.setattr(MS, 'WORKSPACE_BYTES', per_row)     # one row per group
    _, sx, sy = device_grads(cuda(x), cuda(y), 16000, extended, w)
    assert torch.equal(gx, sx) and torch.equal(gy, sy)
    check_parity(cuda(x), cuda(y), 16000, extended)


@pytest.mark.parametrize('extended', [False, True])
def test_invariants(extended):
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(9)
    x, y = signals(rng, length_for_stft_frames(60, 16000), 16000, rows=2)
    plain = stoi(cuda(x, grad=False), cuda(y, grad=False), 16000, extended=extended)
    xt, yt = cuda(x), cuda(y)
    v = stoi(xt, yt, 16000, extended=extended)
    assert v.grad_fn is not None and torch.equal(v.detach(), plain)
    w = torch.tensor([1.0, -0.5], dtype=torch.float64, device='cuda')
    g1 = torch.autograd.grad((v * w).sum(), (xt, yt), retain_graph=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        g2 = torch.autograd.grad((v * w).sum(), (xt, yt), retain_graph=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    gx, = torch.autograd.grad(v.sum(), xt, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()
    # only the estimate requires grad: the reference's chain is skipped
    ye = cuda(y)
    ge, = torch.autograd.grad((stoi(cuda(x, grad=False), ye, 16000, extended=extended) * w).sum(), ye)
    assert torch.equal(ge, g1[1])
    # float32 in, float32 out
    x32 = cuda(x, torch.float32)
    g32, = torch.autograd.grad(stoi(x32, cuda(y, torch.float32, False), 16000, extended=extended).sum(), x32)
    assert g32.dtype == torch.float32
    # NumPy in: NumPy out, no graph
    assert isinstance(stoi(x, y, 16000, extended=extended), np.ndarray)


@pytest.mark.parametrize('extended', [False, True])
def test_short_and_non_finite_rows(extended):
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(10)
    x, y = signals(rng, length_for_stft_frames(60, 10000), 10000, rows=4)
    x[1, :-128 * 25] = 0.0          # 1e-5 path: fewer than 30 STFT frames are kept
    x[2, 1000] = np.inf             # a non-finite reference: every frame dropped, 1e-5
    y[3, 3000] = np.nan             # a non-finite estimate sample: NaN in row 3 only
    xt, yt = cuda(x), cuda(y)
    with pytest.warns(RuntimeWarning):
        v = stoi(xt, yt, 10000, extended=extended)
    assert v[1].item() == 1e-5 and v[2].item() == 1e-5 and np.isnan(v[3].item())
    gx, gy = torch.autograd.grad(v.sum(), (xt, yt))
    for g in (gx, gy):
        assert torch.equal(g[1:3], torch.zeros_like(g[1:3]))
        assert torch.isnan(g[3]).any()
    x0, y0 = cuda(x[:1]), cuda(y[:1])
    ref_x, ref_y = torch.autograd.grad(stoi(x0, y0, 10000, extended=extended).sum(), (x0, y0))
    assert torch.equal(gx[:1], ref_x) and torch.equal(gy[:1], ref_y)


@pytest.mark.parametrize('extended', [False, True])
def test_digital_silence_in_the_estimate(extended):
    rng = np.random.default_rng(11)
    x, y = signals(rng, length_for_stft_frames(120, 10000), 10000, rows=2)
    y[0, 4000:9000] = 0.0
    y[1] = 0.0
    K, M = check_parity(cuda(x), cuda(y), 10000, extended)


@pytest.mark.parametrize('extended', [False, True])
def test_mask_istft_stoi_chain(extended):
    from oracle import autograd_oracle as AO
    from pb_bss_b200.transform import istft, stft
    from pb_bss_b200.evaluation import stoi
    rng = np.random.default_rng(12)
    fs, n = 16000, 16000
    x, noise = signals(rng, n, fs)[0][0], rng.standard_normal(n)
    mix = torch.tensor(x + 0.5 * noise, device='cuda')
    ref = torch.tensor(x, device='cuda')
    Y = stft(mix, size=512, shift=128)
    logits = torch.tensor(rng.standard_normal(tuple(Y.shape)), device='cuda', requires_grad=True)
    est = istft(torch.sigmoid(logits) * Y, size=512, shift=128)[..., :n]
    loss = -stoi(ref, est, fs, extended=extended)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    lr = logits.detach().clone().requires_grad_()
    est_r = AO.istft(torch.sigmoid(lr) * AO.stft(mix, size=512, shift=128), size=512, shift=128)[..., :n]
    v, _, _ = A.stoi(ref[None], est_r[None], fs, extended)
    (-v.sum()).backward()
    torch.testing.assert_close(loss.detach(), -v[0].detach(), rtol=0, atol=1e-12)
    assert_rows_close(logits.grad.reshape(1, -1), lr.grad.reshape(1, -1))
