"""Frame-online WPE on the device (pb_bss_b200.wpe.online_wpe_step, get_power_online, online_wpe) against the NumPy
oracle (oracle/wpe_online_oracle.py): shapes, dtypes, layouts, long streams, chunking, the NaN bin and the errors."""
import numpy as np
import pytest
import torch

from oracle import wpe_online_oracle as O

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps

# Tolerance of online_wpe against the oracle, per bin: max(1e-10, C n eps max_t kappa(R_t)) max|Y_f|.  Both compute
# the same recursion in fp64 and differ only in the order of their sums.  The recursion maintains Q_t = R_t^-1, so a
# relative rounding of order n eps in the data of a step moves Q_t, G_t and hence pred by at most about
# kappa(R_t) n eps relative (the forward error of inverting R_t).  C = 8 covers: two implementations rounding
# independently (2), a complex multiply-add rounding its real and imaginary parts in up to two operations each (2), and
# the two sums of a step that enter pred through G, one for den and one for the rank-1 update (2).
C = 8


def _y(shape, seed=0, dtype=np.complex128):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(dtype)


def _pd(F, n, seed):
    A = _y((F, n, n), seed)
    return A @ A.conj().transpose(0, 2, 1) / n + np.eye(n)


def _wpe():
    from pb_bss_b200 import wpe
    return wpe


def _terms(buf, power, Q, G, alpha, taps, delay):
    """Per bin, the largest sum of |terms| behind each output of the step (pred = y - G^H w, Q' = (Q - k v) / alpha,
    G' = G + k pred^H): a fixed-order sum errs by a few n eps of that, not of its (possibly cancelled) result."""
    buf, Q, G = (np.asarray(a, dtype=np.complex128) for a in (buf, Q, G))
    w = np.abs(O.window(buf, taps, delay))
    pred, _, _ = O.online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    u = np.einsum('fij,fj->fi', Q, O.window(buf, taps, delay))
    den = alpha * np.asarray(power) + np.einsum('fi,fi->f', O.window(buf, taps, delay).conj(), u)
    k = np.abs(u / den[:, None])
    v = np.einsum('fj,fjm->fm', w, np.abs(Q))
    t_pred = np.abs(buf[-1]) + np.einsum('fid,fi->fd', np.abs(G), w)
    t_q = (np.abs(Q) + k[:, :, None] * v[:, None, :]) / alpha
    t_g = np.abs(G) + k[:, :, None] * np.abs(pred)[:, None, :]
    return [t.reshape(t.shape[0], -1).max(axis=1) for t in (t_pred, t_q, t_g)]


def _close_step(got, want, rtol, terms):
    for g, w, scale in zip(got, want, terms):
        g = np.asarray(g.cpu() if isinstance(g, torch.Tensor) else g).astype(np.complex128)
        err = np.abs(g - w).reshape(w.shape[0], -1).max(axis=1)
        assert (err <= rtol * scale).all(), (err / scale).max()


def _step_case(F, D, taps, delay, alpha=0.99, seed=0):
    n = taps * D
    buf = _y((taps + delay + 1, F, D), seed)
    Q = _pd(F, n, seed + 1)
    G = _y((F, n, D), seed + 2)
    power = np.random.default_rng(seed + 3).random(F) + 0.5
    return buf, power, Q, G, alpha


@pytest.mark.parametrize('D', [1, 2, 4, 8])
@pytest.mark.parametrize('taps', [1, 3, 10, 12])
@pytest.mark.parametrize('delay', [0, 1, 2, 5])
def test_step_matches_oracle(D, taps, delay):
    """One step from a well-conditioned Q (den >= alpha lambda > 0): 16 n eps of the terms behind each output."""
    buf, power, Q, G, alpha = _step_case(3, D, taps, delay, seed=D + taps + delay)
    got = _wpe().online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    want = O.online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    _close_step(got, want, 16 * taps * D * EPS, _terms(buf, power, Q, G, alpha, taps, delay))


@pytest.mark.parametrize('F,D,taps,delay', [(513, 8, 10, 2), (1, 8, 12, 2), (513, 8, 12, 0), (4, 30, 3, 5),
                                            (513, 30, 3, 2), (1, 1, 1, 0)])
def test_step_shapes(F, D, taps, delay):
    buf, power, Q, G, alpha = _step_case(F, D, taps, delay, seed=F)
    got = _wpe().online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    want = O.online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    _close_step(got, want, 16 * taps * D * EPS, _terms(buf, power, Q, G, alpha, taps, delay))


def test_step_dtypes_devices_and_views():
    wpe = _wpe()
    F, D, taps, delay = 7, 4, 3, 2
    buf, power, Q, G, alpha = _step_case(F, D, taps, delay)
    want = O.online_wpe_step(buf, power, Q, G, alpha, taps, delay)
    n = taps * D
    terms = _terms(buf, power, Q, G, alpha, taps, delay)
    # nara_wpe's start: real float64 identity and zeros
    p0, Q0, G0 = wpe.online_wpe_step(buf, power, np.broadcast_to(np.eye(n), (F, n, n)).copy(),
                                     np.zeros((F, n, D)), alpha, taps, delay)
    w0 = O.online_wpe_step(buf, power, np.eye(n) + np.zeros((F, n, n)), np.zeros((F, n, D)), alpha, taps, delay)
    assert Q0.dtype == np.complex128 and G0.dtype == np.complex128
    _close_step((p0, Q0, G0), w0, 16 * n * EPS,
                _terms(buf, power, np.eye(n) + np.zeros((F, n, n)), np.zeros((F, n, D)), alpha, taps, delay))
    # CUDA tensors in, CUDA tensors out
    dev = [torch.from_numpy(a).cuda() for a in (buf, power, Q, G)]
    got = wpe.online_wpe_step(dev[0], dev[1], dev[2], dev[3], alpha, taps, delay)
    assert all(isinstance(g, torch.Tensor) and g.is_cuda for g in got)
    _close_step(got, want, 16 * n * EPS, terms)
    # strided views: every other bin of a transposed buffer
    big = _y((taps + delay + 1, D, 2 * F), 9)
    view = torch.from_numpy(big).cuda().transpose(1, 2)[:, ::2]
    ref = big.transpose(0, 2, 1)[:, ::2].copy()
    got = wpe.online_wpe_step(view, dev[1], dev[2], dev[3], alpha, taps, delay)
    _close_step(got, O.online_wpe_step(ref, power, Q, G, alpha, taps, delay), 16 * n * EPS,
                _terms(ref, power, Q, G, alpha, taps, delay))
    # complex64 data: the prediction is rounded once to complex64
    got = wpe.online_wpe_step(buf.astype(np.complex64), power, Q, G, alpha, taps, delay)
    assert got[0].dtype == np.complex64 and got[1].dtype == np.complex128
    want64 = O.online_wpe_step(buf.astype(np.complex64).astype(np.complex128), power, Q, G, alpha, taps, delay)
    _close_step(got, want64, 4 * np.finfo(np.float32).eps, terms)


def test_get_power_online():
    wpe = _wpe()
    x = _y((513, 8, 13), 3)
    np.testing.assert_allclose(wpe.get_power_online(x), O.get_power_online(x), rtol=1e-14)
    np.testing.assert_array_equal(wpe.get_power_online(x), wpe.get_power(x, np.inf)[..., 0])


def _oracle_stream(Y, taps, delay, alpha):
    """Oracle Z and the per-bin tolerance max(1e-10, C n eps max_t kappa(R_t)) (relative to max|Y_f|)."""
    Z, state, kappa = O.online_wpe(Y, taps, delay, alpha, details=True)
    n = taps * Y.shape[-1]
    k = kappa.max(axis=0) if len(kappa) else np.ones(Y.shape[1])
    return Z, state, np.maximum(1e-10, C * n * EPS * k)


def _close_stream(got, want, Y, rtol):
    got, want = np.asarray(got).astype(np.complex128), np.asarray(want).astype(np.complex128)
    if not got.size:
        return
    err = np.abs(got - want).max(axis=(0, 2))
    scale = np.abs(Y).max(axis=(0, 2))
    assert (err <= rtol * scale).all(), (err / scale / rtol).max()


@pytest.mark.parametrize('alpha', [0.99, 0.9999, 1.0])
@pytest.mark.parametrize('T', [0, 1, 5, 500])
def test_online_wpe_matches_oracle(T, alpha):
    F, D, taps, delay = 5, 2, 3, 2
    Y = _y((T, F, D), T)
    Z, state = _wpe().online_wpe(Y, taps, delay, alpha)
    want, wstate, rtol = _oracle_stream(Y, taps, delay, alpha)
    assert Z.shape == Y.shape and Z.dtype == Y.dtype
    _close_stream(Z, want, Y, rtol)
    np.testing.assert_array_equal(state.history, wstate.history)
    assert state.inv_cov.shape == (F, taps * D, taps * D) and state.filter_taps.shape == (F, taps * D, D)


@pytest.mark.parametrize('alpha', [0.99, 0.9999, 1.0])
def test_online_wpe_long_stream(alpha):
    T, F, D, taps, delay = 20000, 2, 2, 3, 1
    Y = _y((T, F, D), 11)
    Z, _ = _wpe().online_wpe(Y, taps, delay, alpha)
    want, _, rtol = _oracle_stream(Y, taps, delay, alpha)
    _close_stream(Z, want, Y, rtol)


@pytest.mark.parametrize('F,D,taps,delay', [(513, 8, 10, 2), (3, 8, 12, 2), (3, 30, 3, 5), (4, 1, 12, 0)])
def test_online_wpe_shapes(F, D, taps, delay):
    T = 60
    Y = _y((T, F, D), F + D)
    Z, _ = _wpe().online_wpe(Y, taps, delay, 0.99)
    want, _, rtol = _oracle_stream(Y, taps, delay, 0.99)
    _close_stream(Z, want, Y, rtol)


def test_online_wpe_stft_layout_complex64_and_views():
    wpe = _wpe()
    D, T, F = 3, 80, 9
    X = _y((D, T, F), 4)
    Y = X.transpose(1, 2, 0)
    want, _, rtol = _oracle_stream(Y.copy(), 4, 1, 0.99)
    Zc, _ = wpe.online_wpe(torch.from_numpy(X).cuda().permute(1, 2, 0), 4, 1, 0.99)
    assert isinstance(Zc, torch.Tensor) and Zc.is_cuda
    _close_stream(Zc.cpu().numpy(), want, Y, rtol)
    Z64, st64 = wpe.online_wpe(Y.astype(np.complex64), 4, 1, 0.99)
    assert Z64.dtype == np.complex64 and st64.history.dtype == np.complex64
    want64, _, rtol64 = _oracle_stream(Y.astype(np.complex64).astype(np.complex128), 4, 1, 0.99)
    _close_stream(Z64, want64, Y, np.maximum(rtol64, 4 * np.finfo(np.float32).eps))
    # leading dims (T, 3, 3, D) are bins like (T, 9, D)
    Z2, _ = wpe.online_wpe(Y.reshape(T, 3, 3, D), 4, 1, 0.99)
    np.testing.assert_array_equal(Z2.reshape(T, F, D), wpe.online_wpe(Y, 4, 1, 0.99)[0])


@pytest.mark.parametrize('cuts', [[1], [2, 3, 4], [5], [250], list(range(1, 40)), [7, 100, 101, 399]])
def test_chunked_is_bitwise_one_call(cuts):
    wpe = _wpe()
    T, F, D, taps, delay = 400, 17, 4, 4, 2   # taps + delay = 6 history frames
    Y = torch.from_numpy(_y((T, F, D), 21)).cuda()
    Z, st = wpe.online_wpe(Y, taps, delay, 0.995)
    parts, state = [], None
    for a, b in zip([0] + cuts, cuts + [T]):
        z, state = wpe.online_wpe(Y[a:b], taps, delay, 0.995, state)
        parts.append(z)
    assert torch.equal(torch.cat(parts), Z)
    for a, b in zip(state, st):
        assert torch.equal(a, b)


def test_repeated_calls_are_bitwise_equal():
    wpe = _wpe()
    Y = _y((300, 33, 8), 5)
    a = wpe.online_wpe(Y, 10, 2, 0.99)
    b = wpe.online_wpe(Y, 10, 2, 0.99)
    np.testing.assert_array_equal(a[0], b[0])
    for x, y in zip(a[1], b[1]):
        np.testing.assert_array_equal(x, y)


def test_step_loop_agrees_with_online_wpe():
    """The device step driven frame by frame with get_power_online of each buffer."""
    wpe = _wpe()
    T, F, D, taps, delay, alpha = 120, 6, 2, 5, 2, 0.99
    Y = _y((T, F, D), 8)
    n, L = taps * D, taps + delay + 1
    Z, _ = wpe.online_wpe(Y, taps, delay, alpha)
    _, _, rtol = _oracle_stream(Y, taps, delay, alpha)
    stream = torch.from_numpy(np.concatenate([np.zeros((L - 1, F, D), complex), Y])).cuda()
    Q = torch.eye(n, dtype=torch.complex128, device='cuda').expand(F, n, n).contiguous()
    G = torch.zeros((F, n, D), dtype=torch.complex128, device='cuda')
    preds = []
    for t in range(T):
        buf = stream[t:t + L]
        p = wpe.get_power_online(buf.permute(1, 2, 0))
        pred, Q, G = wpe.online_wpe_step(buf, p, Q, G, alpha, taps, delay)
        preds.append(pred)
    _close_stream(torch.stack(preds).cpu().numpy(), Z, Y, rtol)


def test_all_zero_bin_is_nan_there_only():
    Y = _y((50, 4, 2), 3)
    Y[:, 2] = 0
    Z, state = _wpe().online_wpe(Y, 3, 1, 0.99)
    assert np.isnan(Z[1:, 2]).all() and np.isnan(state.inv_cov[2]).all()
    assert np.isfinite(np.delete(Z, 2, axis=1)).all()
    assert np.isfinite(np.delete(state.inv_cov, 2, axis=0)).all()


def test_errors():
    wpe = _wpe()
    Y = _y((10, 3, 2))
    for kw in ({'taps': 0}, {'delay': -1}, {'alpha': 0.0}, {'alpha': 1.5}, {'alpha': -0.5}):
        args = dict(taps=3, delay=1, alpha=0.99)
        args.update(kw)
        with pytest.raises(ValueError):
            wpe.online_wpe(Y, **args)
    with pytest.raises(NotImplementedError):
        wpe.online_wpe(_y((10, 3, 8)), 13, 1, 0.99)
    with pytest.raises(NotImplementedError):
        wpe.online_wpe(_y((10, 3, 31)), 1, 1, 0.99)
    with pytest.raises(NotImplementedError):
        wpe.online_wpe(_y((10, 3, 30)), 3, 100000, 0.99)
    with pytest.raises(TypeError):
        wpe.online_wpe(np.ones((10, 3, 2)), 3, 1, 0.99)
    _, st = wpe.online_wpe(Y, 3, 1, 0.99)
    for bad in (st._replace(history=st.history[1:]), st._replace(inv_cov=st.inv_cov[:, 1:]),
                st._replace(filter_taps=st.filter_taps[1:])):
        with pytest.raises(ValueError):
            wpe.online_wpe(Y, 3, 1, 0.99, bad)
    buf, power, Q, G, _ = _step_case(3, 2, 3, 1)
    with pytest.raises(ValueError):
        wpe.online_wpe_step(buf[1:], power, Q, G, 0.99, 3, 1)
    with pytest.raises(ValueError):
        wpe.online_wpe_step(buf, power, Q, G, 0.0, 3, 1)
    with pytest.raises(ValueError):
        wpe.online_wpe_step(buf, power, Q[:, 1:], G, 0.99, 3, 1)
    with pytest.raises(ValueError):
        wpe.online_wpe_step(buf, power[1:], Q, G, 0.99, 3, 1)


def test_dereverberates_synthetic_reverberant_data():
    """A white source through an exponentially decaying room response: once the recursion has settled, the late
    frames' error against the direct path is below that of the observation."""
    rng = np.random.default_rng(0)
    T, F, D, taps, delay, L = 3000, 16, 2, 10, 2, 12
    S = _y((T, F), 1)
    H = _y((L, F, D), 2) * np.exp(-np.arange(L) / 3.0)[:, None, None]
    H[0] = 1.0 + 0.1 * rng.standard_normal((F, D))
    Y = np.zeros((T, F, D), complex)
    for l in range(L):
        Y[l:] += S[:T - l, :, None] * H[l]
    direct = S[:, :, None] * H[0]
    Z, _ = _wpe().online_wpe(Y, taps, delay, 0.9999)
    late = slice(T // 2, None)
    err_z = np.mean(np.abs(Z[late] - direct[late]) ** 2)
    err_y = np.mean(np.abs(Y[late] - direct[late]) ** 2)
    assert err_z < err_y, (err_z, err_y)
