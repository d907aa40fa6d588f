"""pb_bss_b200.transform.gammatone on the device against the unmodified reference (tests/golden/gammatone.npz) and
the NumPy restatement (oracle/gammatone_oracle.py).  Every output must be within 1e-11 of the max |y| of its
(filter, row) in the reference.  The chunked scan (csrc/gammatone.cuh) is checked at the chunk edges of every chunk
length the host chooses, across several carry groups, on 2^22 samples, on more than 65 535 sequences and with
non-finite input."""
import os
import sys
import tempfile

import numpy as np
import pytest

from oracle import gammatone_oracle as GO
from oracle.make_golden_gammatone import CASES

pytestmark = pytest.mark.gpu

REL = 1e-11
CHUNK_LENGTHS = [128, 256, 512, 1024]   # PBB_GAMMATONE_CHUNK_MIN .. PBB_GAMMATONE_CHUNK_MAX


def _assert_close(out, ref, rel=REL):
    """|out - ref| <= rel * max|ref| of each (filter, row), for lists of n arrays of one shape."""
    out, ref = np.stack([np.asarray(v) for v in out]), np.stack(ref)
    assert out.shape == ref.shape and out.dtype == np.float64
    r = ref.reshape(ref.shape[0], -1, ref.shape[-1])
    o = out.reshape(r.shape)
    scale = np.abs(r).max(axis=-1, keepdims=True)
    assert (np.abs(o - r) <= rel * scale).all(), np.max(np.abs(o - r) / np.maximum(scale, 1e-300))


def _launches(lib):
    """Names of the launches recorded since the last pbb_profile_reset (pbb_profile_dump prints them on fd 2)."""
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


@pytest.mark.parametrize('case', sorted(CASES))
def test_fixture_cases_match_the_reference(golden, case):
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    g = golden('gammatone')
    sr, n, lo, hi = g[case + '_params']
    x = g[case + '_x']
    y = gammatone_filterbank(x, int(sr), int(n), lo, hi)
    assert isinstance(y, list) and len(y) == int(n)
    assert all(isinstance(v, np.ndarray) and v.shape == x.shape and v.dtype == np.float64 for v in y)
    _assert_close(y, list(g[case + '_y']))


def _rows_for(L, n, N, limit=40000):
    """The fewest rows for which the host chooses chunk length L at (rows, n, N), or None."""
    from pb_bss_b200.transform.gammatone import chunk_length
    for rows in range(1, limit):
        if chunk_length(rows, n, N) == L:
            return rows
    return None


def _edges(L):
    return [1, 2, L - 1, L, L + 1, 2 * L - 1, 2 * L, 2 * L + 1, 5 * L + 17, 37 * L + 5, 70 * L + 3]


@pytest.mark.parametrize('L', CHUNK_LENGTHS)
def test_chunk_edges_of_every_chunk_length(L):
    """N at the edges of one, two and several chunks, and across one and two carry groups (32 chunks each).  An N for
    which the host never chooses L (a larger chunk would give as many chunks) is skipped; the rest must reach L."""
    import torch
    from pb_bss_b200.transform.gammatone import chunk_length, gammatone_filterbank
    n, reached = 23, 0
    for N in _edges(L):
        rows = _rows_for(L, n, N, limit=40000 // max(1, N // 4096) + 2)
        if rows is None:
            continue
        reached += 1
        x = np.random.default_rng(N).standard_normal((rows, N))
        assert chunk_length(rows, n, N) == L
        y = gammatone_filterbank(torch.from_numpy(x).cuda(), 16000, n)
        _assert_close([v.cpu().numpy() for v in y], GO.gammatone_filterbank(x, 16000, n))
        del y
        torch.cuda.empty_cache()
    assert reached >= 6, reached


def test_empty_and_tiny_signals():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    for shape in ((0,), (3, 0), (0, 5), (2, 0, 7)):
        y = gammatone_filterbank(np.zeros(shape), 16000, 4)
        assert len(y) == 4 and all(v.shape == shape and v.dtype == np.float64 for v in y)
        t = gammatone_filterbank(torch.zeros(shape, device='cuda'), 16000, 4)
        assert all(v.is_cuda and tuple(v.shape) == shape for v in t)
    for N in (1, 2, 3):
        x = np.random.default_rng(N).standard_normal((2, N))
        _assert_close(gammatone_filterbank(x, 16000, 5), GO.gammatone_filterbank(x, 16000, 5))


def test_leading_dims_strides_and_dtypes():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 3, 4, 1500))
    _assert_close(gammatone_filterbank(x, 44100, 6), GO.gammatone_filterbank(x, 44100, 6))
    xt = rng.standard_normal((1500, 3))                        # filter along a non-contiguous last axis
    _assert_close(gammatone_filterbank(xt.T, 16000, 6), GO.gammatone_filterbank(xt.T, 16000, 6))
    tt = torch.from_numpy(xt).cuda().T
    assert not tt.is_contiguous()
    _assert_close([v.cpu().numpy() for v in gammatone_filterbank(tt, 16000, 6)], GO.gammatone_filterbank(xt.T, 16000, 6))
    x32 = rng.standard_normal((3, 2000)).astype(np.float32)
    _assert_close(gammatone_filterbank(x32, 8000, 4), GO.gammatone_filterbank(x32, 8000, 4))
    t32 = gammatone_filterbank(torch.from_numpy(x32).cuda(), 8000, 4)
    assert all(v.dtype == torch.float64 for v in t32)
    _assert_close([v.cpu().numpy() for v in t32], GO.gammatone_filterbank(x32, 8000, 4))
    xi = rng.integers(-2000, 2000, size=(2, 900)).astype(np.int32)
    _assert_close(gammatone_filterbank(xi, 16000, 3), GO.gammatone_filterbank(xi, 16000, 3))
    _assert_close([v.cpu().numpy() for v in gammatone_filterbank(torch.from_numpy(xi).cuda(), 16000, 3)],
                  GO.gammatone_filterbank(xi, 16000, 3))


def test_cuda_in_gives_cuda_out_on_the_current_stream():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    x = torch.from_numpy(np.random.default_rng(4).standard_normal((2, 5000))).cuda()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        y = gammatone_filterbank(x, 16000, 23)
    stream.synchronize()
    assert isinstance(y, list) and len(y) == 23
    assert all(v.is_cuda and v.device == x.device and v.dtype == torch.float64 and v.shape == x.shape for v in y)
    _assert_close([v.cpu().numpy() for v in y], GO.gammatone_filterbank(x.cpu().numpy(), 16000, 23))


def test_more_than_65535_sequences():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    x = np.random.default_rng(5).standard_normal((3000, 300))
    y = gammatone_filterbank(torch.from_numpy(x).cuda(), 16000, 23)
    _assert_close([v.cpu().numpy() for v in y], GO.gammatone_filterbank(x, 16000, 23))


def test_a_signal_of_2_to_the_22_samples():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    x = np.random.default_rng(6).standard_normal(1 << 22)
    for sr in (16000, 48000):
        y = gammatone_filterbank(torch.from_numpy(x).cuda(), sr, 23)
        _assert_close([v.cpu().numpy() for v in y], GO.gammatone_filterbank(x, sr, 23))
        del y


def test_non_finite_input_matches_lfilter():
    """NaN mid-chunk in one row, inf at a chunk edge in another, -inf in the first sample of a third: the non-finite
    outputs sit where lfilter's do, and the finite ones before them are within tolerance."""
    from pb_bss_b200.transform.gammatone import chunk_length, gammatone_filterbank
    rows, n, N = 4, 23, 9000
    L = chunk_length(rows, n, N)
    x = np.random.default_rng(7).standard_normal((rows, N))
    x[0, 3 * L + 57] = np.nan
    x[1, 20 * L] = np.inf
    x[2, 0] = -np.inf
    for sr in (16000, 48000):
        ref = np.stack(GO.gammatone_filterbank(x, sr, n))
        out = np.stack(gammatone_filterbank(x, sr, n))
        np.testing.assert_array_equal(np.isfinite(out), np.isfinite(ref))
        fin = np.isfinite(ref)
        scale = np.where(fin, np.abs(ref), 0).max(axis=-1, keepdims=True)
        scale = np.where(scale > 0, scale, 1.0)
        err = np.abs(np.where(fin, out, 0) - np.where(fin, ref, 0))
        assert (err <= REL * scale).all(), np.max(err / scale)
        assert fin[:, 3].all() and not fin[:, 2].any()


def test_bitwise_reproducible():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    x = torch.from_numpy(np.random.default_rng(8).standard_normal((8, 40000))).cuda()
    a = torch.stack(gammatone_filterbank(x, 16000, 23))
    b = torch.stack(gammatone_filterbank(x, 16000, 23))
    assert torch.equal(a, b)


def test_complex_input_raises_type_error():
    import torch
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    x = np.ones(100, np.complex128)
    with pytest.raises(TypeError):
        gammatone_filterbank(x)
    with pytest.raises(TypeError):
        gammatone_filterbank(torch.from_numpy(x).cuda())


def test_only_the_gammatone_kernels_run():
    import torch
    from pb_bss_b200 import _lib
    from pb_bss_b200.transform.gammatone import gammatone_filterbank
    lib = _lib.load()
    x = torch.from_numpy(np.random.default_rng(9).standard_normal((2, 20000))).cuda()
    gammatone_filterbank(x, 16000, 23)                      # device tables cached outside the recorded window
    lib.pbb_profile_enable(1)
    try:
        lib.pbb_profile_reset()
        gammatone_filterbank(x, 16000, 23)
        assert _launches(lib) == ['gammatone_chunk_state_kernel', 'gammatone_carry_kernel', 'gammatone_output_kernel']
        gammatone_filterbank(x[:, :100], 16000, 23)          # one chunk: no scan
        assert _launches(lib) == ['gammatone_output_kernel']
    finally:
        lib.pbb_profile_enable(0)
