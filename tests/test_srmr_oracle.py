"""CPU checks of SRMR: the NumPy restatement (oracle/srmr_oracle.py) against the unmodified reference
(tests/golden/srmr.npz), the closed-form Hilbert kernel the device convolves with, the host-side modulation filters and
the frame counts of the segment_axis restatement."""
import math

import numpy as np
import pytest

from oracle import srmr_oracle as SO
from oracle.make_golden_srmr import cases as _fixture_cases, signal, vad_output
from pb_bss_b200.evaluation import module_srmr as M

CASES = sorted(_fixture_cases(np.random.RandomState(0)))


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_the_reference(golden, case):
    """1e-11 relative: the gammatone cascade carries 1 / gain (up to 1e10) in its states, and the restatement's
    arithmetic rounds differently from the reference's there."""
    g = golden('srmr')
    sr, n, lo, _ = g[case + '_params']
    x = signal(g, case)
    x = x.astype(np.float64) if x.dtype == np.int16 else x
    np.testing.assert_allclose(SO.srmr(x, int(sr), int(n), lo), g[case + '_value'], rtol=1e-11, atol=0)
    if case + '_vad_keep' in g:
        kept, ref = SO.vad(x, sr), vad_output(g, case)
        assert kept.dtype == ref.dtype and len(ref) < x.shape[-1]
        np.testing.assert_array_equal(kept, ref)


def test_fixture_errors(golden):
    g = golden('srmr')
    assert str(g['error_dim30']) == 'AssertionError'
    assert str(g['error_ndim0']) == 'NotImplementedError'
    with pytest.raises(NotImplementedError):
        SO.srmr(np.float64(1.0))


@pytest.mark.parametrize('N', list(range(1, 65)) + [1000, 1001, 65536, 65537, 160001])
def test_closed_form_kernel_is_the_inverse_dft_of_scipys_multiplier(N):
    g = SO.hilbert_kernel(N)
    ref = np.fft.ifft(SO.hilbert_multiplier(N)).imag
    assert np.abs(g - ref).max() <= 1e-14 * max(1.0, np.abs(ref).max())


def test_kernel_convolution_gives_scipys_hilbert():
    import scipy.signal
    for N in (1, 2, 7, 64, 257, 4097):
        x = np.random.RandomState(N).randn(N)
        M_ = 1 << max(1, int(np.ceil(np.log2(2 * N - 1))))
        k = np.zeros(M_)
        g = SO.hilbert_kernel(N)
        k[:N] = g
        if N > 1:
            k[M_ - N + 1:] = g[1:]
        im = np.fft.irfft(np.fft.rfft(x, M_) * np.fft.rfft(k), M_)[:N]
        a = scipy.signal.hilbert(x)
        assert np.abs(im - a.imag).max() <= 1e-13 * np.abs(a).max()


@pytest.mark.parametrize('sr', [8000, 16000, 44100, 48000])
def test_modulation_coefficients_follow_the_reference_formula(sr):
    c = M.modulation_coefficients(sr)
    ref = SO.modulation_coefficients(sr)
    np.testing.assert_array_equal(c[:, 0], ref[:, 0, 0])
    np.testing.assert_array_equal(-c[:, 0], ref[:, 0, 2])
    np.testing.assert_array_equal(c[:, 1:], ref[:, 1, 1:])
    np.testing.assert_array_equal(M.cutoffs(sr), SO.cutoffs(sr))
    for k, f in enumerate(SO.MOD_FREQS):
        W0 = math.tan(2 * math.pi * f / (2 * sr))
        assert c[k, 0] == (W0 / 2) / (1 + W0 / 2 + W0 ** 2)


@pytest.mark.parametrize('sr', [8000, 16000, 44100, 48000])
def test_modulation_transition_is_the_filter_run_over_one_hop(sr):
    """The 2 x 2 chunk transition pbb_srmr_means carries the states with: the zero-input filter over S samples."""
    import scipy.signal
    W, S = M.frame_lengths(sr)
    c = M.modulation_coefficients(sr)
    from pb_bss_b200.transform.gammatone import chunk_transition
    A = chunk_transition(M._modulation_step, c, 2, S)
    for k in range(8):
        b, a = [c[k, 0], 0, -c[k, 0]], [1, c[k, 1], c[k, 2]]
        x = np.random.RandomState(k).randn(S)
        _, z1 = scipy.signal.lfilter(b, a, x, zi=np.zeros(2))
        _, z2 = scipy.signal.lfilter(b, a, np.zeros(S), zi=z1)
        np.testing.assert_allclose(A[k] @ z1, z2, rtol=0, atol=1e-11 * np.abs(z1).max())


@pytest.mark.parametrize('sr', [8000, 16000, 44100, 48000])
def test_frame_lengths_truncate(sr):
    W, S = SO.frame_lengths(sr)
    assert (W, S) == M.frame_lengths(sr) and W == 4 * S and S == int(sr / 1000) * 64
    if sr == 44100:
        assert (W, S) == (11264, 2816)


@pytest.mark.parametrize('sr', [8000, 16000])
def test_segment_axis_frame_counts(sr):
    W, S = SO.frame_lengths(sr)
    for N, F in ((1, 1), (W - 1, 1), (W, 1), (W + 1, 2), (W + S - 1, 2), (W + S, 2), (W + S + 1, 3), (10 * W, 37)):
        frames = SO.segment_axis(np.arange(1, N + 1, dtype=float), W, S)
        assert frames.shape == (F, W) == (SO.frame_count(N, sr), W)
        assert frames[0, 0] == 1 and frames.sum() >= N * (N + 1) / 2 and (frames[:, -1] == 0).any() == (
            (N - W) % S != 0 or N < W)
