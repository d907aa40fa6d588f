"""Launch accounting: pbb_launch_count counts kernel launches and the profile keeps one record per launch.

For entry points of every csrc/api_*.cu file, and for every place that once launched several kernels under one
profile record or launched one outside any, three counts must agree: the kernels of namespace pbb that
torch.profiler (CUDA activity) sees, the pbb_launch_count() delta, and the records pbb_profile_dump prints."""
import os
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _records(lib):
    """Names of the launches recorded since the last pbb_profile_reset (pbb_profile_dump prints them on fd 2)."""
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
        return [line.split()[1] for line in tmp.read().splitlines() if line.startswith('[pbb]')]


def _rng(seed=0):
    return np.random.default_rng(seed)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _hpd(n, D, seed):
    """n Hermitian positive definite D x D matrices."""
    r = _rng(seed)
    a = r.standard_normal((n, D, 2 * D)) + 1j * r.standard_normal((n, D, 2 * D))
    return a @ a.conj().transpose(0, 2, 1) / (2 * D) + np.eye(D)


def _gaussian_fit():
    from pb_bss_b200.distribution.von_mises_fisher import vmf_fit_fkt
    r = _rng(1)
    F, T, E, K = 6, 40, 3, 2
    emb, w = _cuda(r.standard_normal((F, T, E))), _cuda(r.random((F, K, T)))
    return lambda: vmf_fit_fkt(emb, w, 1e-10, 500.)


def _full_fit():
    from pb_bss_b200.distribution.gaussian import full_fit_bkn
    r = _rng(2)
    x, w = _cuda(r.standard_normal((2, 300, 4))), _cuda(r.random((2, 3, 300)))
    return lambda: full_fit_bkn(x, w)


def _vmf_resultant():
    from pb_bss_b200.distribution.von_mises_fisher import vmf_fit_bkn
    r = _rng(3)
    x, w = _cuda(r.standard_normal((2, 300, 4))), _cuda(r.random((2, 3, 300)))
    return lambda: vmf_fit_bkn(x, w, 1e-10, 500.)


def _souden(ref_channel):
    def make():
        from pb_bss_b200.extraction import beamformer as B
        t, n = _cuda(_hpd(9, 4, 4)), _cuda(_hpd(9, 4, 5))
        return lambda: B.get_mvdr_vector_souden(t, n, ref_channel=ref_channel)
    return make


def _tied_weight(flags):
    """The frequency-tied weight of the coupled EM loop: flags bit 0 ties the frames too, bit 1 the saliency form."""
    def make():
        from pb_bss_b200 import _lib
        from pb_bss_b200.distribution.mixture_model_utils import tied_weight
        F, K, T = 7, 3, 50
        aff = _cuda(_rng(6).random((F, K, T)))
        mode = _lib.WEIGHT_TIED if flags & 1 else _lib.WEIGHT_TIED_TIME
        return lambda: tied_weight(aff, None, mode, bool(flags & 2))
    return make


def _axis_sum_chunks():
    from pb_bss_b200 import _lib
    from pb_bss_b200._nd import axis_sum
    outs, n = 2, 1 << 16
    # more than one chunk per output: a partial per chunk and red_finish_kernel
    assert _lib.load().pbb_reduce_workspace_bytes(outs, n) > outs * 8
    x = _cuda(_rng(7).random((outs, n)))
    return lambda: axis_sum(x, (1,), False)


def _dhtv(metric):
    def make():
        from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
        al = DHTVPermutationAlignment(stft_size=128, segment_start=20, segment_width=20, segment_shift=5,
                                      main_iterations=5, sub_iterations=2, similarity_metric=metric)
        mask = _cuda(_rng(8).random((2, 65, 60)))
        return lambda: al.calculate_mapping(mask)
    return make


def _cacgmm_log_likelihood():
    from pb_bss_b200.distribution import CACGMMTrainer
    r = _rng(9)
    y = r.standard_normal((5, 80, 3)) + 1j * r.standard_normal((5, 80, 3))
    model = CACGMMTrainer().fit(y, num_classes=2, iterations=2)
    yd = _cuda(y)
    return lambda: model.log_likelihood(yd)


def _quantile_mask(T):
    def make():
        from pb_bss_b200.extraction.mask_module import quantile_mask
        x = _rng(10).standard_normal((2, T, 5))
        return lambda: quantile_mask(x)
    return make


def _lorenz_mask():
    from pb_bss_b200.extraction.mask_module import lorenz_mask
    x = _rng(11).standard_normal((2, 100, 65))
    return lambda: lorenz_mask(x)


def _kmeans():
    from pb_bss_b200.distribution.gmm import _kmeans_fit
    x = _rng(12).standard_normal((500, 3))
    return lambda: _kmeans_fit(x, 3)


def _stft():
    from pb_bss_b200.transform.fourier import stft
    x = _rng(13).standard_normal((2, 4000))
    return lambda: stft(x, size=256, shift=64)


def _wpe():
    from pb_bss_b200.wpe import wpe
    r = _rng(14)
    Y = r.standard_normal((4, 2, 60)) + 1j * r.standard_normal((4, 2, 60))
    return lambda: wpe(Y, taps=3, delay=1, iterations=2)


def _si_sdr():
    from pb_bss_b200.evaluation.module_si_sdr import si_sdr
    r = _rng(15)
    ref = r.standard_normal((2, 3000))
    est = ref + 0.3 * r.standard_normal((2, 3000))
    return lambda: si_sdr(ref, est)


def _bss_eval():
    from pb_bss_b200.evaluation.module_mir_eval import mir_eval_sources
    r = _rng(16)
    ref = r.standard_normal((2, 4000))
    est = ref + 0.3 * r.standard_normal((2, 4000))
    return lambda: mir_eval_sources(ref, est)


def _stoi():
    from pb_bss_b200.evaluation.module_stoi import stoi
    r = _rng(17)
    ref = r.standard_normal(20000)
    est = ref + 0.3 * r.standard_normal(20000)
    return lambda: stoi(ref, est, 10000)


def _srmr():
    from pb_bss_b200.evaluation.module_srmr import srmr
    x = _rng(18).standard_normal(16000)
    return lambda: srmr(x, 16000)


# case -> (input maker returning the call, names the records must include)
CASES = {
    'gaussian_fit': (_gaussian_fit, ['gaussian_fit_partial_kernel', 'gaussian_fit_mean_kernel',
                                     'gaussian_fit_cov_kernel']),
    'gaussian_full_fit': (_full_fit, ['gaussian_full_partial_kernel', 'gaussian_full_reduce_kernel']),
    'vmf_resultant': (_vmf_resultant, ['gaussian_full_partial_kernel', 'gaussian_full_reduce_kernel']),
    'souden_ref_channel': (_souden(1), ['souden_kernel', 'colsum_kernel']),
    'souden_chosen_channel': (_souden(None), ['souden_kernel', 'colsum_kernel']),
    'tied_weight': (_tied_weight(0), ['reduce_kernel']),
    'tied_weight_over_time': (_tied_weight(1), ['reduce_kernel<warp>', 'red_finish_kernel']),
    'tied_weight_unit_norm': (_tied_weight(2), ['reduce_kernel', 'scale_nd_kernel<divide>']),
    'tied_weight_over_time_unit_norm': (_tied_weight(3), ['reduce_kernel<warp>', 'red_finish_kernel', 'reduce_kernel',
                                                          'scale_nd_kernel<divide>']),
    'axis_sum_chunks': (_axis_sum_chunks, ['red_finish_kernel']),
    'dhtv_cos': (_dhtv('cos'), ['dhtv_normalize_kernel', 'dhtv_init_mapping_kernel']),
    'dhtv_multiply': (_dhtv('multiply'), ['dhtv_init_mapping_kernel']),
    'cacgmm_log_likelihood': (_cacgmm_log_likelihood, ['sum_rows_kernel']),
    'quantile_mask': (_quantile_mask(100), ['row_select_short_kernel']),
    'quantile_mask_long_rows': (_quantile_mask(5000), ['row_state_init_kernel', 'row_apply_kernel']),
    'lorenz_mask': (_lorenz_mask, ['row_state_init_kernel', 'row_apply_kernel']),
    'kmeans': (_kmeans, ['kmeans_init_kernel', 'kmeans_lloyd_kernel']),
    'stft': (_stft, ['stft_kernel']),
    'wpe': (_wpe, []),
    'si_sdr': (_si_sdr, []),
    'bss_eval': (_bss_eval, []),
    'stoi': (_stoi, []),
    'srmr': (_srmr, []),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_every_launch_is_counted_and_recorded_once(case):
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from pb_bss_b200 import _lib
    make, names = CASES[case]
    lib = _lib.load()
    call = make()
    call()                                     # loads the modules and fills the host-side caches
    torch.cuda.synchronize()
    lib.pbb_profile_enable(1)
    lib.pbb_profile_reset()
    try:
        before = lib.pbb_launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = lib.pbb_launch_count() - before
        records = _records(lib)
    finally:
        lib.pbb_profile_enable(0)
        lib.pbb_profile_reset()
    traced = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and 'pbb::' in e.name]
    assert counted > 0, case
    assert len(traced) == counted == len(records), (case, counted, records, traced)
    assert set(names) <= set(records), (case, records)
