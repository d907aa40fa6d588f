"""ctypes binding of the C ABI declared in include/pbb.h.

The CUDA library is the product: if ``libpbb.so`` is missing or a symbol is
absent this module raises -- there is no CPU fallback anywhere in the package.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PBB_LIB selects an alternative build of the same ABI (kernel-variant experiments)
LIB_PATH = os.environ.get('PBB_LIB') or os.path.join(_HERE, 'libpbb.so')

PBB_C64, PBB_C128 = 0, 1
NORM_NONE, NORM_EIGENVALUE, NORM_TRACE = 0, 1, 2
CW_NORM_1F1, CW_NORM_LOW, CW_NORM_MEDIUM, CW_NORM_HIGH, CW_NORM_TRAN_VU = range(5)
WEIGHT_TIME, WEIGHT_CONST, WEIGHT_TIED_TIME, WEIGHT_TIED, WEIGHT_FRAME = 0, 1, 2, 3, 4


class CacgmmOptions(ctypes.Structure):
    """struct pbb_cacgmm_options (include/pbb.h)."""
    _fields_ = [
        ('iterations', ctypes.c_int),
        ('covariance_norm', ctypes.c_int),
        ('weight_mode', ctypes.c_int),
        ('hermitize', ctypes.c_int),
        ('affiliation_eps', ctypes.c_double),
        ('eigenvalue_floor', ctypes.c_double),
        ('frames_per_block', ctypes.c_int),
        ('reserved', ctypes.c_int),
    ]


PBB_F32, PBB_F64 = 2, 3
PBB_I16, PBB_I32, PBB_I64 = 4, 5, 6
MASK_MAX_DIMS = 8
MASK_IDEAL_BINARY, MASK_WIENER_LIKE, MASK_IDEAL_RATIO, MASK_IDEAL_AMPLITUDE, MASK_PHASE_SENSITIVE, \
    MASK_IDEAL_COMPLEX = range(6)
ROW_SELECT_SHORT_MAX = 4096  # PBB_ROW_SELECT_SHORT_MAX


class MaskLayout(ctypes.Structure):
    """struct pbb_mask_layout (include/pbb.h)."""
    _fields_ = [
        ('nd', ctypes.c_int),
        ('reserved', ctypes.c_int),
        ('shape', ctypes.c_longlong * MASK_MAX_DIMS),
        ('in_stride', ctypes.c_longlong * MASK_MAX_DIMS),
        ('out_stride', ctypes.c_longlong * MASK_MAX_DIMS),
    ]


ND_MAX_DIMS, ND_OPERANDS = 8, 4
WEIGHT_BCAST = 8


class NdLayout(ctypes.Structure):
    """struct pbb_nd_layout (include/pbb.h)."""
    _fields_ = [
        ('nd', ctypes.c_int),
        ('reserved', ctypes.c_int),
        ('shape', ctypes.c_longlong * ND_MAX_DIMS),
        ('stride', (ctypes.c_longlong * ND_MAX_DIMS) * ND_OPERANDS),
    ]


_vp, _i, _d, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_size_t
_ll, _lay = ctypes.c_longlong, ctypes.POINTER(MaskLayout)
_nd = ctypes.POINTER(NdLayout)

# name -> (restype, argtypes); mirrors include/pbb.h one to one
SIGNATURES = {
    'pbb_last_error': (ctypes.c_char_p, []),
    'pbb_version': (_i, []),
    'pbb_launch_count': (ctypes.c_longlong, []),
    'pbb_profile_enable': (None, [_i]),
    'pbb_profile_reset': (None, []),
    'pbb_profile_dump': (None, []),
    'pbb_profile_dominant': (_i, [ctypes.c_char_p, _i, ctypes.POINTER(_d), ctypes.POINTER(_i)]),
    'pbb_normalize_observation': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'pbb_streamed_task_order': (_i, [_i, _i, _i, _i, ctypes.POINTER(_i)]),
    'pbb_em_dispatch': (_i, [_i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    'pbb_em_last_plan': (_i, [ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    'pbb_cacgmm_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_cacgmm_fit': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp,
                            ctypes.POINTER(CacgmmOptions), _vp, _vp, _vp,
                            _vp, _sz, _vp, _vp]),
    'pbb_cacgmm_predict': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i,
                                _vp, _d, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_cacgmm_mstep': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp,
                              ctypes.POINTER(CacgmmOptions), _vp, _vp, _vp,
                              _vp, _sz, _vp, _vp]),
    'pbb_cacgmm_predict_backward_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_cacgmm_predict_backward': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _d, _vp, _vp, _vp, _vp, _vp,
                                         _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'pbb_cacgmm_mstep_backward_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_cacgmm_mstep_backward': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, ctypes.POINTER(CacgmmOptions), _vp,
                                       _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    'pbb_cwmm_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_cwmm_fit': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _i, _d,
                          _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_cwmm_predict': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _sz, _vp, _vp]),
    'pbb_cbmm_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_cbmm_fit': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _d, _d, _d,
                          _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_cbmm_predict': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _d, _vp, _vp, _sz, _vp, _vp]),
    'pbb_bingham_parameters': (_i, [_vp, _i, _i, _d, _d, _vp, _vp, _vp]),
    'pbb_bingham_log_norm': (_i, [_vp, _i, _i, _d, _vp, _vp]),
    'pbb_bingham_log_pdf': (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'pbb_heig_batched': (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_psd_workspace_bytes': (_sz, [_i, _i, _i, _i]),
    'pbb_power_spectral_density': (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    'pbb_gev_batched': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pbb_solve_batched': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    'pbb_mvdr': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_souden': (_i, [_vp, _vp, _vp, _i, _i, _d, _vp, _vp, _vp, _vp, _vp, _vp]),
    'pbb_blind_analytic_normalization': (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    'pbb_dhtv_scratch_doubles': (_sz, [_i, _i, ctypes.POINTER(_i), _i]),
    'pbb_cacg_log_pdf': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'pbb_gaussian_log_pdf': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    'pbb_gaussian_fit_scratch_doubles': (ctypes.c_size_t, [_i, _i, _i]),
    'pbb_gaussian_fit': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_log_pdf_to_affiliation': (_i, [_vp, _vp, _d, _d, _vp, _i, _vp, _d, _i, _i, _i, _i, _vp, _vp, _vp]),
    'pbb_gaussian_full_log_pdf': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'pbb_gaussian_full_fit_scratch_doubles': (_sz, [_i, _i, _i, _i]),
    'pbb_gaussian_full_fit': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_precision_cholesky': (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_vmf_log_pdf': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'pbb_vmf_resultant': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_dhtv_mapping': (_i, [_vp, _i, _i, _i, ctypes.POINTER(_i), _i, _vp, _vp, _vp, _vp]),
    'pbb_dhtv_mapping_ex': (_i, [_vp, _i, _i, _i, ctypes.POINTER(_i), _i, _vp, _vp, _vp, _i, _i, _vp]),
    'pbb_apply_mapping': (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    'pbb_score_matrix': (_i, [_vp, _vp, ctypes.c_longlong, ctypes.c_longlong, _i, _i, _i, _i, _vp, _vp]),
    'pbb_mapping_from_score_matrix': (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    'pbb_chain_mapping': (_i, [_vp, _i, _i, _vp, _vp]),
    'pbb_rank_one_estimate': (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    'pbb_matvec_batched': (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    'pbb_apply_beamforming_vector': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'pbb_apply_beamforming_vector_shared': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    'pbb_apply_beamforming_vector_backward': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_apply_beamforming_vector_shared_backward': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_power_spectral_density_backward': (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'pbb_souden_backward': (_i, [_vp, _vp, _vp, _i, _i, _i, _d, _vp, _vp, _vp]),
    'pbb_eigenvector_backward': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pbb_mvdr_backward': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_blind_analytic_normalization_backward': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pbb_rank_one_estimate_backward': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pbb_matvec_batched_backward': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pbb_solve_batched_strict': (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    'pbb_lcmv': (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_wmwf': (_i, [_vp, _vp, _i, _i, _i, _d, _vp, _vp, _vp, _vp]),
    'pbb_weighted_channel_sum': (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    'pbb_reference_channel_snr': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'pbb_mvdr_merl': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_condition_covariance': (_i, [_vp, _i, _i, _d, _vp, _vp]),
    'pbb_distortionless_normalization': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    'pbb_mvdr_snr_postfilter': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    'pbb_zero_degree_normalization': (_i, [_vp, _i, _i, _i, _vp, _vp]),
    'pbb_phase_correction': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    'pbb_apply_online_beamforming_vector': (_i, [_vp, _vp, _i, _i, _i, _i, _i, ctypes.c_longlong, ctypes.c_longlong,
                                                 ctypes.c_longlong, ctypes.c_longlong, _vp, _vp]),
    'pbb_source_mask': (_i, [_vp, _i, _i, _i, _i, _ll, _ll, _ll, _lay, _d, _vp, _vp]),
    'pbb_row_select_scratch_bytes': (_sz, [_ll, _ll]),
    'pbb_lorenz_mask': (_i, [_vp, _i, _i, _ll, _lay, _lay, _d, _d, _d, _vp, _vp, _sz, _vp, _vp]),
    'pbb_quantile_mask': (_i, [_vp, _i, _lay, _lay, _ll, _ll, _d, _d, _i, _d, _d, _vp, _vp, _sz, _vp]),
    'pbb_biased_binary_mask': (_i, [_vp, _i, _ll, _ll, _lay, _i, _vp, _vp, _vp, _vp, _vp]),
    'pbb_steering_vector': (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp]),
    'pbb_diffuse_noise_coherence': (_i, [_vp, _i, _vp, _i, _d, _vp, _vp]),
    'pbb_array_geometry': (_i, [_i, _vp, _i, _vp, _i, _i, _d, _vp, _vp]),
    'pbb_stft_frames_per_cta': (_i, [_i, _ll, _i, _i]),
    'pbb_stft': (_i, [_vp, _i, _ll, _ll, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_griffin_lim_stft': (_i, [_vp, _i, _ll, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'pbb_istft_workspace_bytes': (_sz, [_ll, _i, _i]),
    'pbb_istft': (_i, [_vp, _ll, _i, _i, _i, _i, _i, _ll, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_stft_backward_workspace_bytes': (_sz, [_ll, _i, _i]),
    'pbb_stft_backward': (_i, [_vp, _ll, _ll, _i, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_istft_backward': (_i, [_vp, _ll, _i, _i, _i, _i, _i, _ll, _vp, _vp, _vp, _vp]),
    'pbb_gammatone_chunk_length': (_i, [_ll, _i, _ll]),
    'pbb_gammatone_workspace_bytes': (_sz, [_ll, _i, _ll]),
    'pbb_gammatone': (_i, [_vp, _i, _ll, _ll, _i, _vp, _vp, _i, _vp, _sz, _vp, _vp]),
    'pbb_srmr_vad_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_srmr_vad': (_i, [_vp, _i, _ll, _ll, _d, _i, _vp, _sz, _vp, _vp, _vp, _vp]),
    'pbb_srmr_fft_log2': (_i, [_ll]),
    'pbb_srmr_hilbert_workspace_bytes': (_sz, [_ll, _ll, _ll]),
    'pbb_srmr_hilbert': (_i, [_vp, _ll, _ll, _i, _vp, _ll, _vp, _sz, _vp]),
    'pbb_srmr_means_workspace_bytes': (_sz, [_ll, _ll, _i, _i]),
    'pbb_srmr_means': (_i, [_vp, _ll, _ll, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_srmr_ratio': (_i, [_vp, _ll, _i, _vp, _vp, _vp, _vp]),
    'pbb_bss_eval_workspace_bytes': (_sz, [_ll, _i, _i, _ll]),
    'pbb_bss_eval': (_i, [_vp, _ll, _i, _i, _ll, _i, _ll, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'pbb_stoi_workspace_bytes': (_sz, [_ll, _ll, _i, _i]),
    'pbb_stoi': (_i, [_vp, _vp, _i, _ll, _ll, _i, _i, _vp, _i, _ll, _vp, _vp, _vp, _ll, _vp, _sz, _vp, _vp, _vp, _vp,
                      _vp, _vp]),
    'pbb_estoi': (_i, [_vp, _vp, _i, _ll, _ll, _i, _i, _vp, _i, _ll, _vp, _vp, _vp, _ll, _vp, _sz, _vp, _vp, _vp, _vp,
                       _vp, _vp]),
    'pbb_stoi_backward_workspace_bytes': (_sz, [_ll, _ll, _i, _i, _i]),
    'pbb_stoi_backward': (_i, [_vp, _vp, _i, _ll, _ll, _i, _i, _vp, _i, _ll, _vp, _vp, _vp, _ll, _vp, _sz, _i, _vp,
                               _vp, _vp, _vp]),
    'pbb_mean_square_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_mean_square': (_i, [_vp, _i, _ll, _ll, _vp, _sz, _vp, _vp]),
    'pbb_si_sdr_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_si_sdr': (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _vp, _sz, _vp, _vp]),
    'pbb_si_sdr_backward_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_si_sdr_backward': (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _vp, _ll, _vp, _vp, _ll, _vp, _vp, _vp, _sz, _vp, _vp,
                                 _vp]),
    'pbb_input_sxr': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_output_sxr_workspace_bytes': (_sz, [_i, _i]),
    'pbb_output_sxr': (_i, [_vp, _vp, _i, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _vp]),
    'pbb_kmeans_workspace_bytes': (_sz, [_ll, _i, _i]),
    'pbb_kmeans_fit': (_i, [_vp, _ll, _i, _i, _ll, _vp, _vp, _i, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    'pbb_kmeans_predict': (_i, [_vp, _ll, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_cacg_from_covariance': (_i, [_vp, _i, _i, _i, _d, _vp, _vp, _vp, _vp]),
    'pbb_cacg_log_pdf_floor': (_i, [_vp, _vp, _i, _i, _i, _i, _d, _vp, _vp, _vp]),
    'pbb_cw_log_norm': (_i, [_vp, _ll, _i, _i, _vp, _vp]),
    'pbb_cw_log_pdf': (_i, [_vp, _i, _ll, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_ccsg_workspace_bytes': (_sz, [_i, _i]),
    'pbb_ccsg_log_pdf': (_i, [_vp, _i, _ll, _i, _i, _i, _vp, _vp, _vp, _sz, _vp, _vp]),
    'pbb_ccsg_sample': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _ll, _i, _vp, _vp, _sz, _vp, _vp]),
    'pbb_ccsg_fit': (_i, [_vp, _i, _i, _i, _i, _vp, _d, _vp, _vp, _sz, _vp]),
    'pbb_affiliation_nd': (_i, [_vp, _i, _vp, _vp, _nd, _i, ctypes.POINTER(_ll), _d, _vp, _vp]),
    'pbb_reduce_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_axis_sum': (_i, [_vp, _i, _vp, _nd, _nd, _i, _d, _vp, _i, _vp, _sz, _vp]),
    'pbb_unit_norm': (_i, [_vp, _i, _nd, _ll, _ll, _ll, _d, _d, _i, _vp, _vp, _sz, _vp]),
    'pbb_force_hermitian': (_i, [_vp, _i, _ll, _i, _vp, _vp]),
    'pbb_abs_square': (_i, [_vp, _i, _ll, _vp, _vp]),
    'pbb_labels_to_one_hot': (_i, [_vp, _ll, _ll, _i, _i, _vp, _vp, _vp, _vp]),
    'pbb_scale_nd': (_i, [_vp, _i, _vp, _nd, _vp, _vp]),
    'pbb_vmf_pdf': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    'pbb_wpe_workspace_bytes': (_sz, [_ll, _i, _ll, _i, _i, _i]),
    'pbb_wpe': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _ll, _ll, _ll, _i, _i, _i, _ll, _i, _ll, _vp, _sz,
                     _vp, _vp]),
    'pbb_wpe_forward': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _ll, _ll, _ll, _i, _i, _i, _ll, _i, _ll, _vp,
                             _sz, _vp, _vp, _vp, _vp]),
    'pbb_wpe_step': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _ll, _ll, _vp, _ll, _ll, _ll, _i, _i, _i, _ll, _vp,
                          _sz, _vp, _vp, _vp]),
    'pbb_wpe_backward_workspace_bytes': (_sz, [_ll, _i, _ll, _i, _i, _i]),
    'pbb_wpe_backward': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _ll, _vp, _sz,
                              _vp]),
    'pbb_wpe_power_backward_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_wpe_power_backward': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _i, _i, _ll, _i, _vp, _vp, _vp, _sz,
                                    _vp]),
    'pbb_wpe_power_workspace_bytes': (_sz, [_ll, _ll]),
    'pbb_wpe_power': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _ll, _i, _vp, _vp, _sz, _vp]),
    'pbb_wpe_build_y_tilde': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _i, _i, _vp, _vp]),
    'pbb_wpe_online_smem_bytes': (_sz, [_i, _i, _i]),
    'pbb_wpe_online': (_i, [_vp, _i, _ll, _i, _ll, _ll, _ll, _ll, _vp, _ll, _ll, _ll, _vp, _vp, _vp, _vp, _ll, _ll,
                            _ll, _vp, _vp, _i, _i, _d, _vp]),
}

_lib = None


def load():
    """Loads libpbb.so (once) and attaches the signatures.  Raises ImportError
    with build instructions if the library or any declared symbol is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f'{LIB_PATH} not found: the CUDA library is not built. Run '
            '`python -c "import __graft_entry__ as g; g.build()"` or '
            '`pb_bss_b200/csrc/build.sh`. There is no CPU fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError(f'{LIB_PATH} does not export {name}; rebuild it') from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class PbbError(RuntimeError):
    pass


def check(rc, what):
    """0 -> ok; < 0 -> ValueError (bad argument, LAPACK INFO<0 convention,
    cf. get_gev_vector.pyx:130-147); > 0 -> CUDA runtime failure."""
    if rc == 0:
        return
    msg = load().pbb_last_error().decode()
    if rc < 0:
        raise ValueError(f'{what}: {msg}')
    raise PbbError(f'{what}: {msg}')
