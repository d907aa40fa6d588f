"""Beamforming side of the hot path (pb_bss/extraction)."""
from . import linalg  # noqa: F401
from .beamformer import (  # noqa: F401
    apply_beamforming_vector,
    apply_online_beamforming_vector,
    blind_analytic_normalization,
    condition_covariance,
    distortionless_normalization,
    get_gev_vector,
    get_lcmv_vector,
    get_lcmv_vector_souden,
    get_mvdr_vector,
    get_mvdr_vector_merl,
    get_mvdr_vector_souden,
    get_optimal_reference_channel,
    get_pca,
    get_pca_vector,
    get_power_spectral_density_matrix,
    get_wmwf_vector,
    mvdr_snr_postfilter,
    phase_correction,
    zero_degree_normalization,
)
from .beamformer_wrapper import get_bf_vector  # noqa: F401
from .beamformer_wrapper import get_bf_vector as get_single_source_bf_vector  # noqa: F401
from . import mask_module  # noqa: F401
from .mask_module import (  # noqa: F401
    biased_binary_mask,
    ideal_amplitude_mask,
    ideal_binary_mask,
    ideal_complex_mask,
    ideal_ratio_mask,
    lorenz_mask,
    phase_sensitive_mask,
    quantile_mask,
    voiced_unvoiced_split_characteristic,
    wiener_like_mask,
)
