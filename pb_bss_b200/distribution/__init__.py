"""The distributions and mixture-model trainers of pb_bss/distribution/__init__.py."""
from .gaussian import DiagonalGaussian, Gaussian, GaussianTrainer, SphericalGaussian  # noqa: F401
from .gmm import GMM, BinaryGMM, BinaryGMMTrainer, GMMTrainer  # noqa: F401
from .von_mises_fisher import VonMisesFisher, VonMisesFisherTrainer  # noqa: F401
from .complex_circular_symmetric_gaussian import (  # noqa: F401
    ComplexCircularSymmetricGaussian,
    ComplexCircularSymmetricGaussianTrainer,
)
from .complex_angular_central_gaussian import (  # noqa: F401
    ComplexAngularCentralGaussian,
    ComplexAngularCentralGaussianTrainer,
)
from .complex_watson import ComplexWatson, ComplexWatsonTrainer  # noqa: F401
from .vmfmm import VMFMM, VMFMMTrainer  # noqa: F401
from .vmfcacgmm import VMFCACGMM, VMFCACGMMTrainer  # noqa: F401
from .gcacgmm import GCACGMM, GCACGMMTrainer  # noqa: F401
from .cacgmm import CACGMM, CACGMMTrainer, sample_cacgmm, normalize_observation  # noqa: F401
from .cwmm import CWMM, CWMMTrainer  # noqa: F401
from .cbmm import CBMM, CBMMTrainer  # noqa: F401
from .complex_bingham import ComplexBingham, ComplexBinghamTrainer  # noqa: F401

from . import utils  # noqa: F401
from . import mixture_model_utils  # noqa: F401
