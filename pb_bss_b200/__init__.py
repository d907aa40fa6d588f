"""pb_bss_b200 -- H100-native drop-in for the EM hot path of fgnt/pb_bss.

Host side: Python mirroring the reference's public API for this path
(``distribution.CACGMMTrainer/CACGMM/CWMMTrainer/CWMM``,
``extraction.get_power_spectral_density_matrix/get_mvdr_vector/get_gev_vector``,
``permutation_alignment.DHTVPermutationAlignment``), plus the STFT / iSTFT ends and
Griffin-Lim / MISI (``transform``).  All arithmetic runs in
hand-written sm_90a CUDA kernels behind the C ABI of ``include/pbb.h``
(``libpbb.so``, bound with ctypes in ``_lib.py``); torch tensors are only the
device-memory containers.  There is no CPU fallback.
"""
import pathlib

from . import _lib  # noqa: F401  (import must not need a GPU)
from . import distribution  # noqa: F401
from . import evaluation  # noqa: F401
from . import extraction  # noqa: F401
from . import permutation_alignment  # noqa: F401
from . import initializer  # noqa: F401
from . import transform  # noqa: F401
from . import math  # noqa: F401
from . import utils  # noqa: F401
from ._device import deferred_status  # noqa: F401

# the reference's pb_bss.project_root: the directory that holds the package
project_root = pathlib.Path(__file__).expanduser().absolute().parent.parent

__all__ = ['distribution', 'extraction', 'permutation_alignment', 'initializer', 'transform']
