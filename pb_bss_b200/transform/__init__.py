from .fourier import stft, istft  # noqa: F401
from .griffin_lim_module import GriffinLim, MISI  # noqa: F401

__all__ = ['stft', 'istft', 'GriffinLim', 'MISI']
