from .module_mir_eval import mir_eval_sources  # noqa: F401
from .module_si_sdr import si_sdr  # noqa: F401
from .module_srmr import srmr  # noqa: F401
from .module_stoi import stoi  # noqa: F401
from .wrapper import InputMetrics, OutputMetrics  # noqa: F401

__all__ = ['mir_eval_sources', 'si_sdr', 'srmr', 'stoi', 'InputMetrics', 'OutputMetrics']
