"""pb_bss/math/solve.py: ``stable_solve`` is the device solver of extraction.linalg (pbb_solve_batched)."""
from ..extraction.linalg import stable_solve  # noqa: F401

__all__ = ['stable_solve']
