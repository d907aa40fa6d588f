"""pb_bss/math on the device."""
from . import solve  # noqa: F401
