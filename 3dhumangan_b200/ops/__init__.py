"""`lib.components.ops` surface: bias_act and upfirdn2d on sm_90a (no 'ref' implementation, no JIT plugin)."""
from . import bias_act, upfirdn2d  # noqa: F401
