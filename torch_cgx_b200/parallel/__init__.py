from .functional import all_reduce, compression, differentiable_all_to_all_dispatch  # noqa: F401
from .hooks import CGXState, cgx_hook, register_cgx_hook  # noqa: F401
