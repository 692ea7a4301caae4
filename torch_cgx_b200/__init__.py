"""torch_cgx_b200 -- Hopper-native compressed-gradient allreduce for PyTorch.

Importing this package loads the native extension and registers the
``torch.distributed`` backend ``"cgx"`` (the reference does the same from a
static constructor in its .so, /root/reference/src/ProcessGroupCGX.h:258-263)::

    import torch_cgx_b200            # or: import torch_cgx  (drop-in alias)
    dist.init_process_group("cgx", init_method="env://")
    model = DDP(model)
    from torch_cgx_b200 import CGXState, cgx_hook
    model.register_comm_hook(CGXState(None, compression_params={"bits": 4, "bucket_size": 512}), cgx_hook)
"""
from __future__ import annotations

__version__ = "0.1.0"

from ._loader import load_native

_C = load_native()

from .backend import (  # noqa: E402
    BACKEND_NAME,
    get_backend,
    register_backend,
    register_layer,
    reset_layers,
    set_quantization_bits,
    set_quantization_bucket_size,
)
from .parallel.functional import (  # noqa: E402
    all_gather_into_tensor,
    all_reduce,
    all_to_all_combine,
    all_to_all_single,
    compression,
    differentiable_all_to_all_combine,
    differentiable_all_to_all_dispatch,
    differentiable_all_to_all_single,
    reduce_scatter_tensor,
)
from .parallel.fsdp import (  # noqa: E402
    CGXAllGather,
    CGXReduceScatter,
    fsdp_shard_table,
    set_cgx_all_gather,
    set_cgx_reduce_scatter,
)
from .parallel.hooks import CGXState, cgx_hook, register_cgx_hook  # noqa: E402
from .parallel.adaptive import AdaptiveCGXState  # noqa: E402
from .parallel.adaptive_fsdp import AdaptiveFSDPState, set_cgx_adaptive  # noqa: E402
from .utils.launch import map_launcher_env  # noqa: E402
from . import models, ops, utils  # noqa: E402,F401

register_backend()

__all__ = [
    "AdaptiveCGXState",
    "AdaptiveFSDPState",
    "BACKEND_NAME",
    "CGXAllGather",
    "CGXReduceScatter",
    "CGXState",
    "all_gather_into_tensor",
    "all_reduce",
    "cgx_hook",
    "compression",
    "fsdp_shard_table",
    "get_backend",
    "map_launcher_env",
    "register_backend",
    "register_cgx_hook",
    "reduce_scatter_tensor",
    "all_to_all_single",
    "all_to_all_combine",
    "differentiable_all_to_all_single",
    "differentiable_all_to_all_combine",
    "differentiable_all_to_all_dispatch",
    "register_layer",
    "reset_layers",
    "set_quantization_bits",
    "set_cgx_adaptive",
    "set_cgx_all_gather",
    "set_cgx_reduce_scatter",
    "set_quantization_bucket_size",
]
