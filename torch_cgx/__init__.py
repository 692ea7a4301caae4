"""Drop-in alias of the reference's extension module name: ``import torch_cgx``
registers the ``cgx`` backend and exposes ``register_layer`` /
``set_quantization_bits`` / ``set_quantization_bucket_size``
(/root/reference/src/ProcessGroupCGX.cc:852-857, README.md:40-48)."""
from torch_cgx_b200 import (  # noqa: F401
    all_to_all_single,
    differentiable_all_to_all_single,
    register_backend,
    register_layer,
    reset_layers,
    set_quantization_bits,
    set_quantization_bucket_size,
)
from torch_cgx_b200.backend import _create_backend as createProcessGroupCGX  # noqa: F401,N812
