"""Tensor-level ops backed by the native kernels (CUDA) or the C++ CPU path."""
from .bit_allocation import allocate_bits  # noqa: F401
from .quantization import compression_ratio, dequantize, fake_quantize, quantization_error, quantize, wire_bytes  # noqa: F401
