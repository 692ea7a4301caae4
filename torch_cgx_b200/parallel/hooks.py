"""DDP communication hook + state (``cgx_utils`` of the reference,
/root/reference/cgx_utils/allreduce_hooks.py:29-73).

Same contract: ``model.register_comm_hook(CGXState(pg, layer_min_size, compression_params), cgx_hook)``;
on the third backward pass (``state.step == 2``, after DDP has rebuilt its
buckets) every gradient of every bucket is registered with the backend so that
1-D / small layers (biases, norms) travel uncompressed and the rest is
quantized per layer.

H100-first differences:
 * the ``tensor.div_(world)`` of the reference's ``_allreduce_fut`` is fused
   into the allreduce kernel (ReduceOp.AVG / ``allreduce_bucket(average=True)``),
   one kernel launch less per bucket and one pass less over the gradients;
 * the hook tells the backend *which* bucket it is reducing
   (``allreduce_bucket(tensor, bucket.index())``) instead of relying on a
   cyclic cursor over call order (/root/reference/src/mpi_allreduce_operations.cc:263-266).
"""

import os
from typing import Dict, Optional, Tuple, Union

import torch
import torch.distributed as dist

from .. import backend as _backend

COMPRESSION_QUANTIZATION_BITS = "CGX_COMPRESSION_QUANTIZATION_BITS"
COMPRESSION_BUCKET_SIZE = "CGX_COMPRESSION_BUCKET_SIZE"
COMPRESSION_MINIMAL_SIZE = "CGX_COMPRESSION_MINIMAL_SIZE"
VALUE_NO_COMPRESS = 32


def _width_and_format(bits: Union[int, str]) -> Tuple[int, Optional[str]]:
    """``bits`` of the compressed allreduce: a max-min width, or an FP8 format name ("e4m3",
    "e5m2", "e4m3_pow2", "e5m2_pow2", "e4m3_sr" or "e5m2_sr"), whose layers are compressed at 8 bits.
    ValueError for any other name."""
    if not isinstance(bits, str):
        return int(bits), None
    from .. import _C

    _C.a2a_bits(bits, False, "allreduce")
    return 8, bits


class CGXState(object):
    """State of :func:`cgx_hook` (argument-compatible with the reference).

    ``compression_params["bits"]`` is a max-min width or an FP8 format, ``"e4m3"`` or ``"e5m2"``
    (the usual choice for gradients), ``"e4m3_pow2"`` / ``"e5m2_pow2"`` with power-of-two scales, or
    ``"e4m3_sr"`` / ``"e5m2_sr"``, rounded stochastically with each rank's own random stream:
    the compressed layers are then registered at 8 bits and sent as FP8 codes with one fp32 scale
    per bucket. ``quantization_bits`` holds the width and
    ``quantization_format`` the format name (None: max-min, or ``CGX_COMPRESSION_FORMAT``'s).
    """

    def __init__(
        self,
        process_group: Optional[dist.ProcessGroup] = None,
        layer_min_size: int = 1024,
        compression_params: Optional[Dict[str, int]] = None,
    ):
        self.process_group = process_group if process_group is not None else dist.group.WORLD
        min_size_to_compress = int(os.getenv(COMPRESSION_MINIMAL_SIZE, "16"))
        self.layer_min_size = max(layer_min_size, min_size_to_compress)
        self.quantization_bits = int(os.getenv(COMPRESSION_QUANTIZATION_BITS, str(VALUE_NO_COMPRESS)))
        self.quantization_bucket_size = int(os.getenv(COMPRESSION_BUCKET_SIZE, "1024"))
        self.quantization_format: Optional[str] = None
        self.step = 0
        self.layer_idx = 0
        # step at which layers are registered (DDP rebuilds buckets after the 1st iteration)
        self.register_step = 2
        if compression_params is not None:
            self.quantization_bits, self.quantization_format = _width_and_format(
                compression_params.get("bits", self.quantization_bits))
            self.quantization_bucket_size = compression_params.get("bucket_size", self.quantization_bucket_size)

    def should_compress_(self, tensor: torch.Tensor) -> bool:
        if tensor.dim() <= 1 or tensor.numel() < self.layer_min_size:
            return False
        return True

    # checkpoint / resume: the only cross-step state is the step counter (the
    # layer table is rebuilt from it) -- the reference has none at all.
    def state_dict(self) -> Dict[str, int]:
        return {
            "step": self.step,
            "layer_min_size": self.layer_min_size,
            "quantization_bits": self.quantization_format or self.quantization_bits,
            "quantization_bucket_size": self.quantization_bucket_size,
        }

    def load_state_dict(self, sd: Dict[str, int]) -> None:
        self.layer_min_size = int(sd.get("layer_min_size", self.layer_min_size))
        self.quantization_bits, self.quantization_format = _width_and_format(
            sd.get("quantization_bits", self.quantization_format or self.quantization_bits))
        self.quantization_bucket_size = int(sd.get("quantization_bucket_size", self.quantization_bucket_size))
        # layers must be re-registered with the (new) process: restart the warm-up
        self.step = 0


_NATIVE_CACHE = {}


def _native_backend(group, tensor: torch.Tensor):
    # resolved once per (group, device type): the lookup costs several microseconds per bucket
    key = (id(group), tensor.device.type)
    hit = _NATIVE_CACHE.get(key)
    if hit is None or hit[0] is not group:
        hit = (group, _backend.get_backend(group, tensor.device))
        _NATIVE_CACHE[key] = hit
    return hit[1]


def _allreduce_fut(process_group, tensor: torch.Tensor, bucket_idx: int = -1,
                   fmt: Optional[str] = None) -> torch.futures.Future[torch.Tensor]:
    """Average ``tensor`` across the group, return a future of the tensor. ``fmt``: the FP8 format
    of the 8-bit layers (None: ``CGX_COMPRESSION_FORMAT``'s)."""
    group_to_use = process_group if process_group is not None else dist.group.WORLD
    native = _native_backend(group_to_use, tensor)
    if native is not None:
        # 1/world is applied inside the kernel, before quantization (same
        # numerics as the reference's div-then-allreduce, without the extra pass)
        work = native.allreduce_bucket(tensor, bucket_idx, True, fmt)
        return work.get_future().then(lambda fut: fut.value()[0])
    # any other backend (nccl / gloo): the reference's recipe verbatim
    tensor.div_(group_to_use.size())
    return (
        dist.all_reduce(tensor, group=group_to_use, async_op=True)
        .get_future()
        .then(lambda fut: fut.value()[0])
    )


def cgx_hook(state: CGXState, bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]:
    per_bucket = getattr(state, "bucket_hook", None)  # AdaptiveCGXState runs its own per-bucket logic
    if per_bucket is not None:
        return per_bucket(bucket)
    if state.step == state.register_step:
        for layer_idx, tensor in enumerate(bucket.gradients()):
            bits = state.quantization_bits if state.should_compress_(tensor) else VALUE_NO_COMPRESS
            _backend.register_layer(bucket.index(), layer_idx, tensor.numel(), bits, state.quantization_bucket_size)
    registered = state.step >= state.register_step
    if bucket.is_last():
        state.step += 1
        state.layer_idx = 0
    return _allreduce_fut(state.process_group, bucket.buffer(), bucket.index() if registered else -1,
                          state.quantization_format)


def register_cgx_hook(ddp_model, state: CGXState, native: Optional[bool] = None):
    """Install the compressed-allreduce hook on a DistributedDataParallel model.

    ``native=None`` (default): with the ``cgx`` backend a :class:`CGXState` gets the **native C++
    hook**, registered directly on DDP's reducer (no Python in the per-bucket path); with any other
    backend, and for an :class:`~torch_cgx_b200.AdaptiveCGXState`, this falls back to
    ``ddp_model.register_comm_hook(state, cgx_hook)``.

    ``native=True`` installs the native hook for either state, adaptive widths included; it raises
    ``ValueError`` when the group has no ``cgx`` backend. ``native=False`` always installs the Python
    hook. Returns the native state handle (also stored as ``state.native``) or None.
    """
    from .. import _C

    params = [p for p in ddp_model.parameters() if p.requires_grad]
    device = params[0].device if params else torch.device("cpu")
    backend = _backend.get_backend(state.process_group, device)
    adaptive = hasattr(state, "bucket_hook")
    if native is None:
        native = backend is not None and not adaptive
    elif native and backend is None:
        raise ValueError("register_cgx_hook(native=True) needs a process group with the cgx backend")
    if not native:
        ddp_model.register_comm_hook(state, cgx_hook)
        return None
    extra = {}
    if adaptive:
        extra = dict(candidates=list(state.candidate_bits), period=int(state.period), assignment=dict(state._loaded))
    handle = _C.register_native_hook(ddp_model.reducer, backend, int(state.layer_min_size),
                                     state.quantization_format or int(state.quantization_bits),
                                     int(state.quantization_bucket_size),
                                     int(state.register_step), **extra)
    try:
        ddp_model.logger._set_comm_hook_name("cgx_native_hook")
    except Exception:  # noqa: BLE001
        pass
    state.native = handle
    return handle
