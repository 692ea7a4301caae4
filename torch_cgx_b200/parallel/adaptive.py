"""Adaptive per-layer bit widths for the DDP hook.

``AdaptiveCGXState`` keeps the *average* width of ``compression_params["bits"]`` but moves bits to
the layers where quantization hurts most. Every ``period`` steps it estimates, per layer and
candidate width, the squared error one quantization round trip would add to the local gradient
(``ops.quantization_error``, one kernel per bucket, before the bucket's allreduce overwrites it).
At the first bucket of the next step it sums the estimates over the group, rank 0 picks the widths
(``ops.allocate_bits``: least total error within the wire bytes of the uniform width) and
broadcasts them, and every rank applies the broadcast widths with ``set_quantization_bits``. Only
broadcast widths are ever applied: ranks that disagreed on a layer's width would corrupt the
allreduce.

Usage (the Python hook; ``register_cgx_hook`` installs it too and returns None)::

    state = cgx.AdaptiveCGXState(None, compression_params={"bits": 4, "bucket_size": 1024}, period=1000)
    ddp.register_comm_hook(state, cgx.cgx_hook)

On a ``cgx`` group, ``cgx.register_cgx_hook(ddp, state, native=True)`` runs the same steps in the
native C++ hook (``csrc/pg/comm_hook.cc``) with the same results; ``assignment``, ``last_errors``,
``adapted_layers``, ``state_dict`` and ``load_state_dict`` then read and write the native state.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .. import _C
from .. import backend as _backend
from ..ops.bit_allocation import allocate_bits, layer_wire_bytes
from ..ops.quantization import quantization_error
from .hooks import VALUE_NO_COMPRESS, CGXState, _allreduce_fut


def _capturing() -> bool:
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


# (numels, bucket_sizes, budget_bytes, current widths, target_bits) of consecutive table rows
AllocationPart = Tuple[Sequence[int], Sequence[int], int, Sequence[int], int]


def _sum_allocate_broadcast(tables: Sequence[torch.Tensor], parts: Sequence[AllocationPart],
                            candidate_bits: Sequence[int], group: dist.ProcessGroup,
                            device: torch.device) -> Tuple[torch.Tensor, List[int]]:
    """The decision step of the adaptive states: sum the concatenated float64 estimate tables over
    ``group``, run one ``allocate_bits`` per part on group rank 0, broadcast its int32 widths.

    ``tables`` are ``[rows, len(candidate_bits)]`` estimates in row order; ``parts`` split those
    rows into consecutive ranges that are allocated separately. Returns the summed table (CPU,
    ``[rows, K]``) and the broadcast width of every row, the same on every rank."""
    K = len(candidate_bits)
    table = torch.cat([t.reshape(-1) for t in tables])
    # float64 never takes the compressed path: the sum does not depend on any CGX_* width setting
    dist.all_reduce(table, group=group)
    table = table.view(-1, K).cpu()
    assert table.shape[0] == sum(len(p[0]) for p in parts)
    choice = torch.zeros(table.shape[0], dtype=torch.int32)
    if group.rank() == 0:
        picked, r = [], 0
        for numels, buckets, budget, current, target in parts:
            n = len(numels)
            picked += allocate_bits(table[r:r + n].numpy(), numels, buckets, candidate_bits, budget, current,
                                    target_bits=target)
            r += n
        choice = torch.tensor(picked, dtype=torch.int32)
    choice = choice.to(device)
    dist.broadcast(choice, src=dist.get_global_rank(group, 0), group=group)
    return table, choice.cpu().tolist()


class AdaptiveCGXState(CGXState):
    """:class:`CGXState` whose compressed layers get widths chosen from ``candidate_bits``.

    ``compression_params["bits"]`` sets the average: the budget is the wire bytes all adapted
    layers take at that uniform width. Which layers are compressed is decided exactly as in
    :class:`CGXState`. After a decision, ``assignment`` maps ``(bucket, layer)`` to its width and
    ``last_errors`` holds the group-summed error table (rows in ``adapted_layers`` order, columns in
    ``candidate_bits`` order). Estimate and decision steps cannot run inside CUDA graph capture.
    """

    def __init__(
        self,
        process_group: Optional[dist.ProcessGroup] = None,
        layer_min_size: int = 1024,
        compression_params: Optional[Dict[str, int]] = None,
        candidate_bits: Sequence[int] = (2, 3, 4, 5, 6, 7, 8),
        period: int = 1000,
    ):
        super().__init__(process_group, layer_min_size, compression_params)
        if self.quantization_format is not None:
            raise ValueError("AdaptiveCGXState: adaptive widths do not take FP8 formats, got "
                             f"bits={self.quantization_format!r}")
        self.candidate_bits = tuple(int(b) for b in candidate_bits)
        if not self.candidate_bits or any(b < 1 or b > 8 for b in self.candidate_bits):
            raise ValueError(f"candidate_bits must be widths in 1..8, got {candidate_bits}")
        if period < 1:
            raise ValueError(f"period must be >= 1, got {period}")
        self.period = int(period)
        self.native = None  # the native hook's state, once register_cgx_hook(..., native=True) installed it
        self.assignment: Dict[Tuple[int, int], int] = {}
        self.last_errors: Optional[torch.Tensor] = None
        self.adapted_layers: list = []  # (bucket, layer, elem_off, numel), registration order
        self._by_bucket: Dict[int, list] = {}
        self._tables: Dict[int, torch.Tensor] = {}  # bucket -> [layers, candidates] estimate
        self._loaded: Dict[Tuple[int, int], int] = {}
        self._step_open = False
        self._device = torch.device("cpu")

    # ---- state of whichever hook runs: the native one once installed --------------------------
    @property
    def assignment(self) -> Dict[Tuple[int, int], int]:
        return dict(self.native.assignment) if self.native is not None else self._assignment

    @assignment.setter
    def assignment(self, value: Dict[Tuple[int, int], int]) -> None:
        self._assignment = value

    @property
    def last_errors(self) -> Optional[torch.Tensor]:
        return self.native.last_errors if self.native is not None else self._last_errors

    @last_errors.setter
    def last_errors(self, value: Optional[torch.Tensor]) -> None:
        self._last_errors = value

    @property
    def adapted_layers(self) -> list:
        return list(self.native.adapted_layers) if self.native is not None else self._adapted_layers

    @adapted_layers.setter
    def adapted_layers(self, value: list) -> None:
        self._adapted_layers = value

    # ---- checkpoint -------------------------------------------------------------------------
    def state_dict(self) -> Dict:
        sd = super().state_dict()
        sd["assignment"] = dict(self.assignment)
        return sd

    def load_state_dict(self, sd: Dict) -> None:
        super().load_state_dict(sd)
        self._loaded = {tuple(k): int(v) for k, v in dict(sd.get("assignment", {})).items()}
        if self.native is not None:
            self.native.load_assignment(self._loaded)

    # ---- per-bucket hook body (called by cgx_hook) -------------------------------------------
    def bucket_hook(self, bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]:
        b = bucket.index()
        if not self._step_open:
            self._step_open = True
            if self._tables:
                self._decide()
        if self.step == self.register_step:
            self._register(bucket)
        adapt = self.quantization_bits <= 8 and self.step >= self.register_step
        if adapt and (self.step - self.register_step) % self.period == 0 and self._by_bucket.get(b):
            self._estimate(b, bucket.buffer())
        registered = self.step >= self.register_step
        if bucket.is_last():
            self.step += 1
            self.layer_idx = 0
            self._step_open = False
        return _allreduce_fut(self.process_group, bucket.buffer(), b if registered else -1)

    def _register(self, bucket: dist.GradBucket) -> None:
        b, off, mine = bucket.index(), 0, []
        for layer_idx, tensor in enumerate(bucket.gradients()):
            compress = self.should_compress_(tensor)
            bits = self.quantization_bits if compress else VALUE_NO_COMPRESS
            _backend.register_layer(b, layer_idx, tensor.numel(), bits, self.quantization_bucket_size)
            if compress and self.quantization_bits <= 8:
                mine.append((b, layer_idx, off, tensor.numel()))
            off += tensor.numel()
        self._by_bucket[b] = mine
        self.adapted_layers = [l for k in sorted(self._by_bucket) for l in self._by_bucket[k]]
        for (_, layer_idx, _, _) in mine:
            bits = self._loaded.get((b, layer_idx))
            if bits is not None:
                _backend.set_quantization_bits(b, layer_idx, bits)
                self.assignment[(b, layer_idx)] = bits

    def _estimate(self, b: int, buf: torch.Tensor) -> None:
        if _capturing():
            raise RuntimeError("AdaptiveCGXState: an estimate step cannot run during CUDA graph capture")
        cfg = _C.engine_config()
        layers = [(off, n, self.quantization_bits, self.quantization_bucket_size) for (_, _, off, n) in self._by_bucket[b]]
        world = self.process_group.size()
        self._device = buf.device
        # the estimate is enqueued before the in-place allreduce, on the same stream: no synchronisation
        self._tables[b] = quantization_error(buf, layers, self.candidate_bits, stochastic=bool(cfg["stochastic"]),
                                             prescale=1.0 / world, skip_incomplete=bool(cfg["skip_incomplete"]))

    def _decide(self) -> None:
        if _capturing():
            raise RuntimeError("AdaptiveCGXState: a decision step cannot run during CUDA graph capture")
        keys = sorted(self._tables)
        tables = [self._tables[k] for k in keys]
        self._tables = {}
        rows = [l for k in keys for l in self._by_bucket[k]]
        bs = self.quantization_bucket_size
        numels = [n for (_, _, _, n) in rows]
        budget = sum(layer_wire_bytes(n, self.quantization_bits, bs) for n in numels)
        current = [self.assignment.get((b, l), self.quantization_bits) for (b, l, _, _) in rows]
        table, choice = _sum_allocate_broadcast(
            tables, [(numels, [bs] * len(rows), budget, current, self.quantization_bits)], self.candidate_bits,
            self.process_group, self._device)
        for (b, l, _, _), bits in zip(rows, choice):
            _backend.set_quantization_bits(b, l, bits)
            self.assignment[(b, l)] = bits
        self.last_errors = table
