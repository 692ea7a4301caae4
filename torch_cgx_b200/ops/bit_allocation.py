"""Per-layer bit widths under a byte budget (adaptive layer-wise compression).

``allocate_bits`` picks one candidate width per layer so that the summed quantization error
(``quantization_error``) is smallest while the summed wire bytes stay within a budget: a
multiple-choice knapsack, solved by dynamic programming over the budget split into ``resolution``
bins. Host logic that runs once per adaptation period, in C++ (``csrc/common/bit_allocation.cc``);
the native DDP hook calls the same function. ``ops.oracle.allocate_bits_reference`` is its NumPy
twin.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np

from .. import _C


def layer_wire_bytes(numel: int, bits: int, bucket_size: int) -> int:
    """Wire bytes of one layer at ``bits``, with the bucket clamped as the plan clamps it."""
    return _C.layer_wire_bytes(int(numel), int(bits), int(bucket_size))


def allocate_bits(
    errors,
    numels: Sequence[int],
    bucket_sizes: Sequence[int],
    candidates: Sequence[int],
    budget_bytes: int,
    current: Optional[Sequence[int]] = None,
    resolution: int = 4096,
    *,
    target_bits: Optional[int] = None,
) -> List[int]:
    """Width per layer minimising sum(errors[l, k]) subject to sum(wire bytes) <= ``budget_bytes``.

    * ``errors``: ``[L, K]`` array-like, the error of layer ``l`` at ``candidates[k]``.
    * Layer costs are :func:`~torch_cgx_b200.ops.wire_bytes`. Each is rounded *up* to whole bins of
      ``budget / resolution`` bytes, so whatever the search returns fits the budget.
    * ``target_bits`` is the uniform width the budget was derived from; by default the widest
      candidate whose uniform assignment fits. If the search ends with more error than the uniform
      assignment at that width, the uniform assignment is returned.
    * A layer with a non-finite error keeps its ``current`` width (``target_bits`` when
      ``current`` is None); its bytes at that width come off the budget.
    * Ties go to fewer bytes, then to the lower candidate index: equal inputs give equal outputs.
    """
    err = np.asarray(errors, dtype=np.float64)
    cands = [int(c) for c in candidates]
    L, K = len(numels), len(cands)
    if err.shape != (L, K):
        raise ValueError(f"allocate_bits: errors has shape {err.shape}, expected ({L}, {K})")
    if K == 0 or resolution < 1:
        raise ValueError("allocate_bits: need at least one candidate and resolution >= 1")
    if len(bucket_sizes) < L:
        raise ValueError(f"allocate_bits: {len(bucket_sizes)} bucket sizes for {L} layers")
    # costs are whole bytes, so sum <= budget and sum <= floor(budget) agree
    return _C.allocate_bits(np.ascontiguousarray(err), [int(n) for n in numels],
                            [int(b) for b in list(bucket_sizes)[:L]], cands, math.floor(budget_bytes),
                            None if current is None else [int(c) for c in current], int(resolution),
                            None if target_bits is None else int(target_bits))
