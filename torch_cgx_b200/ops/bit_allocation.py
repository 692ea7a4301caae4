"""Per-layer bit widths under a byte budget (adaptive layer-wise compression).

``allocate_bits`` picks one candidate width per layer so that the summed quantization error
(``quantization_error``) is smallest while the summed wire bytes stay within a budget: a
multiple-choice knapsack, solved by dynamic programming over the budget split into ``resolution``
bins. Host logic that runs once per adaptation period.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from .quantization import wire_bytes

MAX_BUCKET = 8192  # the plan clamps quantization buckets to this (csrc/common/wire.h: kMaxBlockElems)


def layer_wire_bytes(numel: int, bits: int, bucket_size: int) -> int:
    """Wire bytes of one layer at ``bits``, with the bucket clamped as the plan clamps it."""
    return wire_bytes(int(numel), int(bits), max(1, min(int(bucket_size), MAX_BUCKET)))


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
    cost = np.array([[layer_wire_bytes(n, b, bs) for b in cands] for n, bs in zip(numels, bucket_sizes)],
                    dtype=np.int64).reshape(L, K)
    if target_bits is None:
        fits = [k for k in range(K) if cost[:, k].sum() <= budget_bytes]
        target_bits = max(cands[k] for k in fits) if fits else min(cands)
    keep = [int(c) for c in current] if current is not None else [int(target_bits)] * L
    out = list(keep)
    finite = np.isfinite(err).all(axis=1)
    free = [l for l in range(L) if finite[l]]
    fixed_bytes = sum(layer_wire_bytes(numels[l], keep[l], bucket_sizes[l]) for l in range(L) if not finite[l])
    room = int(budget_bytes) - fixed_bytes
    k_t = cands.index(target_bits) if target_bits in cands else None
    uniform = list(out)
    for l in free:
        uniform[l] = int(target_bits)
    if not free or room <= 0:
        return uniform

    # bins[l, k] = ceil(cost * resolution / room): any choice with sum(bins) <= resolution fits
    R = int(resolution)
    bins = (cost[free] * R + room - 1) // room
    e = err[free]
    # candidates visited in (bytes, index) order with strict improvement: ties keep fewer bytes
    order = np.lexsort((np.arange(K)[None, :].repeat(len(free), 0), cost[free]), axis=1)
    dp = np.zeros(R + 1)  # least error of the layers so far within c bins
    choice = np.zeros((len(free), R + 1), dtype=np.int16)
    for i in range(len(free)):
        best = np.full(R + 1, np.inf)
        pick = np.zeros(R + 1, dtype=np.int16)
        for k in order[i]:
            c = int(bins[i, k])
            if c > R:
                continue
            cand = np.full(R + 1, np.inf)
            cand[c:] = dp[: R + 1 - c] + e[i, k]
            better = cand < best
            best[better] = cand[better]
            pick[better] = k
        dp, choice[i] = best, pick
    if not np.isfinite(dp[R]):
        return uniform
    c = int(np.argmax(dp == dp[R]))  # fewest bins that reach the least error (dp is non-increasing)
    total = dp[R]
    for i in range(len(free) - 1, -1, -1):
        k = int(choice[i, c])
        out[free[i]] = cands[k]
        c -= int(bins[i, k])
    if k_t is not None and cost[free, k_t].sum() <= room and total > e[:, k_t].sum():
        return uniform
    return out
