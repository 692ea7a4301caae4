"""Hostile inputs for the quantizer and the allreduce, shared by the CPU and the GPU tests.

``edge_inputs`` fills one layer of ``n`` elements per rank with random buckets and plants
one edge case into every other bucket (so that every planted bucket has clean neighbours):

    non-finite      one NaN; +Inf; -Inf; both +-Inf; all +Inf (max - min is NaN); all NaN
    span overflow   fp32/bf16 values near +-3e38: max - min overflows, every value finite
    threshold       spans that put unit just below / just above kQuantEps (1e-10)
    tiny            subnormals of the dtype
    wide range      a huge value next to a tiny one in one bucket
    zeros           constant buckets of +0 and of -0
    fp16 overflow   fp16 values near 30000 whose W-rank sum overflows to inf
    outlier         one outlier at element 0, 7, 8, 15, 16, 255 or B-1 of its bucket

Non-finite values sit on one rank only: the bucket's owner or one of its peers (the
owner's accumulator and a peer's quantizer are different code). Finite cases are planted on
every rank. ``bits`` only steers the threshold case.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

NONFINITE = ("nan", "pinf", "ninf", "both_inf", "all_pinf", "all_nan")
FINITE = ("span_overflow", "eps_below", "eps_above", "tiny", "wide_range", "pzero", "nzero", "f16_overflow",
          "outlier")
CASES = NONFINITE + FINITE
OUTLIER_POS = (0, 7, 8, 15, 16, 255)


@dataclass
class Planted:
    case: str
    lo: int       # first element (relative to the layer)
    hi: int
    rank: int     # rank holding a non-finite value, -1 for finite cases (all ranks)

    @property
    def nonfinite(self) -> bool:
        return self.case in NONFINITE


def _applicable(case: str, dtype: torch.dtype) -> bool:
    if case == "span_overflow":
        return dtype != torch.float16   # fp16 cannot hold values whose difference overflows fp32
    if case in ("eps_below", "eps_above"):
        return dtype != torch.float16   # the smallest fp16 step already gives unit > 1e-10
    if case == "f16_overflow":
        return dtype == torch.float16
    return True


def _tiny(dtype: torch.dtype) -> float:
    return {torch.float32: 1e-40, torch.float16: 6e-8, torch.bfloat16: 1e-39}[dtype]


def _fill(case: str, m: int, rank: int, dtype: torch.dtype, bits: int, g: torch.Generator, opos: int) -> torch.Tensor:
    """Values of one planted bucket of m elements on `rank` (finite cases)."""
    r = torch.rand(m, generator=g, dtype=torch.float64)
    if case == "span_overflow":
        v = (r * 2 - 1) * 3.0e38
        v[0], v[-1] = 3.2e38, -3.2e38
    elif case in ("eps_below", "eps_above"):
        # unit = span * fp32(1/levels): a span 1% off the threshold stays on its side after rounding
        span = 1e-10 * ((1 << bits) - 1) * (0.99 if case == "eps_below" else 1.01)
        base = 1e-6 if dtype == torch.float32 else 0.0
        v = base + r * span
        v[0], v[-1] = base, base + span
    elif case == "tiny":
        v = torch.round(r * 40) * _tiny(dtype) * (1 if rank % 2 == 0 else -1)
    elif case == "wide_range":
        big, small = (6e4, 6e-8) if dtype == torch.float16 else (1e30, 1e-30)
        v = (r * 2 - 1) * small
        v[m // 2] = big
    elif case == "pzero":
        v = torch.zeros(m, dtype=torch.float64)
    elif case == "nzero":
        v = torch.full((m,), -0.0, dtype=torch.float64)
    elif case == "f16_overflow":
        v = 30000.0 + r * 2000.0
    elif case == "outlier":
        v = torch.randn(m, generator=g, dtype=torch.float64)
        v[opos] = 1000.0 * (rank + 1)
    else:
        raise ValueError(case)
    return v.to(dtype)


def _poison(case: str, seg: torch.Tensor, g: torch.Generator) -> None:
    m = seg.numel()
    i = int(torch.randint(0, m, (1,), generator=g))
    j = (i + m // 2) % m if m > 1 else i
    if case == "nan":
        seg[i] = float("nan")
    elif case == "pinf":
        seg[i] = float("inf")
    elif case == "ninf":
        seg[i] = float("-inf")
    elif case == "both_inf":
        seg[i] = float("inf")
        seg[j] = float("-inf")
    elif case == "all_pinf":
        seg.fill_(float("inf"))
    elif case == "all_nan":
        seg.fill_(float("nan"))
    else:
        raise ValueError(case)


def edge_inputs(dtype: torch.dtype, n: int, bucket: int, seed: int, *, world: int = 1, bits: int = 4,
                owners: Optional[Sequence[int]] = None, where: str = "owner",
                cases: Sequence[str] = CASES) -> tuple[List[torch.Tensor], List[Planted]]:
    """``world`` tensors of ``n`` elements (one layer, buckets of ``bucket`` from element 0) and the
    list of planted buckets.

    ``owners[i]`` is the rank that reduces element i (SRA); a non-finite value goes to that rank
    (``where="owner"``) or to the next one (``where="peer"``). Without ``owners`` rank 0 is used.
    """
    assert where in ("owner", "peer")
    g = torch.Generator().manual_seed(seed)
    outs = [(torch.randn(n, generator=g, dtype=torch.float64) * (r + 1)).to(dtype) for r in range(world)]
    planted: List[Planted] = []
    todo = [c for c in cases if _applicable(c, dtype)]
    # one outlier bucket per position that exists in a bucket of this size, B-1 included
    expanded = []
    for c in todo:
        if c == "outlier":
            expanded += [("outlier", p) for p in sorted({p for p in OUTLIER_POS if p < bucket} | {bucket - 1})]
        else:
            expanded.append((c, 0))
    nb = -(-n // bucket)
    for k, (case, opos) in enumerate(expanded):
        b = 2 * k + 1
        if b >= nb:
            break
        lo, hi = b * bucket, min(n, (b + 1) * bucket)
        if case == "outlier" and opos >= hi - lo:
            continue
        if case in NONFINITE:
            own = int(owners[lo]) if owners is not None else 0
            rank = own if (where == "owner" or world == 1) else (own + 1) % world
            seg = outs[rank][lo:hi]
            _poison(case, seg, g)
            planted.append(Planted(case, lo, hi, rank))
        else:
            for r in range(world):
                outs[r][lo:hi] = _fill(case, hi - lo, r, dtype, bits, g, opos)
            planted.append(Planted(case if case != "outlier" else f"outlier@{opos}", lo, hi, -1))
    return outs, planted
