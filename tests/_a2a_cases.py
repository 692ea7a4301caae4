"""Split matrices and inputs shared by the all-to-all tests. ``counts[q][r]`` elements go from
rank q to rank r; rank q's input holds row q in destination order."""
from __future__ import annotations

from typing import List

import torch

WORLDS = (1, 2, 3, 5, 8, 16)
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BITS = (1, 2, 3, 4, 5, 8, 32)
BUCKETS = (1, 7, 64, 100, 512, 1024, 8192, 10000)
SPLITS = ("equal", "uneven", "zero_send", "zero_recv", "empty")


def counts(world: int, kind: str, base: int, seed: int) -> List[List[int]]:
    g = torch.Generator().manual_seed(seed)
    if kind == "equal":
        return [[base] * world for _ in range(world)]
    m = torch.randint(0, 2 * base + 1, (world, world), generator=g).tolist()
    if kind == "zero_send":
        m[0] = [0] * world
    elif kind == "zero_recv":
        for q in range(world):
            m[q][world - 1] = 0
    elif kind == "empty":
        m = [[0] * world for _ in range(world)]
    return m


def inputs(c: List[List[int]], dtype: torch.dtype, seed: int) -> List[torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(sum(row), generator=g, dtype=torch.float64) * (q + 1)).to(dtype) for q, row in enumerate(c)]


def outputs(c: List[List[int]], dtype: torch.dtype, device="cpu") -> List[torch.Tensor]:
    W = len(c)
    return [torch.full((sum(c[q][r] for q in range(W)),), float("nan"), dtype=dtype, device=device) for r in range(W)]


def base_elems(bucket: int) -> int:
    """A chunk size with a partial bucket, and above one block for buckets past the clamp."""
    return max(300, bucket + bucket // 3 + 5) if bucket <= 1024 else 9000 + bucket // 7
