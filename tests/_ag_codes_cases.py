"""Shared pieces of the FP8 all-gather codes-output tests (CPU and GPU tiers)."""
from __future__ import annotations

from typing import List, Tuple

import torch

from torch_cgx_b200 import _C

FMTS = ("e4m3", "e5m2")
TDT = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
# bucket -> shard size S (a multiple of it)
BUCKET_SHARDS = {64: 3 * 1024, 100: 2500, 128: 5 * 1024, 512: 3 * 1536, 1024: 6 * 1024, 7168: 2 * 7168,
                 8192: 2 * 8192}
WORLDS = (1, 2, 3, 8, 16)


def shards(world: int, S: int, dtype: torch.dtype, seed: int, device="cpu") -> List[torch.Tensor]:
    """one shard per rank, a different scale in every bucket-sized stretch"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(world):
        x = torch.randn(S, generator=g) * torch.exp(torch.randn(S, generator=g) * 2)
        out.append(x.to(dtype).to(device))
    return out


def codes_buffers(world: int, S: int, bucket: int, fmt: str, device="cpu") -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """per rank: codes (the format's float8, filled with 0x55) and scales (NaN)"""
    codes = [torch.full((world * S,), 0x55, dtype=torch.uint8, device=device).view(TDT[fmt]) for _ in range(world)]
    scales = [torch.full((world * S // bucket,), float("nan"), device=device) for _ in range(world)]
    return codes, scales


def table(S: int, bucket: int):
    return [(0, S, 8, bucket)]


def simulate_codes(xs, fmt, bucket):
    W, S = len(xs), xs[0].numel()
    codes, scales = codes_buffers(W, S, bucket, fmt)
    _C.all_gather_simulate(xs, codes, table(S, bucket), bits=fmt, output_scales=scales)
    return codes, scales


def decode(codes: torch.Tensor, scales: torch.Tensor, bucket: int, dtype: torch.dtype) -> torch.Tensor:
    """T(codes.float() * scale), one fp32 multiply and then the dtype's rounding"""
    return (codes.reshape(-1).float() * scales.reshape(-1).repeat_interleave(bucket)).to(dtype)


def assert_codes(got, ref, what=""):
    """FP8 codes byte for byte, except that any NaN code equals any other"""
    got, ref = got.detach().cpu().reshape(-1), ref.detach().cpu().reshape(-1)
    assert got.dtype == ref.dtype and got.numel() == ref.numel(), f"{what}: {got.dtype}/{got.numel()} vs {ref.dtype}/{ref.numel()}"
    gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
    assert torch.equal(gn, rn), f"{what}: NaN codes differ at {int((gn != rn).nonzero()[0])}"
    diff = (got.view(torch.uint8) != ref.view(torch.uint8)) & ~gn
    assert not diff.any(), f"{what}: {int(diff.sum())} codes differ, first at {int(diff.nonzero()[0])}"
