"""Shared pieces of the allreduce engine tests (test_engine_local_cpu.py, test_engine_local_gpu.py):
W real AllreduceEngines in one process (C.LocalEngineGroup), checked bit for bit and stage by stage
against ``oracle.engine_reference``."""
from __future__ import annotations

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same

C = cgx._C
TIMEOUT_MS = 20_000  # a wrong schedule shows up as a status error, not a long wait


@pytest.fixture(autouse=True)
def clean_environment(monkeypatch):
    """No compression, stochastic rounding or registered layers leak in from the caller or other tests."""
    for k in ("CGX_COMPRESSION_QUANTIZATION_BITS", "CGX_COMPRESSION_BUCKET_SIZE", "CGX_STOCHASTIC_ROUNDING",
              "CGX_SEED", "CGX_COMPRESSION_SKIP_INCOMPLETE_BUCKETS", "CGX_COMPRESSION_MINIMAL_SIZE",
              "CGX_COMPRESSION_FAKE_RATIO", "CGX_DEBUG_DUMMY_COMPRESSION"):
        monkeypatch.delenv(k, raising=False)
    C.reset_layers()
    yield
    C.reset_layers()


def set_stochastic(monkeypatch, on, seed=0):
    monkeypatch.setenv("CGX_STOCHASTIC_ROUNDING", "1" if on else "0")
    monkeypatch.setenv("CGX_SEED", str(seed))


def mixed_table(sizes_bits):
    """Consecutive layers from (numel, bits, bucket) triples."""
    out, off = [], 0
    for n, bits, bucket in sizes_bits:
        out.append((off, n, bits, bucket))
        off += n
    return out, off


def inputs_for(world, total, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(total, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def comparable(stage, with_layers=True):
    s = dict(stage)
    s["layers"] = [tuple(int(v) for v in l) for l in s["layers"]]
    if not with_layers:
        s.pop("layers")
    return s


def assert_log(group, expected, world, *, fast=False):
    """Every rank's stage log equals the reference's; a fast-path call logs its fused launches without
    their layer tables."""
    for r in range(world):
        got = [comparable(s, not fast) for s in group.log(r)]
        want = [comparable(s, not fast) for s in expected[r]]
        assert got == want, f"rank {r}: stages differ\n got {got}\nwant {want}"


def assert_results(got, want, what):
    for r, (a, b) in enumerate(zip(got, want)):
        assert_same(a.cpu().reshape(-1), b.reshape(-1), f"{what}: rank {r}")
