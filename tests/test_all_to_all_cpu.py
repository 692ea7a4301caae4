"""Compressed all-to-all on the CPU: the simulator against the independent numpy reference, the
device item helper against build_plan, the windows, the differentiable form's backward, and the
split validation of the public API."""
from __future__ import annotations

import itertools

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200 import _C
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import BITS, BUCKETS, DTYPES, SPLITS, WORLDS, base_elems, counts, inputs, outputs
from _bitwise import assert_same
from _edge_inputs import edge_inputs

_DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _simulate(xs, c, bits, bucket, **kw):
    outs = outputs(c, xs[0].dtype)
    _C.all_to_all_simulate(xs, outs, c, bits=bits, bucket_size=bucket, **kw)
    return outs


def _check(xs, c, bits, bucket, what):
    got = _simulate(xs, c, bits, bucket)
    ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket)
    for r in range(len(xs)):
        assert_same(got[r], ref[r], f"{what} rank {r}")


# every (dtype, bits, bucket) at a world size that cycles through WORLDS, and every split kind
@pytest.mark.parametrize("dtype,bits,bucket", list(itertools.product(DTYPES, BITS, BUCKETS)))
def test_simulator_matches_reference(dtype, bits, bucket):
    i = DTYPES.index(dtype) * 7 + BITS.index(bits) * 3 + BUCKETS.index(bucket)
    W = WORLDS[i % len(WORLDS)]
    base = base_elems(bucket) if W <= 5 else max(300, min(base_elems(bucket), 2000))
    kind = SPLITS[i % len(SPLITS)]
    c = counts(W, kind, base, seed=i)
    _check(inputs(c, dtype, i), c, bits, bucket, f"W={W} {kind}")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind", SPLITS)
def test_simulator_every_world_and_split(world, kind):
    c = counts(world, kind, 700, seed=world)
    _check(inputs(c, torch.bfloat16, world), c, 4, 512, f"W={world} {kind}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bits", [2, 4, 8])
def test_simulator_edge_inputs(dtype, bits):
    W, bucket = 3, 64
    n = 40 * bucket  # equal splits on bucket boundaries: every planted bucket is one chunk bucket
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=bits, world=W, bits=bits)
    assert planted
    _check(xs, [[n] * W for _ in range(W)], bits, bucket, "edge")


def test_stochastic_depends_on_seed_and_seq():
    c = counts(3, "uneven", 2000, seed=1)
    xs = inputs(c, torch.float32, 1)
    a = _simulate(xs, c, 3, 128, stochastic=True, seed=5, seq=1)
    b = _simulate(xs, c, 3, 128, stochastic=True, seed=5, seq=1)
    d = _simulate(xs, c, 3, 128, stochastic=True, seed=5, seq=2)
    for r in range(3):
        assert_same(a[r], b[r])
    assert any(not torch.equal(a[r], d[r]) for r in range(3))


# ---- the device item helper is build_plan's one-layer table ------------------------------------
_SIZES = [1, 7, 8, 100, 511, 512, 513, 1023, 1024, 1025, 4096, 8191, 8192, 8193, 20000, 70001]


@pytest.mark.parametrize("bits,bucket", [(4, 8), (4, 64), (8, 512), (2, 1024), (3, 7), (5, 100), (1, 1),
                                         (8, 2048), (8, 8192), (4, 10000), (32, 512)])
@pytest.mark.parametrize("dtype", [0, 1])
def test_item_helper_equals_build_plan(bits, bucket, dtype):
    for n in _SIZES:
        plan = _C.build_plan([(0, n, bits, bucket)], 1, 1, dtype, False, 1 << 30)
        got = _C.a2a_items(n, bits, bucket, dtype)
        assert torch.equal(got, plan["items"]), (n, bits, bucket)
        # the record bytes of the chunk, which the generic reducer sends from a2a.h alone
        w = _C.a2a_windows(n, bits, bucket, dtype, 1 << 30, 1)
        assert sum(b[2] for lane in w["lanes"] for win in lane for b in win) == plan["chunk_wire_bytes"][0]
        # slice size: 1024-element slices exactly for 1024-element buckets
        assert plan["slice_elems"] == (1024 if bits < 32 and bucket == 1024 else 512)


@pytest.mark.parametrize("bits,bucket", [(4, 512), (8, 1024), (3, 7), (2, 10000), (32, 512), (1, 1)])
@pytest.mark.parametrize("slot_bytes,lanes", [(1 << 16, 4), (1 << 20, 16), (300000, 3)])
def test_windows_tile_the_chunk(bits, bucket, slot_bytes, lanes):
    n = 123457
    w = _C.a2a_windows(n, bits, bucket, 2, slot_bytes, lanes)
    eff = min(bucket, 8192) if bits < 32 else 512
    if w["window_blocks"] == 0:
        assert w["block_wire"] > w["lane_slot"]
        return
    seen = []
    for lane in w["lanes"]:
        for win in lane:
            assert 0 < len(win) <= w["window_blocks"]
            assert sum(b[2] for b in win) <= w["lane_slot"]
            for off, m, _ in win:
                assert off % eff == 0
                seen.append((off, m))
    seen.sort()
    pos = 0
    for off, m in seen:
        assert off == pos
        pos += m
    assert pos == n


# ---- the differentiable form, with the collective substituted -----------------------------------
def test_backward_swaps_splits_at_grad_bits(monkeypatch):
    from torch_cgx_b200.parallel import functional as F

    calls = []

    def fake(output, input, output_split_sizes=None, input_split_sizes=None, bits=8, bucket_size=512, group=None,
             async_op=False, stochastic=False, seed=None):
        calls.append((list(output_split_sizes or []), list(input_split_sizes or []), bits, bucket_size))
        output.copy_(input[: output.shape[0]] if output.shape[0] <= input.shape[0]
                     else torch.cat([input, input.new_zeros((output.shape[0] - input.shape[0],) + input.shape[1:])]))

    monkeypatch.setattr(F, "all_to_all_single", fake)
    monkeypatch.setattr(F.dist, "get_world_size", lambda group=None: 2)
    x = torch.randn(5, 3, requires_grad=True)
    y = cgx.differentiable_all_to_all_single(x, [1, 3], [2, 3], bits=4, grad_bits=32, bucket_size=64)
    assert y.shape == (4, 3)
    y.sum().backward()
    assert calls[0] == ([1, 3], [2, 3], 4, 64)
    assert calls[1] == ([2, 3], [1, 3], 32, 64)
    assert x.grad.shape == x.shape
    calls.clear()
    y = cgx.differentiable_all_to_all_single(x, [2, 3], [2, 3], bits=2)
    y.sum().backward()
    assert calls[1][2] == 2  # grad_bits=None means bits


# ---- validation ---------------------------------------------------------------------------------
def test_simulator_rejects_bad_counts():
    xs = [torch.zeros(4), torch.zeros(4)]
    with pytest.raises(RuntimeError, match="W x W"):
        _C.all_to_all_simulate(xs, [torch.zeros(4)] * 2, [[2, 2]], bits=4)
    with pytest.raises(RuntimeError, match="negative"):
        _C.all_to_all_simulate(xs, [torch.zeros(4)] * 2, [[5, -1], [2, 2]], bits=4)
    with pytest.raises(RuntimeError, match="row and column"):
        _C.all_to_all_simulate(xs, [torch.zeros(4)] * 2, [[1, 2], [2, 2]], bits=4)


# ---- the generic reducer path on host memory ----------------------------------------------------
@pytest.mark.parametrize("bits,bucket", [(4, 512), (8, 1024), (3, 7), (32, 512)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_reducer_matches_simulator(bits, bucket, dtype):
    W = 3
    c = counts(W, "uneven", 3000, seed=bits)
    xs = inputs(c, dtype, bits)
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    outs = outputs(c, dtype)
    red.all_to_all(xs, outs, c, bits=bits, bucket_size=bucket, stochastic=True, seed=3, seq=9)
    sim = _simulate(xs, c, bits, bucket, stochastic=True, seed=3, seq=9)
    for r in range(W):
        assert_same(outs[r], sim[r], f"rank {r}")


def test_generic_reducer_plan_cache_is_bounded():
    # more distinct chunk sizes than the plan cache holds: results stay exact across the drop
    W, dtype = 2, torch.float32
    red = _C.LocalReducerGroup(W, "SRA", 5000)
    for it in range(140):
        c = [[10 + it, 300 + it], [200 + 2 * it, 5 + it]]
        xs = inputs(c, dtype, it)
        outs = outputs(c, dtype)
        red.all_to_all(xs, outs, c, bits=3, bucket_size=16)
        sim = _simulate(xs, c, 3, 16)
        for r in range(W):
            assert_same(outs[r], sim[r], f"call {it} rank {r}")
            assert red.num_plans(r) <= 256
