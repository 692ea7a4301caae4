"""Fixed cases of the generic reducers (SRA / Ring / all-to-all / compressed broadcast) run by
``C.LocalReducerGroup``, shared by the host tier (test_reducers_local_cpu.py) and the device tier
(test_reducers_local_gpu.py): layer tables, inputs (random or the hostile ones of _edge_inputs) and
the independent reference of each operation (torch_cgx_b200/ops/oracle.py)."""
from __future__ import annotations

from itertools import product

import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _edge_inputs import edge_inputs

C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
WORLDS = [1, 2, 3, 4, 5, 8, 16]
BITS = [1, 2, 3, 4, 5, 6, 7, 8, 32]
BUCKETS = [1, 7, 8, 100, 512, 1024, 8192, 10_000]  # 10000 is clamped to 8192
# allreduce with each reducer, and the compressed broadcast from the first and from the last rank
OPS = ["SRA", "RING", "ALLTOALL", "BCAST_FIRST", "BCAST_LAST"]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def table(n_main: int, bits: int, bucket: int, mixed: bool):
    """(layers, total). Mixed: a raw head of 37 elements (the main layer starts at an odd offset),
    a raw layer of 301 and a 5-bit layer. Plain: one layer between 5 leading and 7 trailing
    elements that belong to no layer."""
    if mixed:
        layers = [(0, 37, 32, 512), (37, n_main, bits, bucket), (37 + n_main, 301, 32, 512),
                  (338 + n_main, 2001, 5, 64)]
        return layers, 338 + n_main + 2001
    return [(5, n_main, bits, bucket)], 5 + n_main + 7


def configs():
    """One case per (world, dtype); bits, bucket size, averaging, skip_incomplete, table shape
    and input source rotate so that every value of each appears."""
    out = []
    for i, (world, dtype) in enumerate(product(WORLDS, DTYPES)):
        bits, bucket = BITS[i % len(BITS)], BUCKETS[i % len(BUCKETS)]
        eff = O.effective_bucket(bucket)
        out.append(dict(world=world, dtype=dtype, bits=bits, bucket=bucket, average=i % 2 == 0,
                        skip_incomplete=i % 3 == 1, mixed=i % 2 == 1, source=("randn", "edge_owner", "edge_peer")[i % 3],
                        n_main=3000 + 2 * eff + eff // 3 + 5 * i, seed=i))
    return out


def config_id(c) -> str:
    return (f"w{c['world']}-{str(c['dtype'])[6:]}-q{c['bits']}-b{c['bucket']}-{'avg' if c['average'] else 'sum'}"
            f"{'-skip' if c['skip_incomplete'] else ''}{'-mixed' if c['mixed'] else ''}-{c['source']}")


def make_case(c):
    """(inputs, layers) of a configuration: CPU tensors, one per rank."""
    W, dtype = c["world"], c["dtype"]
    layers, total = table(c["n_main"], c["bits"], c["bucket"], c["mixed"])
    g = torch.Generator().manual_seed(c["seed"])
    ins = [(torch.randn(total, generator=g) * (r + 1)).to(dtype) for r in range(W)]
    if c["source"] != "randn":
        off, n = (37 if c["mixed"] else 5), c["n_main"]  # the main layer
        owners = O.block_owners(layers, total, W, 1, dtype, c["skip_incomplete"], O.GENERIC_MIN_LANE_ELEMS)
        owners = owners[off:off + n]
        owners[owners < 0] = 0
        xs, _ = edge_inputs(dtype, n, O.effective_bucket(c["bucket"]), 1000 + c["seed"], world=W,
                            bits=min(c["bits"], 8), owners=owners,
                            where="owner" if c["source"] == "edge_owner" else "peer")
        for r in range(W):
            ins[r][off:off + n] = xs[r]
    return ins, layers


def reference(op, ins, layers, *, average=False, skip_incomplete=False):
    kw = dict(skip_incomplete=skip_incomplete)
    if op == "SRA":
        return O.sra_reference(ins, layers, lanes=1, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS, average=average, **kw)
    if op == "RING":
        return O.ring_reference(ins, layers, average=average, **kw)
    if op == "ALLTOALL":
        return O.alltoall_reference(ins, layers, average=average, **kw)
    return O.broadcast_compressed_reference(ins, layers, root=root_of(op, len(ins)), **kw)


def root_of(op, world):
    return 0 if op == "BCAST_FIRST" else world - 1


def group_for(op, world, record=False):
    g = C.LocalReducerGroup(world, op if not op.startswith("BCAST") else "SRA", 20_000)
    g.set_recording(record)
    return g


def run_op(g, op, tensors, layers, *, average=False, skip_incomplete=False, stochastic=False, seed=11, seq=3):
    """Run `op` in place on `tensors` (one per virtual rank) through group `g`."""
    if op.startswith("BCAST"):
        g.broadcast_compressed(tensors, layers, root_of(op, len(tensors)), skip_incomplete, stochastic, seed, seq)
    else:
        g.allreduce(tensors, layers, average, skip_incomplete, stochastic, seed, seq)


def expected_bytes_sent(op, layers, world, dtype, skip_incomplete):
    """Per rank: the bytes each reducer sends, from the plan's chunk_wire_bytes."""
    W = world
    if op.startswith("BCAST"):
        if W == 1:
            return [0]
        p = C.build_plan(layers, world=1, lanes=1, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete,
                         min_lane_elems=O.GENERIC_MIN_LANE_ELEMS)
        root = root_of(op, W)
        return [p["chunk_wire_bytes"][0] * (W - 1) if r == root else 0 for r in range(W)]
    p = C.build_plan(layers, world=W, lanes=1, dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete,
                     min_lane_elems=O.GENERIC_MIN_LANE_ELEMS)
    cw = p["chunk_wire_bytes"]
    if op == "SRA":  # phase 1: every peer's chunk; phase 2: the own reduced chunk to every peer
        return [sum(cw[q] for q in range(W) if q != r) + (W - 1) * cw[r] for r in range(W)]
    if op == "RING":  # reduce-scatter hops send chunk r - s, all-gather hops forward chunk r + 1 - s
        return [sum(cw[(r - s) % W] + cw[(r + 1 - s) % W] for s in range(W - 1)) for r in range(W)]
    row = (p["max_chunk_wire"] + 255) // 256 * 256  # all-to-all: the whole wire image to every peer
    return [(W - 1) * W * row for _ in range(W)]


PLAN_CACHE_BOUND = 256  # plans a generic reducer keeps before it drops its cache (Reducer::kMaxPlans)


def check_many_layouts(world, device, calls=300):
    """More distinct allreduce layouts than a reducer's plan cache holds, through one SRA group on
    `device`: every call equals sra_simulate bit for bit (stochastic rounding, so the RNG streams
    count too), across the drop, and no rank's cache ever holds more than PLAN_CACHE_BOUND plans."""
    from _bitwise import assert_same

    g = C.LocalReducerGroup(world, "SRA", 20_000)
    gen = torch.Generator().manual_seed(world)
    most = 0
    for i in range(calls):
        n = 700 + 3 * i
        layers = [(0, 37, 32, 512), (37, n - 37, 4, 64)]
        ins = [torch.randn(n, generator=gen) * (r + 1) for r in range(world)]
        got = [t.clone().to(device) for t in ins]
        g.allreduce(got, layers, True, False, True, 7, i)
        sim = [t.clone() for t in ins]
        C.sra_simulate(sim, layers, 1, True, False, True, 7, i, O.GENERIC_MIN_LANE_ELEMS)
        for r in range(world):
            assert_same(got[r].cpu(), sim[r], f"call {i} rank {r}")
        held = [g.num_plans(r) for r in range(world)]
        assert max(held) <= PLAN_CACHE_BOUND, f"call {i}: {held} plans cached"
        most = max(most, *held)
    assert most == PLAN_CACHE_BOUND and max(held) < PLAN_CACHE_BOUND, "the plan cache never filled and dropped"
