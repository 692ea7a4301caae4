"""The compressed reduce-scatter kernel (rs_kernel) on one H100 with W virtual ranks
(C.LocalSraGroup), against the CPU simulator and the independent reference, bit for bit and
NaN-aware; the process-group path at world 1; and, with >= 2 GPUs, the public API and FSDP2.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view and the input itself must be unchanged afterwards."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import CASES
from test_reduce_scatter_cpu import rs_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
BUCKETS = [1, 7, 64, 100, 512, 1024, 8192]
WORLDS = [1, 2, 3, 5, 8, 16]
GUARD = 64
SENTINEL = -7.25
MIN_LANE = 256


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def replicated(shard_layers, world, S):
    return [(c * S + o, n, b, k) for c in range(world) for (o, n, b, k) in shard_layers]


def slot_for(shard_layers, world, S, dtype, skip_incomplete):
    wire = C.build_plan(replicated(shard_layers, world, S), world=world, lanes=lanes_for(world, dtype),
                        dtype=DT_CODE[dtype], skip_incomplete=skip_incomplete, min_lane_elems=MIN_LANE)["max_chunk_wire"]
    return (wire + 255) // 256 * 256 + 256


def make_group(world, dtype, slot):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, MIN_LANE)


def guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def assert_guards(buf, offset, n, what):
    b = buf.cpu()
    assert_same(b[:offset], torch.full((offset,), SENTINEL, dtype=b.dtype), f"{what}: before the view")
    assert_same(b[offset + n:], torch.full((GUARD,), SENTINEL, dtype=b.dtype), f"{what}: after the view")


def run_rs(g, ins, shard_layers, *, average=False, skip_incomplete=False, stochastic=False, offset=1,
           alias=False, seed=5, seq=2):
    """Reduce-scatter CPU inputs on the group; returns the outputs on the CPU. Checks the guard
    bands, that the input is unchanged (but for chunk r when the output aliases it) and the status."""
    W, dtype = len(ins), ins[0].dtype
    S = ins[0].numel() // W
    ibufs = [guarded(x, offset) for x in ins]
    if alias:
        outs = [v[r * S:(r + 1) * S] for r, (_, v) in enumerate(ibufs)]
        obufs = None
    else:
        obufs = [guarded(torch.full((S,), SENTINEL, dtype=dtype), (offset + 2) % 6 + 1) for _ in range(W)]
        outs = [v for _, v in obufs]
    g.reduce_scatter([v for _, v in ibufs], outs, shard_layers, average, skip_incomplete, stochastic, seed, seq)
    torch.cuda.synchronize()
    g.check()
    for r, (buf, view) in enumerate(ibufs):
        assert_guards(buf, offset, W * S, f"rank {r} input")
        keep = torch.ones(W * S, dtype=torch.bool)
        if alias:
            keep[r * S:(r + 1) * S] = False
        assert_same(view.cpu()[keep], ins[r][keep], f"rank {r}: input modified")
    if obufs:
        for r, (buf, _) in enumerate(obufs):
            assert_guards(buf, (offset + 2) % 6 + 1, S, f"rank {r} output")
    return [o.cpu().clone() for o in outs]


def simulate(ins, shard_layers, *, average=False, skip_incomplete=False, stochastic=False, seed=5, seq=2):
    W = len(ins)
    outs = [torch.full((ins[0].numel() // W,), SENTINEL, dtype=ins[0].dtype) for _ in range(W)]
    C.reduce_scatter_simulate(ins, outs, shard_layers, lanes_for(W, ins[0].dtype), average, skip_incomplete,
                              stochastic, seed, seq, MIN_LANE)
    return outs


def _configs():
    i = 0
    for dtype in DTYPES:
        for bits in range(1, 9):
            for bucket in BUCKETS:
                W = WORLDS[i % len(WORLDS)]
                yield pytest.param(W, dtype, bits, bucket, i, id=f"w{W}-{str(dtype)[6:]}-q{bits}-b{bucket}")
                i += 1


@pytest.mark.parametrize("world,dtype,bits,bucket,i", list(_configs()))
def test_kernel_matches_simulator_and_reference_on_edge_inputs(world, dtype, bits, bucket, i):
    nq = min(max(16 * bucket, 2000), 2 * 8192) + bucket // 2
    shard_layers = [(0, 37, 32, 512), (37, nq, bits, bucket), (37 + nq, 301, 32, 512)]
    if i % 2 == 0:  # no common bit width: the generic-width kernel
        shard_layers.append((338 + nq, 700, 5, 64))
    S = shard_layers[-1][0] + shard_layers[-1][1]
    average, skip_incomplete = i % 3 == 1, i % 5 == 2
    ins = rs_inputs(world, S, dtype, 1000 + i, "edge_owner" if i % 2 else "edge_peer", shard_layers, cases=CASES)
    g = make_group(world, dtype, slot_for(shard_layers, world, S, dtype, skip_incomplete))
    got = run_rs(g, ins, shard_layers, average=average, skip_incomplete=skip_incomplete, offset=(1, 3, 5)[i % 3],
                 alias=i % 4 == 3)
    sim = simulate(ins, shard_layers, average=average, skip_incomplete=skip_incomplete)
    ref = O.reduce_scatter_reference(ins, shard_layers, average=average, skip_incomplete=skip_incomplete)
    for r in range(world):
        assert_same(got[r], sim[r], f"rank {r} vs simulator")
        assert_same(got[r], ref[r], f"rank {r} vs reference")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_full_slices_of_small_buckets_and_stochastic_rounding(dtype):
    # 8/16/32/256-element buckets inside 512-element full slices, 1024-element slices, then
    # stochastic rounding: the simulator gives the bits, the reference's bound checks the values
    W = 5
    for bucket in (8, 16, 32, 256, 1024):
        shard_layers = [(0, 37, 32, 512), (37, 24 * 1024 + bucket // 2, 4, bucket)]
        S = 37 + 24 * 1024 + bucket // 2
        ins = rs_inputs(W, S, dtype, bucket)
        g = make_group(W, dtype, slot_for(shard_layers, W, S, dtype, False))
        for stochastic in (False, True):
            got = run_rs(g, ins, shard_layers, average=True, stochastic=stochastic, offset=3)
            sim = simulate(ins, shard_layers, average=True, stochastic=stochastic)
            for r in range(W):
                assert_same(got[r], sim[r], f"bucket {bucket} stochastic {stochastic} rank {r}")
            if stochastic:
                for r, (exact, bound) in enumerate(O.reduce_scatter_exact_and_bound(ins, shard_layers, average=True,
                                                                                     stochastic=True)):
                    v = got[r].double().numpy()
                    assert (np.abs(v - exact) <= bound).all(), f"rank {r} outside the one-round bound"


def test_many_windows_equal_one_window():
    W, dtype = 3, torch.bfloat16
    shard_layers = [(0, 5000, 3, 100), (5000, 20_000, 2, 10_000), (25_000, 999, 32, 512), (25_999, 9000, 8, 512)]
    S = 34_999
    ins = rs_inputs(W, S, dtype, 9)
    for skip_incomplete in (False, True):
        big = run_rs(make_group(W, dtype, slot_for(shard_layers, W, S, dtype, skip_incomplete)), ins, shard_layers,
                     skip_incomplete=skip_incomplete, stochastic=True)
        assert len(C.reduce_scatter_windows(shard_layers, W, lanes_for(W, dtype), DT_CODE[dtype], skip_incomplete,
                                            MIN_LANE, 8192)) > 4
        small = run_rs(make_group(W, dtype, 8192), ins, shard_layers, skip_incomplete=skip_incomplete,
                       stochastic=True, offset=5)
        sim = simulate(ins, shard_layers, skip_incomplete=skip_incomplete, stochastic=True)
        for r in range(W):
            assert_same(small[r], big[r], f"rank {r}: several windows vs one")
            assert_same(small[r], sim[r], f"rank {r} vs simulator")


def test_interleaved_calls_on_one_group_match_the_simulators():
    # reduce-scatter, allreduce and one-shot calls share the heap, its slots, flags and epochs
    W, dtype = 4, torch.float32
    rs_layers = [(0, 3000, 4, 512), (3000, 101, 32, 512)]
    S = 3101
    ar_layers = [(0, 20_000, 3, 64), (20_000, 500, 32, 512)]
    slot = max(slot_for(rs_layers, W, S, dtype, False), 64 << 10)
    g = make_group(W, dtype, slot)
    for step in range(6):
        kind = ("rs", "ar", "os", "rs", "rs", "ar")[step]
        g2 = torch.Generator().manual_seed(step)
        if kind == "rs":
            ins = [torch.randn(W * S, generator=g2) * (r + 1) for r in range(W)]
            got = run_rs(g, ins, rs_layers, average=step % 2 == 0, seq=step)
            sim = simulate(ins, rs_layers, average=step % 2 == 0, seq=step)
        else:
            ins = [torch.randn(20_500, generator=g2) * (r + 1) for r in range(W)]
            views = [x.to(dev()) for x in ins]
            (g.allreduce_oneshot if kind == "os" else g.allreduce)(views, ar_layers, False, False, False, 5, step)
            torch.cuda.synchronize()
            g.check()
            got = [v.cpu() for v in views]
            sim = [t.clone() for t in ins]
            fn = C.oneshot_simulate if kind == "os" else C.sra_simulate
            fn(sim, ar_layers, lanes_for(W, dtype), False, False, False, 5, step, MIN_LANE)
        for r in range(W):
            assert_same(got[r], sim[r], f"call {step} ({kind}) rank {r}")


def test_fp32_allreduce_is_the_requantized_reduce_scatter():
    W, dtype = 4, torch.float32
    shard_layers = [(0, 700, 32, 512), (700, 9000, 4, 256), (9700, 300, 6, 100)]
    S = 10_000
    ins = rs_inputs(W, S, dtype, 21)
    layers = replicated(shard_layers, W, S)
    g = make_group(W, dtype, max(slot_for(shard_layers, W, S, dtype, False), 64 << 10))
    rs = run_rs(g, ins, shard_layers)
    views = [x.to(dev()) for x in ins]
    g.allreduce(views, layers, False, False, False, 0, 0)  # chunk c of the allreduce is shard c
    torch.cuda.synchronize()
    g.check()
    expect = O.quantize_dequantize_layers(torch.cat(rs), layers)
    for r in range(W):
        assert_same(views[r].cpu(), expect, f"rank {r}")


def test_bad_arguments_are_rejected():
    g = make_group(2, torch.float32, 1 << 20)
    x = [torch.randn(2000, device=dev()) for _ in range(2)]
    with pytest.raises(ValueError, match="overlaps"):
        g.reduce_scatter(x, [x[0][500:1500], x[1][500:1500]], [(0, 1000, 4, 512)])
    with pytest.raises(ValueError, match="tile"):
        g.reduce_scatter(x, [torch.empty(1000, device=dev()) for _ in range(2)], [(0, 900, 4, 512)])


# ---- process group, world 1 --------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        be = cgx.get_backend()
        x = torch.randn(100_003, device="cuda")
        for dtype in DTYPES:
            xi = x.to(dtype)
            out = torch.full_like(xi, SENTINEL)
            cgx.reduce_scatter_tensor(out, xi, bits=4, average=dtype == torch.float16)
            assert_same(out, xi, f"{dtype}: world 1 output")
        y = x.clone()
        cgx.reduce_scatter_tensor(y, y, bits=2)  # the output is the rank's own chunk of the input
        assert_same(y, x)
        w = cgx.reduce_scatter_tensor(out := torch.empty_like(x), x, async_op=True, stochastic=True, seed=3)
        w.wait()
        assert_same(out, x)
        before = list(be.stats())
        cgx.reduce_scatter_tensor(torch.empty_like(x), x)
        assert be.stats()[0] == before[0] + 1 and be.stats()[1] > before[1]
        # the plain collective keeps going to the delegate: the counters do not move
        before = list(be.stats())
        z = torch.empty_like(x)
        dist.reduce_scatter_tensor(z, x)
        torch.cuda.synchronize()
        assert torch.equal(z, x) and list(be.stats()) == before
        with pytest.raises(RuntimeError, match="CUDA"):
            cgx.reduce_scatter_tensor(torch.empty(10), torch.empty(10))
        with pytest.raises(RuntimeError, match="float32"):
            cgx.reduce_scatter_tensor(torch.empty(10, device="cuda", dtype=torch.int32),
                                      torch.empty(10, device="cuda", dtype=torch.int32))
        with pytest.raises(RuntimeError, match="expected world size"):
            cgx.reduce_scatter_tensor(torch.empty(10, device="cuda"), torch.empty(11, device="cuda"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_process_group_world1():
    spawn(_pg_world1, 1)


def _refused_after_abort(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    be = cgx.get_backend()
    x = torch.randn(100_003, device="cuda")
    dist.all_reduce(x)  # the heap is up and every path has run once
    cgx.reduce_scatter_tensor(torch.empty_like(x), x)
    cgx.all_gather_into_tensor(torch.empty_like(x), x)
    torch.cuda.synchronize()
    be.abort()
    assert "aborted" in be.failure()
    before = list(be.stats())
    calls = {"all_reduce": lambda: dist.all_reduce(x),
             "reduce_scatter_tensor": lambda: cgx.reduce_scatter_tensor(torch.empty_like(x), x),
             "all_gather_into_tensor": lambda: cgx.all_gather_into_tensor(torch.empty_like(x), x)}
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="aborted"):
            call()
        assert list(be.stats()) == before, f"{name} launched after the abort"
    os._exit(0)


def test_every_collective_is_refused_after_abort():
    # the allreduce, the reduce-scatter and the all-gather share the refusal of a failed group
    spawn(_refused_after_abort, 1)


# ---- several GPUs ----------------------------------------------------------------------------
def _inputs_of_all_ranks(world, S, dtype):
    g = torch.Generator().manual_seed(world)
    return [(torch.randn(world * S, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def _pg_bitwise(rank, world):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            for bits, bucket, average in ((2, 512, False), (4, 100, True), (8, 1024, False)):
                S = 70_001
                ins = _inputs_of_all_ranks(world, S, dtype)
                out = torch.empty(S, dtype=dtype, device="cuda")
                cgx.reduce_scatter_tensor(out, ins[rank].cuda(), bits=bits, bucket_size=bucket, average=average)
                ref = O.reduce_scatter_reference(ins, [(0, S, bits, bucket)], average=average)[rank]
                assert_same(out.cpu(), ref, f"{dtype} bits {bits}")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_reduce_scatter_tensor_matches_reference(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_bitwise, world, timeout=600)


def _fsdp_mlp(rank, world, steps):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        losses = {}
        for kind in ("nccl", "cgx"):
            torch.manual_seed(0)
            model = torch.nn.Sequential(*[torch.nn.Sequential(torch.nn.Linear(512, 512), torch.nn.GELU())
                                          for _ in range(4)], torch.nn.Linear(512, 10)).cuda()
            for m in model[:4]:
                fully_shard(m)
            fully_shard(model)
            if kind == "cgx":
                cgx.set_cgx_reduce_scatter(model, bits=8)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            g = torch.Generator(device="cuda").manual_seed(rank)
            before = cgx.get_backend().stats()[1]
            out = []
            for _ in range(steps):
                x = torch.randn(64, 512, device="cuda", generator=g)
                y = (x[:, :10] > 0).float().argmax(1)
                loss = torch.nn.functional.cross_entropy(model(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad()
                out.append(loss.item())
            launched = cgx.get_backend().stats()[1] - before
            assert (launched > 0) == (kind == "cgx"), f"{kind}: {launched} compressed reduce-scatter launches"
            losses[kind] = np.array(out)
        # 8-bit gradients: the loss curve stays within 2% of the uncompressed one
        assert np.all(np.abs(losses["cgx"] - losses["nccl"]) <= 0.02 * losses["nccl"]), losses
        assert losses["cgx"][-1] < losses["cgx"][0]
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_fsdp2_mlp_tracks_nccl():
    spawn(_fsdp_mlp, 2, args=(20,), timeout=600)
