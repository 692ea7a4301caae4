"""The compressed all-gather kernel (ag_kernel) on one H100 with W virtual ranks (C.LocalSraGroup),
against the CPU simulator and the independent reference, bit for bit and NaN-aware; its calls
interleaved with the other kernels on one heap; the process-group path and the FSDP2 comm at
world 1; and, with >= 2 GPUs, the public API and FSDP2.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view and a separate input must be unchanged afterwards."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import CASES
from test_all_gather_cpu import ag_inputs
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


def slot_for(shard_layers, world, S, dtype):
    wire = C.build_plan(replicated(shard_layers, world, S), world=world, lanes=lanes_for(world, dtype),
                        dtype=DT_CODE[dtype], skip_incomplete=False, min_lane_elems=MIN_LANE)["max_chunk_wire"]
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


def run_ag(g, ins, shard_layers, *, stochastic=False, offset=1, in_place=False, seed=5, seq=2):
    """All-gather CPU shards on the group; returns the outputs on the CPU. Checks the guard bands,
    that a separate input is unchanged, and the status. in_place: the input is chunk r of the output."""
    W, dtype = len(ins), ins[0].dtype
    S = ins[0].numel()
    oofs = (offset + 2) % 6 + 1
    obufs = [guarded(torch.full((W * S,), SENTINEL, dtype=dtype), oofs) for _ in range(W)]
    outs = [v for _, v in obufs]
    if in_place:
        for r, x in enumerate(ins):
            outs[r][r * S:(r + 1) * S].copy_(x)
        views, ibufs = [o[r * S:(r + 1) * S] for r, o in enumerate(outs)], None
    else:
        ibufs = [guarded(x, offset) for x in ins]
        views = [v for _, v in ibufs]
    g.all_gather(views, outs, shard_layers, stochastic, seed, seq)
    torch.cuda.synchronize()
    g.check()
    for r, (buf, _) in enumerate(obufs):
        assert_guards(buf, oofs, W * S, f"rank {r} output")
    if ibufs:
        for r, (buf, view) in enumerate(ibufs):
            assert_guards(buf, offset, S, f"rank {r} input")
            assert_same(view.cpu(), ins[r], f"rank {r}: input modified")
    return [o.cpu().clone() for o in outs]


def simulate(ins, shard_layers, *, stochastic=False, seed=5, seq=2):
    W = len(ins)
    outs = [torch.full((W * ins[0].numel(),), SENTINEL, dtype=ins[0].dtype) for _ in range(W)]
    C.all_gather_simulate(ins, outs, shard_layers, stochastic, seed, seq)
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
    ins = ag_inputs(world, S, dtype, 1000 + i, "edge_owner" if i % 2 else "edge_peer", shard_layers, cases=CASES)
    g = make_group(world, dtype, slot_for(shard_layers, world, S, dtype))
    got = run_ag(g, ins, shard_layers, offset=(1, 3, 5)[i % 3], in_place=i % 4 == 3)
    sim = simulate(ins, shard_layers)
    ref = O.all_gather_reference(ins, shard_layers)
    for r in range(world):
        assert_same(got[r], sim[r], f"rank {r} vs simulator")
        assert_same(got[r], ref, f"rank {r} vs reference")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_full_slices_of_small_buckets_and_stochastic_rounding(dtype):
    # 8/16/32/256-element buckets inside 512-element full slices, 1024-element slices, then
    # stochastic rounding: the simulator gives the bits, the reference's bound checks the values
    W = 5
    for bucket in (8, 16, 32, 256, 1024):
        shard_layers = [(0, 37, 32, 512), (37, 24 * 1024 + bucket // 2, 4, bucket)]
        S = 37 + 24 * 1024 + bucket // 2
        ins = ag_inputs(W, S, dtype, bucket)
        g = make_group(W, dtype, slot_for(shard_layers, W, S, dtype))
        for stochastic in (False, True):
            got = run_ag(g, ins, shard_layers, stochastic=stochastic, offset=3, in_place=stochastic)
            sim = simulate(ins, shard_layers, stochastic=stochastic)
            for r in range(W):
                assert_same(got[r], sim[r], f"bucket {bucket} stochastic {stochastic} rank {r}")
            if stochastic:
                for q, x in enumerate(ins):
                    exact, bound = O.exact_sum_and_bound([x], shard_layers, stochastic=True, oneshot=True)
                    v = got[0][q * S:(q + 1) * S].double().numpy()
                    assert (np.abs(v - exact) <= bound).all(), f"shard {q} outside the one-round bound"


def test_many_windows_equal_one_window():
    W, dtype = 3, torch.bfloat16
    shard_layers = [(0, 5000, 3, 100), (5000, 20_000, 2, 10_000), (25_000, 999, 32, 512), (25_999, 9000, 8, 512)]
    S = 34_999
    ins = ag_inputs(W, S, dtype, 9)
    big = run_ag(make_group(W, dtype, slot_for(shard_layers, W, S, dtype)), ins, shard_layers, stochastic=True)
    assert len(C.reduce_scatter_windows(shard_layers, W, lanes_for(W, dtype), DT_CODE[dtype], False, MIN_LANE,
                                        8192)) > 4
    small = run_ag(make_group(W, dtype, 8192), ins, shard_layers, stochastic=True, offset=5, in_place=True)
    sim = simulate(ins, shard_layers, stochastic=True)
    for r in range(W):
        assert_same(small[r], big[r], f"rank {r}: several windows vs one")
        assert_same(small[r], sim[r], f"rank {r} vs simulator")


def test_interleaved_calls_on_one_group_match_the_simulators():
    # all-gather, reduce-scatter, allreduce and one-shot calls share the heap, its slots, flags and
    # epochs; one fixed sequence, run once
    W, dtype = 4, torch.float32
    shard_layers = [(0, 3000, 4, 512), (3000, 101, 32, 512)]
    S = 3101
    ar_layers = [(0, 20_000, 3, 64), (20_000, 500, 32, 512)]
    g = make_group(W, dtype, max(slot_for(shard_layers, W, S, dtype), 64 << 10))
    for step, kind in enumerate(("ag", "rs", "ag", "ar", "ag", "os", "ag", "ag", "rs", "ar")):
        g2 = torch.Generator().manual_seed(step)
        if kind == "ag":
            ins = [torch.randn(S, generator=g2) * (r + 1) for r in range(W)]
            got = run_ag(g, ins, shard_layers, stochastic=step % 2 == 0, seq=step, in_place=step == 4)
            sim = simulate(ins, shard_layers, stochastic=step % 2 == 0, seq=step)
        elif kind == "rs":
            ins = [torch.randn(W * S, generator=g2) * (r + 1) for r in range(W)]
            outs = [torch.empty(S, device=dev()) for _ in range(W)]
            g.reduce_scatter([x.to(dev()) for x in ins], outs, shard_layers, True, False, False, 5, step)
            torch.cuda.synchronize()
            g.check()
            got = [o.cpu() for o in outs]
            sim = [torch.empty(S) for _ in range(W)]
            C.reduce_scatter_simulate(ins, sim, shard_layers, lanes_for(W, dtype), True, False, False, 5, step,
                                      MIN_LANE)
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


@pytest.mark.parametrize("average", [False, True])
def test_fp32_allreduce_is_all_gather_of_reduce_scatter(average):
    W, dtype = 4, torch.float32
    shard_layers = [(0, 700, 32, 512), (700, 9000, 4, 256), (9700, 300, 6, 100)]
    S = 10_000
    ins = rs_inputs(W, S, dtype, 21)
    g = make_group(W, dtype, max(slot_for(shard_layers, W, S, dtype), 64 << 10))
    shards = [torch.empty(S, device=dev()) for _ in range(W)]
    g.reduce_scatter([x.to(dev()) for x in ins], shards, shard_layers, average, False, False, 0, 0)
    gathered = [torch.empty(W * S, device=dev()) for _ in range(W)]
    g.all_gather(shards, gathered, shard_layers, False, 0, 0)
    views = [x.to(dev()) for x in ins]
    g.allreduce(views, replicated(shard_layers, W, S), average, False, False, 0, 0)  # chunk c is shard c
    torch.cuda.synchronize()
    g.check()
    for r in range(W):
        assert_same(gathered[r].cpu(), views[r].cpu(), f"rank {r}")


def test_bad_arguments_are_rejected():
    g = make_group(2, torch.float32, 1 << 20)
    out = [torch.randn(2000, device=dev()) for _ in range(2)]
    with pytest.raises(ValueError, match="overlaps"):
        g.all_gather([o[500:1500] for o in out], out, [(0, 1000, 4, 512)])
    with pytest.raises(ValueError, match="tile"):
        g.all_gather([torch.empty(1000, device=dev()) for _ in range(2)], out, [(0, 900, 4, 512)])


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
            cgx.all_gather_into_tensor(out, xi, bits=4)
            assert_same(out, O.quantize_dequantize_layers(xi.cpu(), [(0, xi.numel(), 4, 512)]), f"{dtype}")
            assert_same(xi, x.to(dtype), f"{dtype}: input modified")
        table = [(0, 50_000, 3, 100), (50_000, 3, 32, 512), (50_003, 50_000, 8, 1024)]
        expect = O.quantize_dequantize_layers(x.cpu(), table)
        y = x.clone()
        cgx.all_gather_into_tensor(y, y, layers=table)  # the input is the rank's own chunk of the output
        assert_same(y, expect)
        w = cgx.all_gather_into_tensor(out := torch.empty_like(x), x, async_op=True, layers=table)
        w.wait()
        assert_same(out, expect)
        before = list(be.stats())
        cgx.all_gather_into_tensor(torch.empty_like(x), x)
        assert be.stats()[0] == before[0] + 1 and be.stats()[1] > before[1]
        # the plain collective keeps going to the delegate: the counters do not move
        before = list(be.stats())
        z = torch.empty_like(x)
        dist.all_gather_into_tensor(z, x)
        torch.cuda.synchronize()
        assert torch.equal(z, x) and list(be.stats()) == before
        with pytest.raises(RuntimeError, match="CUDA"):
            cgx.all_gather_into_tensor(torch.empty(10), torch.empty(10))
        with pytest.raises(RuntimeError, match="float32"):
            cgx.all_gather_into_tensor(torch.empty(10, device="cuda", dtype=torch.int32),
                                       torch.empty(10, device="cuda", dtype=torch.int32))
        with pytest.raises(RuntimeError, match="expected world size"):
            cgx.all_gather_into_tensor(torch.empty(11, device="cuda"), torch.empty(10, device="cuda"))
        buf = torch.zeros(300, device="cuda")
        with pytest.raises((ValueError, RuntimeError), match="overlaps"):
            cgx.all_gather_into_tensor(buf[:200], buf[100:300])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_process_group_world1():
    spawn(_pg_world1, 1)


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(512, 256), torch.nn.LayerNorm(256), torch.nn.GELU(),
                               torch.nn.Linear(256, 10))


def _fsdp_comm_world1(rank, world):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        model = _mlp().cuda()
        fully_shard(model)
        (comm,) = cgx.set_cgx_all_gather(model, bits=8, bucket_size=512)
        fsdp_params = model._get_fsdp_state()._fsdp_param_group.fsdp_params
        # the private FSDP2 attributes the table is built from
        assert [tuple(p._orig_size) for p in fsdp_params] == [(256, 512), (256,), (256,), (256,), (10, 256), (10,)]
        assert [p.padded_sharded_param_size.numel() for p in fsdp_params] == [256 * 512, 256, 256, 256, 2560, 10]
        assert comm.layers == cgx.fsdp_shard_table(
            [(p._orig_size, p.padded_sharded_param_size.numel()) for p in fsdp_params], bits=8, bucket_size=512)
        assert [l[2] for l in comm.layers] == [8, 32, 32, 32, 8, 32]
        # FSDP2 skips the comm at world 1, so it is called directly on the all-gather buffer FSDP builds
        flat = torch.cat([fp._sharded_param_data.detach().reshape(-1) for fp in fsdp_params])
        assert flat.numel() == comm.numel
        out = comm.allocate((flat.numel(),), dtype=flat.dtype, device=flat.device)
        out.copy_(flat)
        before = cgx.get_backend().stats()[1]
        comm(output_tensor=out, input_tensor=out[:flat.numel()], group=dist.group.WORLD, async_op=False)
        assert cgx.get_backend().stats()[1] > before
        assert_same(out, O.quantize_dequantize_layers(flat.cpu(), comm.layers))
        with pytest.raises(RuntimeError, match="module"):
            comm(output_tensor=out[:-1], input_tensor=out[:-1], group=dist.group.WORLD)
        # a uint8 buffer (mixed-dtype inputs) goes to the delegate unchanged
        b = torch.arange(100, dtype=torch.uint8, device="cuda")
        ob = torch.empty_like(b)
        comm(output_tensor=ob, input_tensor=b, group=dist.group.WORLD)
        torch.cuda.synchronize()
        assert torch.equal(ob, b)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_fsdp_all_gather_comm_world1():
    spawn(_fsdp_comm_world1, 1)


# ---- several GPUs ----------------------------------------------------------------------------
def _pg_bitwise(rank, world):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            for bits, bucket in ((2, 512), (4, 100), (8, 1024)):
                S = 70_001
                g = torch.Generator().manual_seed(world)
                ins = [(torch.randn(S, generator=g) * (r + 1)).to(dtype) for r in range(world)]
                out = torch.empty(world * S, dtype=dtype, device="cuda")
                cgx.all_gather_into_tensor(out, ins[rank].cuda(), bits=bits, bucket_size=bucket)
                ref = O.all_gather_reference(ins, [(0, S, bits, bucket)])
                assert_same(out.cpu(), ref, f"{dtype} bits {bits}")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_all_gather_into_tensor_matches_reference(world):
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
            model = torch.nn.Sequential(*[_mlp_block() for _ in range(3)], torch.nn.Linear(512, 10)).cuda()
            for m in model[:3]:
                fully_shard(m)
            fully_shard(model)
            if kind == "cgx":
                cgx.set_cgx_all_gather(model, bits=8)
                cgx.set_cgx_reduce_scatter(model, bits=8)
            opt = torch.optim.SGD(model.parameters(), lr=0.05)
            g = torch.Generator(device="cuda").manual_seed(rank)
            out = []
            for _ in range(steps):
                x = torch.randn(64, 512, device="cuda", generator=g)
                y = (x[:, :10] > 0).float().argmax(1)
                loss = torch.nn.functional.cross_entropy(model(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad()
                out.append(loss.item())
            losses[kind] = np.array(out)
            if kind == "cgx":
                block = model[0]
                sharded = [p.to_local().detach().clone() for p in block.parameters()]
                group = block._get_fsdp_state()._fsdp_param_group
                comm, fsdp_params = group._all_gather_comm, group.fsdp_params
                S = sum(l[1] for l in comm.layers)
                # what FSDP all-gathers: every parameter's padded shard, in all-gather order
                local = torch.cat([fp._sharded_param_data.detach().reshape(-1) for fp in fsdp_params])
                assert local.numel() == S
                block.unshard()
                full = torch.cat([p.detach().reshape(-1) for p in block.parameters()])
                # bit-identical on every rank, and the reference of every rank's padded shard
                gathered = [torch.empty_like(full) for _ in range(world)]
                dist.all_gather(gathered, full)
                for q in range(1, world):
                    assert_same(gathered[q], gathered[0], f"rank {q} unsharded parameters")
                shards = [torch.empty(S, device="cuda") for _ in range(world)]
                dist.all_gather(shards, local.contiguous())
                ref = O.all_gather_reference([s.cpu() for s in shards], comm.layers)
                offs, o = [], 0
                for p in fsdp_params:
                    offs.append(o)
                    o += p.padded_sharded_param_size.numel()
                for p, fp, off in zip(block.parameters(), fsdp_params, offs):
                    n = fp.padded_sharded_param_size.numel()
                    want = torch.cat([ref[q * S + off:q * S + off + n] for q in range(world)])[:p.numel()]
                    assert_same(p.detach().reshape(-1).cpu(), want, f"parameter {fp._param_fqn}")
                block.reshard()
                for a, p in zip(sharded, block.parameters()):
                    assert_same(p.to_local(), a, "the sharded parameter was changed by the gather")
        # 8-bit weights and gradients: the loss curve stays within 3% of the uncompressed one
        assert np.all(np.abs(losses["cgx"] - losses["nccl"]) <= 0.03 * losses["nccl"]), losses
        assert losses["cgx"][-1] < losses["cgx"][0]
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _mlp_block():
    return torch.nn.Sequential(torch.nn.Linear(512, 512), torch.nn.LayerNorm(512), torch.nn.GELU())


@pytest.mark.multigpu
def test_fsdp2_mlp_with_layernorm_tracks_nccl():
    spawn(_fsdp_mlp, 2, args=(20,), timeout=600)
