"""FP8 wire formats of the compressed reduce-scatter and all-gather (rs_kernel / ag_kernel with CODEC
e4m3 / e5m2) on one H100 with W virtual ranks (C.LocalSraGroup): bitwise equal, NaN-aware, to the
CPU simulator and to the independent reference over dtypes, both formats, 512- and 1024-element
slices, worlds 2-8, mixed tables with raw layers, edge inputs, views at odd element offsets and an
output that is the input's own chunk; many windows against one; FP8, max-min and all-to-all calls
on one heap; a CUDA graph; the generic reducer's device kernels against the fused kernel and their
wire messages against the host backend's; the FP8 reduce-scatter against the FP8 all-to-all; the
process group and the FSDP comms at world 1; and, with >= 2 GPUs, the public API on both transports
and an FSDP2 MLP with an e4m3 all-gather and an e5m2 reduce-scatter.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view must be unchanged afterwards."""
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
FMTS = ("e4m3", "e5m2")
GUARD = 64
SENTINEL = -7.25
MIN_LANE = 256
MIXED = [(0, 37, 32, 512), (37, 30_000, 8, 1024), (30_037, 301, 32, 512), (30_338, 4501, 8, 100),
         (34_839, 9000, 8, 512)]
S_MIXED = 43_839


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def slot_for(table, world, S, dtype):
    rep = [(c * S + o, n, b, k) for c in range(world) for (o, n, b, k) in table]
    wire = C.build_plan(rep, world=world, lanes=lanes_for(world, dtype), dtype=DT_CODE[dtype],
                        skip_incomplete=False, min_lane_elems=MIN_LANE)["max_chunk_wire"]
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


def full_inputs(world, S, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(world * S, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def own(full):
    W = len(full)
    S = full[0].numel() // W
    return [full[r][r * S:(r + 1) * S].clone() for r in range(W)]


def run_rs(g, full, table, fmt, *, average=False, offset=1, in_place=False):
    W, dtype = len(full), full[0].dtype
    S = full[0].numel() // W
    ibufs = [guarded(x, offset) for x in full]
    if in_place:
        outs = [v[r * S:(r + 1) * S] for r, (_, v) in enumerate(ibufs)]
        obufs = None
    else:
        oofs = (offset + 2) % 6 + 1
        obufs = [(guarded(torch.zeros(S, dtype=dtype), oofs), oofs) for _ in range(W)]
        outs = [v for (_, v), _ in obufs]
    g.reduce_scatter([v for _, v in ibufs], outs, table, average, False, False, 5, 2, bits=fmt)
    torch.cuda.synchronize()
    g.check()
    for r, (buf, view) in enumerate(ibufs):
        assert_guards(buf, offset, W * S, f"rank {r} input")
        if not in_place:
            assert_same(view.cpu(), full[r], f"rank {r}: input modified")
    if obufs:
        for r, ((buf, _), oofs) in enumerate(obufs):
            assert_guards(buf, oofs, S, f"rank {r} output")
    return [o.cpu().clone() for o in outs]


def run_ag(g, shards, table, fmt, *, offset=1, in_place=False):
    W, dtype = len(shards), shards[0].dtype
    S = shards[0].numel()
    oofs = (offset + 2) % 6 + 1
    obufs = [guarded(torch.full((W * S,), SENTINEL, dtype=dtype), oofs) for _ in range(W)]
    outs = [v for _, v in obufs]
    if in_place:
        for r, x in enumerate(shards):
            outs[r][r * S:(r + 1) * S].copy_(x)
        views, ibufs = [o[r * S:(r + 1) * S] for r, o in enumerate(outs)], None
    else:
        ibufs = [guarded(x, offset) for x in shards]
        views = [v for _, v in ibufs]
    g.all_gather(views, outs, table, False, 5, 2, bits=fmt)
    torch.cuda.synchronize()
    g.check()
    for r, (buf, _) in enumerate(obufs):
        assert_guards(buf, oofs, W * S, f"rank {r} output")
    if ibufs:
        for r, (buf, view) in enumerate(ibufs):
            assert_guards(buf, offset, S, f"rank {r} input")
            assert_same(view.cpu(), shards[r], f"rank {r}: input modified")
    return [o.cpu().clone() for o in outs]


def sim_rs(full, table, fmt, average=False):
    W = len(full)
    outs = [torch.empty(full[0].numel() // W, dtype=full[0].dtype) for _ in range(W)]
    C.reduce_scatter_simulate(full, outs, table, average=average, bits=fmt)
    return outs


def sim_ag(shards, table, fmt):
    W = len(shards)
    outs = [torch.empty(W * shards[0].numel(), dtype=shards[0].dtype) for _ in range(W)]
    C.all_gather_simulate(shards, outs, table, bits=fmt)
    return outs


def check_rs(got, full, table, fmt, what, average=False):
    sim = sim_rs(full, table, fmt, average)
    ref = O.reduce_scatter_reference(full, table, average=average, fmt=fmt)
    for r in range(len(full)):
        assert_same(got[r], sim[r], f"{what}: rank {r} vs simulator")
        assert_same(got[r], ref[r], f"{what}: rank {r} vs reference")


def check_ag(got, shards, table, fmt, what):
    sim = sim_ag(shards, table, fmt)
    ref = O.all_gather_reference(shards, table, fmt)
    for r in range(len(shards)):
        assert_same(got[r], sim[r], f"{what}: rank {r} vs simulator")
        assert_same(got[r], ref, f"{what}: rank {r} vs reference")


# ---- the fused kernels ----------------------------------------------------------------------------
def _configs():
    i = 0
    for dtype in DTYPES:
        for fmt in FMTS:
            for bucket in (512, 1024, 64, 300):
                W = (2, 3, 5, 8)[i % 4]
                yield pytest.param(W, dtype, fmt, bucket, i, id=f"w{W}-{str(dtype)[6:]}-{fmt}-b{bucket}")
                i += 1


@pytest.mark.parametrize("world,dtype,fmt,bucket,i", list(_configs()))
def test_fused_matches_simulator_and_reference(world, dtype, fmt, bucket, i):
    table = [(0, 37, 32, 512), (37, 24 * 1024 + bucket // 2, 8, bucket), (24 * 1024 + 37 + bucket // 2, 301, 32, 512)]
    S = table[-1][0] + table[-1][1]
    full = full_inputs(world, S, dtype, 100 + i)
    g = make_group(world, dtype, slot_for(table, world, S, dtype))
    offset, in_place = (1, 3, 5)[i % 3], i % 4 == 3
    got = run_rs(g, full, table, fmt, average=i % 2 == 1, offset=offset, in_place=in_place)
    check_rs(got, full, table, fmt, "rs", average=i % 2 == 1)
    got = run_ag(g, own(full), table, fmt, offset=offset, in_place=in_place)
    check_ag(got, own(full), table, fmt, "ag")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_fused_mixed_table(dtype, fmt):
    W = 4
    full = full_inputs(W, S_MIXED, dtype, 7)
    g = make_group(W, dtype, slot_for(MIXED, W, S_MIXED, dtype))
    check_rs(run_rs(g, full, MIXED, fmt, average=True, offset=3), full, MIXED, fmt, "rs mixed", average=True)
    check_ag(run_ag(g, own(full), MIXED, fmt, offset=5), own(full), MIXED, fmt, "ag mixed")


@pytest.mark.parametrize("where", ["owner", "peer"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("bucket", [512, 1024, 100])
def test_fused_edge_inputs(bucket, dtype, fmt, where):
    W = 3
    S = 70 * bucket + 13
    table = [(0, S, 8, bucket)]
    xs, _ = edge_inputs(dtype, S, bucket, 11, world=W, bits=8, owners=[1] * S, where=where)
    g0 = torch.Generator().manual_seed(3)
    full = [torch.cat([(torch.randn(S, generator=g0)).to(dtype) if c != 1 else xs[r] for c in range(W)])
            for r in range(W)]
    g = make_group(W, dtype, slot_for(table, W, S, dtype))
    check_rs(run_rs(g, full, table, fmt), full, table, fmt, f"rs edge {where}")
    check_ag(run_ag(g, [x.clone() for x in xs], table, fmt, in_place=True), xs, table, fmt, f"ag edge {where}")


@pytest.mark.parametrize("fmt", FMTS)
def test_many_windows_equal_one_window(fmt):
    W, dtype = 3, torch.bfloat16
    S = S_MIXED
    full = full_inputs(W, S, dtype, 9)
    assert len(C.reduce_scatter_windows(MIXED, W, lanes_for(W, dtype), DT_CODE[dtype], False, MIN_LANE, 8192)) > 4
    for small, big in ((make_group(W, dtype, 8192), make_group(W, dtype, slot_for(MIXED, W, S, dtype))),):
        a = run_rs(small, full, MIXED, fmt, offset=5)
        b = run_rs(big, full, MIXED, fmt)
        c = run_ag(small, own(full), MIXED, fmt, in_place=True)
        d = run_ag(big, own(full), MIXED, fmt)
        for r in range(W):
            assert_same(a[r], b[r], f"rs rank {r}: several windows vs one")
            assert_same(c[r], d[r], f"ag rank {r}: several windows vs one")
    check_rs(a, full, MIXED, fmt, "rs windows")
    check_ag(c, own(full), MIXED, fmt, "ag windows")


def test_fp8_max_min_and_all_to_all_interleaved_on_one_heap():
    W, dtype, S = 4, torch.float16, 20_000
    table8 = [(0, S, 8, 512)]
    g = make_group(W, dtype, max(slot_for(table8, W, S, dtype), 1 << 20))  # room for the all-to-all's blocks
    for it, bits in enumerate(["e4m3", 8, "e5m2", 4, "e4m3"]):
        full = full_inputs(W, S, dtype, it)
        fmt = bits if isinstance(bits, str) else None
        table = [(0, S, bits if fmt is None else 8, 512)]
        check_rs(run_rs(g, full, table, fmt), full, table, fmt, f"rs call {it}")
        check_ag(run_ag(g, own(full), table, fmt), own(full), table, fmt, f"ag call {it}")
        c = [[3000] * W for _ in range(W)]
        xs = [x[:3000 * W].contiguous() for x in full]
        outs = [torch.empty(3000 * W, dtype=dtype, device=dev()) for _ in range(W)]
        g.all_to_all([x.to(dev()) for x in xs], outs, c, bits="e5m2" if it % 2 else "e4m3", bucket_size=512)
        torch.cuda.synchronize()
        ref = O.all_to_all_reference(xs, c, bits="e5m2" if it % 2 else "e4m3", bucket_size=512)
        for r in range(W):
            assert_same(outs[r].cpu(), ref[r], f"a2a call {it} rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph(fmt):
    W, dtype, S = 4, torch.float32, 30_000
    table = [(0, 37, 32, 512), (37, S - 37, 8, 1024)]
    g = make_group(W, dtype, slot_for(table, W, S, dtype))
    ins = [torch.empty(W * S, device=dev()) for _ in range(W)]
    rs_out = [torch.empty(S, device=dev()) for _ in range(W)]
    ag_out = [torch.empty(W * S, device=dev()) for _ in range(W)]
    shards = [x[r * S:(r + 1) * S] for r, x in enumerate(ins)]

    def step():
        g.reduce_scatter(ins, rs_out, table, True, False, False, 0, 0, bits=fmt)
        g.all_gather(shards, ag_out, table, False, 0, 0, bits=fmt)

    for t, x in zip(ins, full_inputs(W, S, dtype, 0)):
        t.copy_(x)
    step()  # plans are built and uploaded outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        step()
    torch.cuda.synchronize()
    for it in range(3):
        full = full_inputs(W, S, dtype, 10 + it)
        for t, x in zip(ins, full):
            t.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        check_rs([o.cpu() for o in rs_out], full, table, fmt, f"replay {it} rs", average=True)
        check_ag([o.cpu() for o in ag_out], own(full), table, fmt, f"replay {it} ag")


# ---- the generic reducer (NCCL transport's path, and the cross-node stage) -----------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_generic_device_path_equals_fused_and_host(dtype, fmt):
    W = 3
    full = full_inputs(W, S_MIXED, dtype, 21)
    fused_rs = run_rs(make_group(W, dtype, slot_for(MIXED, W, S_MIXED, dtype)), full, MIXED, fmt, average=True)
    fused_ag = run_ag(make_group(W, dtype, slot_for(MIXED, W, S_MIXED, dtype)), own(full), MIXED, fmt)
    got = {}
    for where in ("cpu", "cuda"):
        red = C.LocalReducerGroup(W, "SRA", 5000)
        red.set_recording(True)
        rs = [torch.empty(S_MIXED, dtype=dtype, device=where) for _ in range(W)]
        red.reduce_scatter([x.to(where) for x in full], rs, MIXED, average=True, bits=fmt)
        torch.cuda.synchronize()
        msgs = sorted(((m[1], m[2], m[3]) for m in red.messages()), key=lambda m: m[:2])  # the last call's
        # a fresh group: the records' padding is never written, so it shows the scratch's zeros on both
        # backends instead of what the reduce-scatter left there
        red = C.LocalReducerGroup(W, "SRA", 5000)
        red.set_recording(True)
        ag = [torch.empty(W * S_MIXED, dtype=dtype, device=where) for _ in range(W)]
        red.all_gather([x.to(where) for x in own(full)], ag, MIXED, bits=fmt)
        torch.cuda.synchronize()
        msgs += sorted(((m[1], m[2], m[3]) for m in red.messages()), key=lambda m: m[:2])
        got[where] = ([o.cpu() for o in rs], [o.cpu() for o in ag], msgs)
    for r in range(W):
        assert_same(got["cuda"][0][r], fused_rs[r], f"generic rs vs fused rank {r}")
        assert_same(got["cuda"][1][r], fused_ag[r], f"generic ag vs fused rank {r}")
        assert_same(got["cpu"][0][r], fused_rs[r], f"host rs vs fused rank {r}")
    cpu_m, cuda_m = got["cpu"][2], got["cuda"][2]
    assert len(cpu_m) == len(cuda_m) == 2 * W * (W - 1)
    for i, (a, b) in enumerate(zip(cpu_m, cuda_m)):
        assert a[:2] == b[:2] and torch.equal(a[2], b[2]), f"{'rs' if i < W * (W - 1) else 'ag'} message {a[:2]} differs"


def test_reduce_scatter_is_own_plus_the_all_to_all_decodes():
    """fp32, one layer, prescale 1: the FP8 reduce-scatter equals the owner's value plus the slot-ordered
    sum of what the FP8 all-to-all decodes of the same chunks, bit for bit (two kernels, one codec)"""
    W, S, bucket = 4, 16_384, 512
    table = [(0, S, 8, bucket)]
    full = full_inputs(W, S, torch.float32, 31)
    for fmt in FMTS:
        g = make_group(W, torch.float32, max(slot_for(table, W, S, torch.float32), 1 << 20))
        rs = run_rs(g, full, table, fmt)
        c = [[S] * W for _ in range(W)]
        outs = [torch.empty(W * S, device=dev()) for _ in range(W)]
        g.all_to_all([x.to(dev()) for x in full], outs, c, bits=fmt, bucket_size=bucket)
        torch.cuda.synchronize()
        for r in range(W):
            dec = outs[r].cpu().view(W, S)
            acc = full[r][r * S:(r + 1) * S].clone()
            for q in range(W):
                if q != r:
                    acc = acc + dec[q]
            assert_same(rs[r], acc, f"{fmt} rank {r}")


# ---- process group and FSDP comms, world 1 ---------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        x = torch.randn(100_003, device="cuda")
        table = [(0, 50_000, 8, 100), (50_000, 3, 32, 512), (50_003, 50_000, 8, 1024)]
        for dtype in DTYPES:
            xi = x.to(dtype)
            for fmt in FMTS:
                out = torch.empty_like(xi)
                cgx.all_gather_into_tensor(out, xi, bits=fmt, bucket_size=512)
                assert_same(out, O.fp8_quantize_dequantize(xi.cpu(), fmt, 512), f"{dtype} {fmt}")
                y = xi.clone()
                cgx.all_gather_into_tensor(y, y, bits=fmt, layers=table)
                assert_same(y, O.quantize_dequantize_layers(xi.cpu(), table, fmt=fmt), f"{dtype} {fmt} table")
                # world 1: the reduce-scatter has no peer, its output is the (prescaled) input
                r = torch.empty_like(xi)
                cgx.reduce_scatter_tensor(r, xi, bits=fmt, average=True, layers=table)
                assert_same(r, xi, f"{dtype} {fmt} rs")
        with pytest.raises(ValueError, match="round"):
            cgx.reduce_scatter_tensor(torch.empty_like(x), x, bits="e5m2", stochastic=True)
        with pytest.raises(ValueError, match="bits 8 or 32"):
            cgx.all_gather_into_tensor(torch.empty_like(x), x, bits="e4m3", layers=[(0, x.numel(), 4, 512)])
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_process_group_world1():
    spawn(_pg_world1, 1)


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(512, 256), torch.nn.LayerNorm(256), torch.nn.GELU(),
                               torch.nn.Linear(256, 10))


def _fsdp_world1(rank, world):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        model = _mlp().cuda()
        fully_shard(model)
        (comm,) = cgx.set_cgx_all_gather(model, bits="e4m3", bucket_size=512)
        rs = cgx.set_cgx_reduce_scatter(model, bits="e5m2")
        assert rs.bits == "e5m2" and [l[2] for l in comm.layers] == [8, 32, 32, 32, 8, 32]
        fsdp_params = model._get_fsdp_state()._fsdp_param_group.fsdp_params
        flat = torch.cat([fp._sharded_param_data.detach().reshape(-1) for fp in fsdp_params])
        out = comm.allocate((flat.numel(),), dtype=flat.dtype, device=flat.device)
        out.copy_(flat)
        comm(output_tensor=out, input_tensor=out[:flat.numel()], group=dist.group.WORLD, async_op=False)
        assert_same(out, O.quantize_dequantize_layers(flat.cpu(), comm.layers, fmt="e4m3"))
        g = torch.randn(4096, device="cuda")
        o = torch.empty_like(g)
        rs(output_tensor=o, input_tensor=g, group=dist.group.WORLD, op=dist.ReduceOp.AVG)
        torch.cuda.synchronize()
        assert_same(o, g)
        # training steps run through both comms
        opt = torch.optim.SGD(model.parameters(), lr=0.01)
        for _ in range(2):
            loss = model(torch.randn(8, 512, device="cuda")).square().mean()
            loss.backward()
            opt.step()
            opt.zero_grad()
        assert torch.isfinite(loss).item()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_fsdp_comms_world1():
    spawn(_fsdp_world1, 1)


# ---- several GPUs ----------------------------------------------------------------------------------
def _pg_bitwise(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            for fmt, bucket in (("e4m3", 512), ("e5m2", 1024), ("e4m3", 100)):
                S = 70_001
                full = full_inputs(world, S, dtype, world)
                out = torch.empty(S, dtype=dtype, device="cuda")
                cgx.reduce_scatter_tensor(out, full[rank].cuda(), bits=fmt, bucket_size=bucket, average=True)
                ref = O.reduce_scatter_reference(full, [(0, S, 8, bucket)], average=True, fmt=fmt)
                assert_same(out.cpu(), ref[rank], f"rs {dtype} {fmt}")
                gathered = torch.empty(world * S, dtype=dtype, device="cuda")
                cgx.all_gather_into_tensor(gathered, own(full)[rank].cuda(), bits=fmt, bucket_size=bucket)
                assert_same(gathered.cpu(), O.all_gather_reference(own(full), [(0, S, 8, bucket)], fmt),
                            f"ag {dtype} {fmt}")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
@pytest.mark.parametrize("world", [2, 4])
def test_public_api_matches_reference(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_bitwise, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport}, timeout=600)


def _fsdp_tracks_nccl(rank, world):
    from torch.distributed.fsdp import fully_shard

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        models = []
        for fp8 in (False, True):
            torch.manual_seed(0)
            m = _mlp().cuda()
            fully_shard(m)
            if fp8:
                cgx.set_cgx_all_gather(m, bits="e4m3")
                cgx.set_cgx_reduce_scatter(m, bits="e5m2")
            models.append((m, torch.optim.SGD(m.parameters(), lr=0.05)))
        torch.manual_seed(1 + rank)
        for _ in range(20):
            x = torch.randn(32, 512, device="cuda")
            y = torch.randint(0, 10, (32,), device="cuda")
            losses = []
            for m, opt in models:
                loss = torch.nn.functional.cross_entropy(m(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad()
                losses.append(loss.item())
            assert abs(losses[1] - losses[0]) < 0.05 * abs(losses[0]) + 0.05, losses
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_fsdp2_mlp_fp8_tracks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_fsdp_tracks_nccl, 2, timeout=600)
