"""The compressed all-to-all kernel (a2a_kernel) on one H100 with W virtual ranks (C.LocalSraGroup),
against the CPU simulator and the independent reference, bit for bit and NaN-aware; small slots
with many windows per pair; its calls interleaved with the other kernels on one heap; stochastic
rounding; the generic reducer path; the public API at world 1 (eager and in a CUDA graph); and,
with >= 2 GPUs, the public API and a tiny expert-parallel MoE layer.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view and the inputs must be unchanged afterwards."""
import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import BITS, BUCKETS, DTYPES, SPLITS, WORLDS, base_elems, counts, inputs, outputs
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
GUARD = 64
SENTINEL = -7.25


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20, lanes=None):
    return C.LocalSraGroup(world, lanes or lanes_for(world, dtype), slot, 5000, 256)


def guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def run_fused(g, xs, c, bits, bucket, offset=0, **kw):
    ins = [guarded(x.to(dev()), offset) for x in xs]
    outs = [guarded(o.to(dev()), offset) for o in outputs(c, xs[0].dtype)]
    g.all_to_all([v for _, v in ins], [v for _, v in outs], c, bits=bits, bucket_size=bucket, **kw)
    torch.cuda.synchronize()
    g.check()
    for (buf, v), x in zip(ins, xs):
        assert_same(v.cpu(), x, "input modified")
    for buf, v in ins + outs:
        n = v.numel()
        assert (buf[:offset] == SENTINEL).all() and (buf[offset + n:] == SENTINEL).all(), "sentinel overwritten"
    return [v.cpu() for _, v in outs]


def check(got, xs, c, bits, bucket, what, **kw):
    sim = outputs(c, xs[0].dtype)
    C.all_to_all_simulate(xs, sim, c, bits=bits, bucket_size=bucket, **kw)
    ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket) if not kw.get("stochastic") else sim
    for r in range(len(xs)):
        assert_same(got[r], sim[r], f"{what}: rank {r} vs simulator")
        assert_same(got[r], ref[r], f"{what}: rank {r} vs reference")


@pytest.mark.parametrize("dtype,bits,bucket", list(itertools.product(DTYPES, BITS, BUCKETS)))
def test_fused_matches_simulator_and_reference(dtype, bits, bucket):
    i = DTYPES.index(dtype) * 7 + BITS.index(bits) * 3 + BUCKETS.index(bucket)
    W = WORLDS[i % len(WORLDS)]
    base = base_elems(bucket) if W <= 5 else max(300, min(base_elems(bucket), 2000))
    kind = SPLITS[i % len(SPLITS)]
    c = counts(W, kind, base, seed=i)
    xs = inputs(c, dtype, i)
    got = run_fused(make_group(W, dtype), xs, c, bits, bucket, offset=(1, 3, 5)[i % 3])
    check(got, xs, c, bits, bucket, f"W={W} {kind}")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind", SPLITS)
def test_fused_every_world_and_split(world, kind):
    c = counts(world, kind, 3000, seed=world)
    xs = inputs(c, torch.bfloat16, world)
    got = run_fused(make_group(world, torch.bfloat16), xs, c, 4, 512, offset=3)
    check(got, xs, c, 4, 512, f"W={world} {kind}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_edge_inputs(dtype):
    W, bucket, n = 3, 64, 40 * 64
    xs, _ = edge_inputs(dtype, n * W, bucket, seed=2, world=W, bits=4)
    c = [[n] * W for _ in range(W)]
    check(run_fused(make_group(W, dtype), xs, c, 4, bucket, offset=1), xs, c, 4, bucket, "edge")


@pytest.mark.parametrize("bits,bucket", [(8, 512), (4, 1024), (3, 100), (32, 512)])
def test_small_slots_many_windows(bits, bucket):
    # lanes' shares of two blocks: pairs with zero, one and many windows, different per pair
    W, lanes, dtype = 4, 2, torch.bfloat16
    block = C.a2a_windows(1, bits, bucket, DT_CODE[dtype], 1 << 20, 1)["block_wire"]
    g = make_group(W, dtype, slot=((2 * lanes * block + 16 * lanes) + 255) // 256 * 256, lanes=lanes)
    c = [[0, 9000, 70000, 123457], [8192, 0, 1, 0], [50000, 0, 33, 16385], [0, 200000, 5, 7]]
    for q in range(W):
        c[q][q] = 1000 * q
    w = C.a2a_windows(200000, bits, bucket, DT_CODE[dtype], g_slot(g, lanes, block), lanes)
    assert len(w["lanes"][0]) > 3
    xs = inputs(c, dtype, 7)
    check(run_fused(g, xs, c, bits, bucket, offset=5), xs, c, bits, bucket, "small slots")


def g_slot(g, lanes, block):  # `g` unused: a slot holding two blocks per lane
    return ((2 * lanes * block + 16 * lanes) + 255) // 256 * 256


def test_mixed_calls_on_one_heap():
    W, dtype, S = 4, torch.float32, 20_000
    g = make_group(W, dtype)
    shard = [(0, S, 4, 512)]
    for it in range(2):
        c = counts(W, "uneven", 5000, seed=it)
        xs = inputs(c, dtype, it)
        check(run_fused(g, xs, c, 4, 512), xs, c, 4, 512, f"a2a {it}")
        rs_in = [torch.randn(W * S, dtype=dtype) for _ in range(W)]
        rs_out = [torch.zeros(S, dtype=dtype, device=dev()) for _ in range(W)]
        g.reduce_scatter([x.to(dev()) for x in rs_in], rs_out, shard, False, False, False, 0, 0)
        ag_in = [torch.randn(S, dtype=dtype) for _ in range(W)]
        ag_out = [torch.zeros(W * S, dtype=dtype, device=dev()) for _ in range(W)]
        g.all_gather([x.to(dev()) for x in ag_in], ag_out, shard, False, 0, 0)
        ar = [torch.randn(W * S, dtype=dtype) for _ in range(W)]
        ar_dev = [x.to(dev()) for x in ar]
        g.allreduce(ar_dev, [(0, W * S, 4, 512)], False, False, False, 0, 0)
        torch.cuda.synchronize()
        g.check()
        rs_ref = [torch.zeros(S, dtype=dtype) for _ in range(W)]
        C.reduce_scatter_simulate(rs_in, rs_ref, shard, lanes=lanes_for(W, dtype), min_lane_elems=256)
        ag_ref = O.all_gather_reference(ag_in, shard)
        ar_ref = [x.clone() for x in ar]
        C.sra_simulate(ar_ref, [(0, W * S, 4, 512)], lanes=lanes_for(W, dtype), min_lane_elems=256)
        for r in range(W):
            assert_same(rs_out[r].cpu(), rs_ref[r], f"rs {it} rank {r}")
            assert_same(ag_out[r].cpu(), ag_ref, f"ag {it} rank {r}")
            assert_same(ar_dev[r].cpu(), ar_ref[r], f"ar {it} rank {r}")


def test_stochastic_matches_simulator_and_changes_with_seq():
    W, dtype = 3, torch.float32
    g = make_group(W, dtype)
    c = counts(W, "uneven", 6000, seed=3)
    xs = inputs(c, dtype, 3)
    a = run_fused(g, xs, c, 3, 128, stochastic=True, seed=11, seq=1)
    check(a, xs, c, 3, 128, "stochastic seq 1", stochastic=True, seed=11, seq=1)
    b = run_fused(g, xs, c, 3, 128, stochastic=True, seed=11, seq=2)
    check(b, xs, c, 3, 128, "stochastic seq 2", stochastic=True, seed=11, seq=2)
    assert any(not torch.equal(a[r], b[r]) for r in range(W) if a[r].numel())


@pytest.mark.parametrize("bits,bucket", [(4, 512), (8, 1024), (3, 7), (32, 512)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_path_equals_fused(bits, bucket, dtype):
    W = 3
    c = counts(W, "uneven", 4000, seed=bits)
    xs = inputs(c, dtype, bits)
    fused = run_fused(make_group(W, dtype), xs, c, bits, bucket)
    red = C.LocalReducerGroup(W, "SRA", 5000)
    ins = [x.to(dev()) for x in xs]
    outs = outputs(c, dtype, device=dev())
    red.all_to_all(ins, outs, c, bits=bits, bucket_size=bucket)
    torch.cuda.synchronize()
    for r in range(W):
        assert_same(outs[r].cpu(), fused[r], f"generic vs fused rank {r}")


def test_generic_path_across_many_chunk_sizes():
    # more distinct chunk sizes than the generic reducer's plan cache holds: it is dropped and rebuilt
    # mid-run, and the plans rebuilt after the drop are uploaded again
    W, dtype = 2, torch.bfloat16
    red = C.LocalReducerGroup(W, "SRA", 5000)
    for it in range(140):
        c = [[100 + it, 3000 + 7 * it], [2000 + 5 * it, 50 + it]]
        xs = inputs(c, dtype, it)
        outs = outputs(c, dtype, device=dev())
        red.all_to_all([x.to(dev()) for x in xs], outs, c, bits=4, bucket_size=64)
        torch.cuda.synchronize()
        sim = outputs(c, dtype)
        C.all_to_all_simulate(xs, sim, c, bits=4, bucket_size=64)
        for r in range(W):
            assert_same(outs[r].cpu(), sim[r], f"call {it} rank {r}")
            assert red.num_plans(r) <= 256


def test_cuda_graph_virtual_ranks():
    """Capture one call of W = 4 virtual ranks with fixed uneven splits and small slots (many windows
    per pair), then replay it on new data interleaved with eager calls: the window tags come from the
    device epoch, so replays and eager calls keep agreeing on every flag."""
    W, lanes, dtype, bits, bucket = 4, 2, torch.float32, 4, 512
    block = C.a2a_windows(1, bits, bucket, DT_CODE[dtype], 1 << 20, 1)["block_wire"]
    g = make_group(W, dtype, slot=g_slot(g=None, lanes=lanes, block=block), lanes=lanes)
    c = [[1000, 70000, 0, 9000], [8192, 500, 40000, 1], [0, 33, 2000, 100000], [65000, 0, 5, 300]]
    ins = [torch.empty(sum(row), device=dev(), dtype=dtype) for row in c]
    outs = [torch.empty(sum(c[q][r] for q in range(W)), device=dev(), dtype=dtype) for r in range(W)]
    xs = inputs(c, dtype, 0)
    for t, x in zip(ins, xs):
        t.copy_(x)
    g.all_to_all(ins, outs, c, bits=bits, bucket_size=bucket)  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        g.all_to_all(ins, outs, c, bits=bits, bucket_size=bucket)
    torch.cuda.synchronize()
    for it in range(3):
        xs = inputs(c, dtype, 100 + it)
        for t, x in zip(ins, xs):
            t.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        check([o.cpu() for o in outs], xs, c, bits, bucket, f"replay {it}")
        ys = inputs(c, dtype, 200 + it)
        check(run_fused(g, ys, c, bits, bucket, offset=3), ys, c, bits, bucket, f"eager {it}")


# ---- the public API at world 1 -------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            x = torch.randn(1000, 7, device="cuda").to(dtype)
            out = torch.full_like(x, SENTINEL)
            cgx.all_to_all_single(out, x, bits=4)
            assert_same(out, x, f"{dtype}: the own chunk is a copy")
            out2 = torch.full_like(x, SENTINEL)
            dist.all_to_all_single(out2, x)  # the uncompressed delegate
            assert_same(out2, x, f"{dtype}: dist.all_to_all_single")
        y = cgx.differentiable_all_to_all_single(x.float().requires_grad_(), [1000], [1000], bits=4)
        y.sum().backward()
        with pytest.raises(RuntimeError, match="sums to"):
            cgx.all_to_all_single(torch.empty(10, device="cuda"), torch.empty(10, device="cuda"), [9], [10])
        with pytest.raises(RuntimeError, match="entries"):
            cgx.all_to_all_single(torch.empty(10, device="cuda"), torch.empty(10, device="cuda"), [5, 5], [10])
        with pytest.raises(RuntimeError, match="negative"):
            cgx.all_to_all_single(torch.empty(10, device="cuda"), torch.empty(10, device="cuda"), [-1], [10])
        with pytest.raises(RuntimeError, match="rows"):
            cgx.all_to_all_single(torch.empty(10, 2, device="cuda"), torch.empty(10, 3, device="cuda"))
        with pytest.raises(ValueError, match="overlaps"):
            t = torch.empty(20, device="cuda")
            cgx.all_to_all_single(t[5:15], t[0:10])
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def _graph_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        x = torch.randn(50_000, device="cuda")
        out = torch.empty_like(x)
        cgx.all_to_all_single(out, x, bits=4)  # initialise outside the capture
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            cgx.all_to_all_single(out, x, [50_000], [50_000], bits=4)
        for it in range(3):
            x.copy_(torch.randn(50_000, device="cuda"))
            graph.replay()
            torch.cuda.synchronize()
            assert_same(out, x, f"replay {it}")
            eager = torch.empty_like(x)
            cgx.all_to_all_single(eager, x, bits=4)
            assert_same(eager, x, f"eager {it}")
    finally:
        dist.destroy_process_group()


def test_cuda_graph_world1():
    spawn(_graph_world1, 1)


# ---- several GPUs ------------------------------------------------------------------------------
def _pg_bitwise(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for it, (dtype, bits, bucket) in enumerate([(torch.bfloat16, 8, 512), (torch.float32, 4, 1024),
                                                   (torch.float16, 3, 100), (torch.float32, 32, 512)]):
            c = counts(world, "uneven", 4000, seed=it)
            xs = inputs(c, dtype, it)
            out = torch.full((sum(c[q][rank] for q in range(world)),), SENTINEL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, xs[rank].cuda(), [c[q][rank] for q in range(world)], c[rank], bits=bits,
                                  bucket_size=bucket)
            ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket)[rank]
            assert_same(out.cpu(), ref, f"{transport} {dtype} bits={bits}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
def test_public_api_matches_reference(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_bitwise, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport}, timeout=600)


def _graph_world2(rank, world):
    """Capture a fixed uneven-split call at world 2 with small slots (many windows per pair) and replay
    it on new data, interleaved with eager calls, against the reference; with stochastic rounding,
    replays advance the random stream."""
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        c = [[30_000, 250_000], [170_000, 4_000]]
        recv = [c[q][rank] for q in range(world)]
        x = torch.empty(sum(c[rank]), device="cuda")
        out = torch.empty(sum(recv), device="cuda")
        cgx.all_to_all_single(out, x.normal_(), recv, c[rank], bits=4)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            cgx.all_to_all_single(out, x, recv, c[rank], bits=4)
        for it in range(3):
            xs = inputs(c, torch.float32, 10 + it)
            x.copy_(xs[rank])
            graph.replay()
            torch.cuda.synchronize()
            assert_same(out.cpu(), O.all_to_all_reference(xs, c, bits=4, bucket_size=512)[rank], f"replay {it}")
            eager = torch.empty_like(out)
            cgx.all_to_all_single(eager, x, recv, c[rank], bits=4)
            assert_same(eager.cpu(), out.cpu(), f"eager {it}")
        sgraph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(sgraph, stream=s):
            cgx.all_to_all_single(out, x, recv, c[rank], bits=2, stochastic=True, seed=7)
        sgraph.replay()
        torch.cuda.synchronize()
        first = out.clone()
        sgraph.replay()
        torch.cuda.synchronize()
        peer = 1 - rank
        lo = sum(recv[:peer])
        assert not torch.equal(first[lo:lo + recv[peer]], out[lo:lo + recv[peer]]), "replays reuse the stream"
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_cuda_graph_world2():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_graph_world2, 2, env={"CGX_FUSION_BUFFER_SIZE_MB": "1"}, timeout=600)


def _moe(rank, world):
    """Top-1 expert parallelism, one expert per rank: tokens dispatched to their expert's rank, the
    expert applied, the results combined back. Forward and backward against a reference composed
    from the oracle; with grad_bits=32 the backward's exchange is exact."""
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)
        T, D = 96, 64
        xs = [torch.randn(T, D, generator=g) for _ in range(world)]
        route = [torch.randint(0, world, (T,), generator=g) for _ in range(world)]
        ws = [torch.randn(D, D, generator=g) / D ** 0.5 for _ in range(world)]
        order = [torch.argsort(rt, stable=True) for rt in route]
        send = [[int((rt == q).sum()) for q in range(world)] for rt in route]  # send[r][q] tokens
        x = xs[rank][order[rank]].cuda().requires_grad_()
        recv = [send[q][rank] for q in range(world)]
        tokens = cgx.differentiable_all_to_all_single(x, recv, send[rank], bits=8, grad_bits=32)
        w = ws[rank].cuda().requires_grad_()
        y = tokens @ w
        back = cgx.differentiable_all_to_all_single(y, send[rank], recv, bits=8, grad_bits=32)
        back.sum().backward()
        # reference: the dispatch through the oracle, the expert in fp32, the combine through the oracle
        counts_d = [[send[q][r] * D for r in range(world)] for q in range(world)]
        disp = O.all_to_all_reference([xs[q][order[q]] for q in range(world)], counts_d, bits=8, bucket_size=512)
        ys = [(disp[r].view(-1, D).cuda() @ ws[r].cuda()).cpu() for r in range(world)]
        counts_c = [[send[r][q] * D for r in range(world)] for q in range(world)]
        comb = O.all_to_all_reference(ys, counts_c, bits=8, bucket_size=512)
        assert_same(tokens.detach().cpu().reshape(-1), disp[rank], "dispatch")
        assert_same(back.detach().cpu().reshape(-1), comb[rank], "combine")
        # backward of sum(): d back = 1, exact through the combine; d tokens = 1 @ w^T, exact back
        torch.testing.assert_close(w.grad, tokens.detach().t() @ torch.ones_like(y), rtol=1e-5, atol=1e-5)
        experts = route[rank][order[rank]]
        gx = torch.stack([ws[int(e)].sum(dim=1) for e in experts])
        torch.testing.assert_close(x.grad.cpu(), gx, rtol=1e-5, atol=1e-5)
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_moe_layer_forward_backward():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_moe, 2, timeout=600)
