"""FP8 wire formats of the compressed all-to-all (a2a_kernel with CODEC e4m3 / e5m2) on one H100 with
W virtual ranks (C.LocalSraGroup): bitwise equal, NaN-aware, to the CPU simulator (the host codec)
and to the independent numpy / torch.float8 reference over dtypes, both formats, buckets, worlds
and split kinds; the routed form with top-k repeats; small slots with many windows per pair; FP8,
max-min and raw calls on one heap; a CUDA graph; the generic reducer's device kernels against the
fused kernel and its wire messages against the host backend's; the public API at world 1; and, with
>= 2 GPUs, the public API on both transports and an MoE layer with e4m3 dispatch and e5m2 gradients.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view and the inputs must be unchanged afterwards."""
import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel.hooks import _native_backend

from _a2a_cases import DTYPES, counts, inputs, outputs
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
FMTS = ("e4m3", "e5m2")
F_BUCKETS = (64, 100, 128, 512, 1024, 8192)
F_WORLDS = (2, 3, 8, 16)
F_SPLITS = ("equal", "uneven", "empty")
GUARD = 64
SENTINEL = -7.25


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20, lanes=None):
    return C.LocalSraGroup(world, lanes or lanes_for(world, dtype), slot, 5000, 256)


def small_slot(bits, bucket, dtype, lanes):
    """a slot that holds two blocks per lane: pairs with zero, one and many windows"""
    block = C.a2a_windows(1, bits, bucket, DT_CODE[dtype], 1 << 20, 1)["block_wire"]
    return ((2 * lanes * block + 16 * lanes) + 255) // 256 * 256


def guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


def run_fused(g, xs, c, bits, bucket, offset=0):
    ins = [guarded(x.to(dev()), offset) for x in xs]
    outs = [guarded(o.to(dev()), offset) for o in outputs(c, xs[0].dtype)]
    g.all_to_all([v for _, v in ins], [v for _, v in outs], c, bits=bits, bucket_size=bucket)
    torch.cuda.synchronize()
    g.check()
    for (buf, v), x in zip(ins, xs):
        assert_same(v.cpu(), x, "input modified")
    for buf, v in ins + outs:
        n = v.numel()
        assert (buf[:offset] == SENTINEL).all() and (buf[offset + n:] == SENTINEL).all(), "sentinel overwritten"
    return [v.cpu() for _, v in outs]


def check(got, xs, c, bits, bucket, what):
    sim = outputs(c, xs[0].dtype)
    C.all_to_all_simulate(xs, sim, c, bits=bits, bucket_size=bucket)
    ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=bucket)
    for r in range(len(xs)):
        assert_same(got[r], sim[r], f"{what}: rank {r} vs simulator")
        assert_same(got[r], ref[r], f"{what}: rank {r} vs reference")


# ---- the fused kernel against the simulator and the reference ------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, F_BUCKETS)))
def test_fused_matches_simulator_and_reference(dtype, fmt, bucket):
    i = DTYPES.index(dtype) * 12 + FMTS.index(fmt) * 6 + F_BUCKETS.index(bucket)
    for j, W in enumerate(F_WORLDS):
        kind = F_SPLITS[(i + j) % len(F_SPLITS)]
        base = max(300, bucket + bucket // 3 + 5) if W <= 3 else max(300, min(bucket + 77, 2000))
        c = counts(W, kind, base, seed=i * 7 + j)
        xs = inputs(c, dtype, i * 7 + j)
        got = run_fused(make_group(W, dtype), xs, c, fmt, bucket, offset=(1, 3, 5)[(i + j) % 3])
        check(got, xs, c, fmt, bucket, f"W={W} {kind}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world", F_WORLDS)
@pytest.mark.parametrize("kind", F_SPLITS)
def test_fused_every_world_and_split(fmt, world, kind):
    c = counts(world, kind, 3000, seed=world)
    xs = inputs(c, torch.bfloat16, world)
    got = run_fused(make_group(world, torch.bfloat16), xs, c, fmt, 512, offset=3)
    check(got, xs, c, fmt, 512, f"W={world} {kind}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [64, 512])
def test_fused_edge_inputs(dtype, fmt, bucket):
    W, n = 3, 12 * 512
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=2, world=W, bits=8)
    assert planted
    c = [[n] * W for _ in range(W)]
    check(run_fused(make_group(W, dtype), xs, c, fmt, bucket, offset=1), xs, c, fmt, bucket, "edge")


# ---- the routed form -------------------------------------------------------------------------------
def _routed_case(W, H, dtype, seed):
    """top-k style: rank q sends rows[q][r] rows gathered by an index with repeats, rank r scatters
    what it receives by a permutation into a larger output"""
    g = torch.Generator().manual_seed(seed)
    rows = counts(W, "uneven", 4, seed=seed)
    c = [[rows[q][r] * H for r in range(W)] for q in range(W)]
    send = [sum(rows[q]) for q in range(W)]
    recv = [sum(rows[q][r] for q in range(W)) for r in range(W)]
    xs = [(torch.randn(max(1, s // 2 + 1), H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype)
          for q, s in enumerate(send)]
    ii = [torch.randint(0, x.shape[0], (s,), generator=g) for x, s in zip(xs, send)]
    oi = [torch.randperm(m + 5, generator=g)[:m] for m in recv]
    out0 = [torch.randn(m + 5, H, generator=g).to(dtype) for m in recv]
    return c, xs, ii, oi, out0


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H,bucket", [(512, 512), (1024, 1024), (7168, 512), (7168, 128)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_routed_matches_reference(fmt, H, bucket, dtype):
    W = 4
    assert C.a2a_rows_fit(H, 8, bucket, DT_CODE[dtype])
    c, xs, ii, oi, out0 = _routed_case(W, H, dtype, seed=H + bucket)
    g = make_group(W, dtype)
    ins = [x.to(dev()) for x in xs]
    outs = [o.to(dev()) for o in out0]
    g.all_to_all([x.reshape(-1) for x in ins], [o.reshape(-1) for o in outs], c, bits=fmt, bucket_size=bucket,
                 input_index=[ix.to(dev()) for ix in ii], output_index=[ix.to(dev()) for ix in oi], row=H)
    torch.cuda.synchronize()
    g.check()
    ref = O.routed_all_to_all_reference(xs, c, ii, oi, H, bits=fmt, bucket_size=bucket, outputs=out0)
    # the simulator composition: index_select, the plain exchange, index_copy_
    send = [x.index_select(0, ix).reshape(-1) for x, ix in zip(xs, ii)]
    sim = outputs(c, dtype)
    C.all_to_all_simulate(send, sim, c, bits=fmt, bucket_size=bucket)
    for r in range(W):
        want = out0[r].clone().index_copy_(0, oi[r], sim[r].reshape(-1, H)).reshape(-1)
        assert_same(outs[r].cpu().reshape(-1), want, f"rank {r} vs simulator")
        assert_same(outs[r].cpu().reshape(-1), ref[r], f"rank {r} vs reference")


# ---- windows, heap sharing, graphs -------------------------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 512), ("e5m2", 1024), ("e4m3", 100), ("e5m2", 8192)])
def test_small_slots_many_windows(fmt, bucket):
    W, lanes, dtype = 4, 2, torch.bfloat16
    slot = small_slot(8, bucket, dtype, lanes)
    g = make_group(W, dtype, slot=slot, lanes=lanes)
    c = [[0, 9000, 70000, 123457], [8192, 0, 1, 0], [50000, 0, 33, 16385], [0, 200000, 5, 7]]
    for q in range(W):
        c[q][q] = 1000 * q
    assert len(C.a2a_windows(200000, 8, bucket, DT_CODE[dtype], slot, lanes)["lanes"][0]) > 3
    xs = inputs(c, dtype, 7)
    check(run_fused(g, xs, c, fmt, bucket, offset=5), xs, c, fmt, bucket, "small slots")


def test_fp8_max_min_and_raw_interleaved_on_one_heap():
    W, dtype = 4, torch.float16
    g = make_group(W, dtype)
    for it, bits in enumerate(["e4m3", 8, 32, "e5m2", 4, "e4m3"]):
        c = counts(W, "uneven", 3000, seed=it)
        xs = inputs(c, dtype, it)
        check(run_fused(g, xs, c, bits, 512, offset=(1, 3, 5)[it % 3]), xs, c, bits, 512, f"call {it} bits={bits}")


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph_virtual_ranks(fmt):
    """one FP8 call of W = 4 virtual ranks with fixed uneven splits and small slots, captured and
    replayed on new data, interleaved with eager max-min calls"""
    W, lanes, dtype, bucket = 4, 2, torch.float32, 512
    g = make_group(W, dtype, slot=small_slot(8, bucket, dtype, lanes), lanes=lanes)
    c = [[1000, 70000, 0, 9000], [8192, 500, 40000, 1], [0, 33, 2000, 100000], [65000, 0, 5, 300]]
    ins = [torch.empty(sum(row), device=dev(), dtype=dtype) for row in c]
    outs = [torch.empty(sum(c[q][r] for q in range(W)), device=dev(), dtype=dtype) for r in range(W)]
    for t, x in zip(ins, inputs(c, dtype, 0)):
        t.copy_(x)
    g.all_to_all(ins, outs, c, bits=fmt, bucket_size=bucket)  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        g.all_to_all(ins, outs, c, bits=fmt, bucket_size=bucket)
    torch.cuda.synchronize()
    for it in range(3):
        xs = inputs(c, dtype, 100 + it)
        for t, x in zip(ins, xs):
            t.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        check([o.cpu() for o in outs], xs, c, fmt, bucket, f"replay {it}")
        ys = inputs(c, dtype, 200 + it)
        check(run_fused(g, ys, c, 8, bucket, offset=3), ys, c, 8, bucket, f"eager max-min {it}")


# ---- the generic reducer (NCCL transport's path) -----------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 512), ("e5m2", 1024), ("e4m3", 7), ("e5m2", 10000)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_path_equals_fused(fmt, bucket, dtype):
    W = 3
    c = counts(W, "uneven", 4000, seed=bucket)
    xs = inputs(c, dtype, bucket)
    fused = run_fused(make_group(W, dtype), xs, c, fmt, bucket)
    red = C.LocalReducerGroup(W, "SRA", 5000)
    outs = outputs(c, dtype, device=dev())
    red.all_to_all([x.to(dev()) for x in xs], outs, c, bits=fmt, bucket_size=bucket)
    torch.cuda.synchronize()
    for r in range(W):
        assert_same(outs[r].cpu(), fused[r], f"generic vs fused rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_device_messages_equal_host(fmt, dtype):
    """the device item kernels put the host codec's bytes on the wire, poisoned buckets included"""
    W, bucket = 3, 64
    n = 40 * bucket + 13  # a partial last bucket
    xs, _ = edge_inputs(dtype, n * W, bucket, seed=4, world=W, bits=8)
    c = [[n] * W for _ in range(W)]
    got = {}
    for where in ("cpu", "cuda"):
        red = C.LocalReducerGroup(W, "SRA", 5000)
        red.set_recording(True)
        outs = outputs(c, dtype, device=where)
        red.all_to_all([x.to(where) for x in xs], outs, c, bits=fmt, bucket_size=bucket)
        torch.cuda.synchronize()
        got[where] = ([o.cpu() for o in outs], {(m[1], m[2]): m[3] for m in red.messages()})
    assert len(got["cpu"][1]) == W * (W - 1)
    assert got["cpu"][1].keys() == got["cuda"][1].keys()
    for k, m in got["cpu"][1].items():
        assert torch.equal(m, got["cuda"][1][k]), f"message {k} differs"
    for r in range(W):
        assert_same(got["cuda"][0][r], got["cpu"][0][r], f"rank {r}")


# ---- the public API at world 1 -------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            x = torch.randn(1000, 7, device="cuda").to(dtype)
            for fmt in FMTS:
                out = torch.full_like(x, SENTINEL)
                cgx.all_to_all_single(out, x, bits=fmt)
                assert_same(out, x, f"{dtype} {fmt}: the own chunk is a copy")
        x = torch.randn(64, 1024, device="cuda")
        ii = torch.randint(0, 64, (100,), device="cuda")
        out = torch.full((100, 1024), SENTINEL, device="cuda")
        cgx.all_to_all_single(out, x, [100], [100], bits="e4m3", input_index=ii)
        assert_same(out, x.index_select(0, ii), "routed own chunk")
        with pytest.raises(ValueError, match="round"):
            cgx.all_to_all_single(torch.empty(10, device="cuda"), torch.ones(10, device="cuda"), bits="e4m3",
                                  stochastic=True)
        with pytest.raises(ValueError):
            cgx.all_to_all_single(torch.empty(10, device="cuda"), torch.ones(10, device="cuda"), bits="e3m4")
        # the native binding parses the same vocabulary itself
        native = _native_backend(dist.group.WORLD, x)
        with pytest.raises(ValueError):
            native.all_to_all_compressed(torch.empty(10, device="cuda"), torch.ones(10, device="cuda"), [], [],
                                         "e5m2", 512, True, -1, None, None)
        xa = torch.randn(300, 64, device="cuda", requires_grad=True)
        y = cgx.differentiable_all_to_all_single(xa, [300], [300], bits="e4m3", grad_bits="e5m2")
        w = torch.randn(300, 64, device="cuda")
        (y * w).sum().backward()
        assert_same(y.detach(), xa.detach(), "differentiable forward")
        assert_same(xa.grad, w, "differentiable backward")
        with pytest.raises(ValueError):
            cgx.differentiable_all_to_all_single(xa, bits=8, grad_bits="e5m2", stochastic=True)
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


# ---- several GPUs ------------------------------------------------------------------------------
def _pg_bitwise(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for it, (dtype, fmt, bucket) in enumerate([(torch.bfloat16, "e4m3", 512), (torch.float32, "e5m2", 1024),
                                                  (torch.float16, "e4m3", 100), (torch.float32, "e5m2", 64)]):
            c = counts(world, "uneven", 4000, seed=it)
            xs = inputs(c, dtype, it)
            out = torch.full((sum(c[q][rank] for q in range(world)),), SENTINEL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, xs[rank].cuda(), [c[q][rank] for q in range(world)], c[rank], bits=fmt,
                                  bucket_size=bucket)
            ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=bucket)[rank]
            assert_same(out.cpu(), ref, f"{transport} {dtype} {fmt}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
def test_public_api_matches_reference(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_bitwise, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport}, timeout=600)


def _moe_fp8(rank, world):
    """Top-2 routing, one expert per rank, e4m3 dispatch and e5m2 gradients, routed by index: forward
    and backward bitwise against autograd through the composition with the same formats."""
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True)
    try:
        g = torch.Generator().manual_seed(0)
        T, D, k = 64, 1024, 2
        route = [torch.stack([torch.randperm(world, generator=g)[:k] for _ in range(T)]) for _ in range(world)]
        ws = [torch.randn(D, D, generator=g) / D ** 0.5 for _ in range(world)]
        xs = [torch.randn(T, D, generator=g) for _ in range(world)]
        order = [torch.argsort(rt.reshape(-1), stable=True) for rt in route]
        send = [[int((rt == q).sum()) for q in range(world)] for rt in route]
        recv = [send[q][rank] for q in range(world)]
        ii, oi = (order[rank] // k).cuda(), order[rank].cuda()
        w = ws[rank].cuda()
        kw = dict(bits="e4m3", grad_bits="e5m2")

        def layer(x, routed):
            if routed:
                tok = cgx.differentiable_all_to_all_single(x, recv, send[rank], input_index=ii, **kw)
                return cgx.differentiable_all_to_all_single(tok @ w, send[rank], recv, output_index=oi,
                                                            output_rows=T * k, **kw)
            tok = cgx.differentiable_all_to_all_single(x.index_select(0, ii), recv, send[rank], **kw)
            back = cgx.differentiable_all_to_all_single(tok @ w, send[rank], recv, **kw)
            return torch.zeros(T * k, D, device="cuda").index_copy(0, oi, back)

        gate = torch.rand(T * k, 1, generator=g).cuda()
        outs, grads = [], []
        for routed in (True, False):
            x = xs[rank].cuda().requires_grad_()
            out = (layer(x, routed) * gate).view(T, k, D).sum(1)
            out.square().sum().backward()
            outs.append(out.detach())
            grads.append(x.grad)
        assert_same(outs[0], outs[1], "forward")
        assert_same(grads[0], grads[1], "backward")
        assert torch.isfinite(outs[0]).all() and torch.isfinite(grads[0]).all()
    finally:
        torch.use_deterministic_algorithms(False)
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_moe_fp8_dispatch_forward_backward():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_moe_fp8, 2, env={"CUBLAS_WORKSPACE_CONFIG": ":4096:8"}, timeout=600)
