"""FP8 wire formats of the compressed allreduce (sra_kernel / oneshot_kernel with CODEC e4m3 / e5m2) on
one H100 with W virtual ranks (C.LocalSraGroup): bitwise equal, NaN-aware, to the CPU simulator and
to the independent reference over dtypes, both formats, 512- and 1024-element slices, worlds 2-8,
mixed tables with raw layers, views at odd element offsets, edge inputs, groups halved by small heap
slots and pipeline stages; FP8, max-min and FP8 reduce-scatter calls on one heap; a CUDA graph; the
generic reducers' device kernels against the fused kernel and their wire messages against the host
backend's; the engine at world > 1 (fusion groups, the one-shot choice, the registered-bucket fast
path); ``cgx.all_reduce``, the process group and both DDP hooks at world 1; and, with >= 2 GPUs, the
public API on both transports and a DDP MLP with e5m2 gradients."""
import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs
from _engine_cases import (TIMEOUT_MS, assert_log, assert_results, clean_environment,  # noqa: F401
                           inputs_for, mixed_table)

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
N_MIXED = 43_839


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def slot_for(table, world, dtype, oneshot=False):
    plan = C.build_plan(table, world=1 if oneshot else world, lanes=lanes_for(world, dtype), dtype=DT_CODE[dtype],
                        skip_incomplete=False, min_lane_elems=MIN_LANE)
    return (plan["max_chunk_wire"] + 255) // 256 * 256 + 256


def make_group(world, dtype, slot):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, MIN_LANE)


def inputs(world, n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * (r + 1)).to(dtype) for r in range(world)]


def run(g, xs, table, fmt, *, oneshot=False, average=False, offset=1):
    """The fused allreduce of views at `offset` into sentinel-guarded buffers; returns the results."""
    bufs = []
    for x in xs:
        buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
        buf[offset:offset + x.numel()].copy_(x)
        bufs.append(buf)
    views = [b[offset:offset + x.numel()] for b, x in zip(bufs, xs)]
    (g.allreduce_oneshot if oneshot else g.allreduce)(views, table, average, False, False, 0, 1, bits=fmt)
    torch.cuda.synchronize()
    g.check()
    for r, b in enumerate(bufs):
        c = b.cpu()
        assert (c[:offset] == SENTINEL).all() and (c[offset + xs[r].numel():] == SENTINEL).all(), f"rank {r} guards"
    return [v.cpu().clone() for v in views]


def check(got, xs, table, fmt, what, *, oneshot=False, average=False):
    out = [x.clone() for x in xs]
    if oneshot:
        C.oneshot_simulate(out, table, lanes_for(len(xs), xs[0].dtype), average, min_lane_elems=MIN_LANE, bits=fmt)
        ref = O.oneshot_reference(xs, table, average=average, fmt=fmt)
    else:
        C.sra_simulate(out, table, lanes_for(len(xs), xs[0].dtype), average, min_lane_elems=MIN_LANE, bits=fmt)
        ref = O.sra_reference(xs, table, lanes=lanes_for(len(xs), xs[0].dtype), min_lane_elems=MIN_LANE,
                              average=average, fmt=fmt)
    for r in range(len(xs)):
        assert_same(got[r], out[r], f"{what}: rank {r} vs simulator")
        assert_same(got[r], ref[r], f"{what}: rank {r} vs reference")


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
    n = table[-1][0] + table[-1][1] + 9  # elements outside every layer are kept
    xs = inputs(world, n, dtype, 100 + i)
    g = make_group(world, dtype, max(slot_for(table, world, dtype), slot_for(table, world, dtype, True)))
    offset = (1, 3, 5, 0)[i % 4]  # 0: vector-aligned views
    check(run(g, xs, table, fmt, average=i % 2 == 1, offset=offset), xs, table, fmt, "sra", average=i % 2 == 1)
    check(run(g, xs, table, fmt, oneshot=True, offset=offset), xs, table, fmt, "oneshot", oneshot=True)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_fused_mixed_table(dtype, fmt):
    W = 4
    xs = inputs(W, N_MIXED, dtype, 7)
    g = make_group(W, dtype, max(slot_for(MIXED, W, dtype), slot_for(MIXED, W, dtype, True)))
    check(run(g, xs, MIXED, fmt, average=True, offset=3), xs, MIXED, fmt, "sra mixed", average=True)
    check(run(g, xs, MIXED, fmt, oneshot=True, offset=0), xs, MIXED, fmt, "oneshot mixed", oneshot=True)


@pytest.mark.parametrize("where", ["owner", "peer"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("bucket", [512, 1024, 100])
def test_fused_edge_inputs(bucket, dtype, fmt, where):
    W = 3
    n = 70 * bucket + 13
    table = [(0, n, 8, bucket)]
    owners = O.block_owners(table, n, W, lanes_for(W, dtype), dtype, False, MIN_LANE)
    xs, _ = edge_inputs(dtype, n, bucket, 11, world=W, bits=8, owners=owners, where=where)
    g = make_group(W, dtype, max(slot_for(table, W, dtype), slot_for(table, W, dtype, True)))
    check(run(g, xs, table, fmt, offset=0), xs, table, fmt, f"sra edge {where}")
    check(run(g, xs, table, fmt, oneshot=True, offset=1), xs, table, fmt, f"oneshot edge {where}", oneshot=True)


@pytest.mark.parametrize("stages", [2, 3, 4])
@pytest.mark.parametrize("fmt", FMTS)
def test_stages(fmt, stages, monkeypatch):
    monkeypatch.setenv("CGX_STAGES", str(stages))  # read when the group's kernels are set up
    W, dtype = 4, torch.bfloat16
    xs = inputs(W, N_MIXED, dtype, stages)
    g = make_group(W, dtype, slot_for(MIXED, W, dtype))
    check(run(g, xs, MIXED, fmt, average=True), xs, MIXED, fmt, f"stages {stages}", average=True)


# ---- the engine at world > 1: fusion groups, halving, one-shot choice, the fast path -----------------
ENGINE_TABLE = [(37, 32, 512), (90_000, 8, 512), (301, 32, 512), (2001, 8, 64), (700, 8, 100), (60_000, 8, 1024)]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,slot", [(2, 1 << 20), (4, 1 << 14), (8, 1 << 20)])
def test_engine_groups_and_oneshot(world, slot, fmt):
    cfg = dict(fusion_bytes=64 << 10, oneshot_max_bytes=16 << 10)
    layers, total = mixed_table(ENGINE_TABLE)
    g = C.LocalEngineGroup(world, world, cfg, 2, slot, TIMEOUT_MS)
    slots = g.slot_bytes()
    state = [t.to(dev()) for t in inputs_for(world, total, torch.float16, world)]
    for k in (1, 2):
        want, stages = O.engine_reference([s.cpu() for s in state], layers, local_size=world, config=cfg, lanes=2,
                                          slot_bytes=slots, average=k == 2, call_seq=k, fmt=fmt)
        g.allreduce_layers(state, layers, k == 2, bits=fmt)
        assert_results(state, want, f"call {k}")
        assert_log(g, stages, world)
    kinds = {s["kind"] for s in g.log(0)}
    assert "sra" in kinds and "oneshot" in kinds, kinds


@pytest.mark.parametrize("fmt", FMTS)
def test_engine_registered_bucket_fast_path(fmt, monkeypatch):
    world = 4
    cfg = dict(fusion_bytes=64 << 10, oneshot_max_bytes=16 << 10)
    layers, total = mixed_table(ENGINE_TABLE)
    for i, (off, n, bits, bucket) in enumerate(layers):
        C.register_layer(0, i, n, bits, bucket)
    monkeypatch.setenv("CGX_COMPRESSION_QUANTIZATION_BITS", "8")
    monkeypatch.setenv("CGX_COMPRESSION_BUCKET_SIZE", "512")
    g = C.LocalEngineGroup(world, world, cfg, 2, 1 << 20, TIMEOUT_MS)
    state = [t.to(dev()) for t in inputs_for(world, total, torch.bfloat16, 5)]
    for k in (1, 2, 3):
        want, stages = O.engine_reference([s.cpu() for s in state], layers, local_size=world, config=cfg, lanes=2,
                                          slot_bytes=g.slot_bytes(), average=True, call_seq=k, fmt=fmt)
        g.allreduce(state, True, 0, False, bits=fmt)
        assert_results(state, want, f"call {k}")
        assert_log(g, stages, world, fast=k > 1)
    # the fast path keys on the format: max-min next, from the same recording's layers
    want, stages = O.engine_reference([s.cpu() for s in state], layers, local_size=world, config=cfg, lanes=2,
                                      slot_bytes=g.slot_bytes(), average=True, call_seq=4)
    g.allreduce(state, True, 0, False)
    assert_results(state, want, "max-min after FP8")


# ---- interleaving, graphs ---------------------------------------------------------------------------
def test_fp8_max_min_and_reduce_scatter_interleaved_on_one_heap():
    W, dtype, n = 4, torch.float16, 40_000
    g = make_group(W, dtype, 1 << 20)
    for it, bits in enumerate(["e4m3", 8, "e5m2", 4, "e4m3"]):
        xs = inputs(W, n, dtype, it)
        fmt = bits if isinstance(bits, str) else None
        table = [(0, n, 8 if fmt else bits, 512)]
        check(run(g, xs, table, fmt), xs, table, fmt, f"sra call {it}")
        check(run(g, xs, table, fmt, oneshot=True), xs, table, fmt, f"oneshot call {it}", oneshot=True)
        S = n // W
        outs = [torch.empty(S, dtype=dtype, device=dev()) for _ in range(W)]
        rs_fmt = "e5m2" if it % 2 else "e4m3"
        g.reduce_scatter([x.to(dev()) for x in xs], outs, [(0, S, 8, 512)], False, False, False, 0, 0, bits=rs_fmt)
        torch.cuda.synchronize()
        ref = O.reduce_scatter_reference(xs, [(0, S, 8, 512)], fmt=rs_fmt)
        for r in range(W):
            assert_same(outs[r].cpu(), ref[r], f"rs call {it} rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph(fmt):
    W, dtype, n = 4, torch.float32, 60_000
    table = [(0, 37, 32, 512), (37, n - 37, 8, 1024)]
    g = make_group(W, dtype, max(slot_for(table, W, dtype), slot_for(table, W, dtype, True)))
    ts = [torch.empty(n, device=dev()) for _ in range(W)]
    os_ts = [torch.empty(n, device=dev()) for _ in range(W)]

    def step():
        g.allreduce(ts, table, True, False, False, 0, 1, bits=fmt)
        g.allreduce_oneshot(os_ts, table, False, False, False, 0, 1, bits=fmt)

    for t, o, x in zip(ts, os_ts, inputs(W, n, dtype, 0)):
        t.copy_(x)
        o.copy_(x)
    step()  # plans are built and uploaded outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        step()
    torch.cuda.synchronize()
    for it in range(3):
        xs = inputs(W, n, dtype, 10 + it)
        for t, o, x in zip(ts, os_ts, xs):
            t.copy_(x)
            o.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        check([t.cpu() for t in ts], xs, table, fmt, f"replay {it} sra", average=True)
        check([t.cpu() for t in os_ts], xs, table, fmt, f"replay {it} oneshot", oneshot=True)


# ---- the generic reducers on the device -------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_generic_device_path_equals_fused_and_host(dtype, fmt):
    W = 3
    xs = inputs(W, N_MIXED, dtype, 21)
    # the generic SRA is the lanes = 1 plan's arithmetic: compare with a one-lane fused group
    fused_g = C.LocalSraGroup(W, 1, slot_for(MIXED, W, dtype) * 4, 5000, O.GENERIC_MIN_LANE_ELEMS)
    bufs = [x.to(dev()) for x in xs]
    fused_g.allreduce(bufs, MIXED, True, False, False, 0, 1, bits=fmt)
    torch.cuda.synchronize()
    fused = [b.cpu() for b in bufs]
    got = {}
    for where in ("cpu", "cuda"):
        for kind in ("SRA", "RING"):
            red = C.LocalReducerGroup(W, kind, 5000)
            red.set_recording(True)
            out = [x.clone().to(where) for x in xs]
            red.allreduce(out, MIXED, average=True, bits=fmt)
            torch.cuda.synchronize()
            msgs = sorted(((m[1], m[2], m[3]) for m in red.messages()), key=lambda m: m[:2])
            got[where, kind] = ([o.cpu() for o in out], msgs)
        red = C.LocalReducerGroup(W, "SRA", 5000)
        out = [x.clone().to(where) for x in xs]
        red.broadcast_compressed(out, MIXED, 1, bits=fmt)
        torch.cuda.synchronize()
        got[where, "bcast"] = ([o.cpu() for o in out], [])
    want = {"SRA": O.sra_reference(xs, MIXED, lanes=1, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS, average=True, fmt=fmt),
            "RING": O.ring_reference(xs, MIXED, average=True, fmt=fmt),
            "bcast": O.broadcast_compressed_reference(xs, MIXED, root=1, fmt=fmt)}
    for kind in ("SRA", "RING", "bcast"):
        assert_results(got["cpu", kind][0], want[kind], f"host {kind} vs reference")
        assert_results(got["cuda", kind][0], want[kind], f"device {kind} vs reference")
    assert_results(fused, want["SRA"], "fused one-lane SRA vs reference")
    for r in range(W):
        assert_same(got["cuda", "SRA"][0][r], fused[r], f"generic sra vs fused rank {r}")
    # the SRA's messages byte for byte (a fresh group: the records' padding is never written, so it
    # shows the scratch's zeros on both backends; the Ring reuses one scratch across its hops)
    cpu_m, cuda_m = got["cpu", "SRA"][1], got["cuda", "SRA"][1]
    assert len(cpu_m) == len(cuda_m) == 2 * W * (W - 1)
    for a, b in zip(cpu_m, cuda_m):
        assert a[:2] == b[:2] and torch.equal(a[2], b[2]), f"SRA message {a[:2]} differs"


# ---- public API, process group and DDP hooks at world 1 ---------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        x = torch.randn(100_003, device="cuda")
        for dtype in DTYPES:
            xi = x.to(dtype)
            for fmt in FMTS:
                y = xi.clone()
                cgx.all_reduce(y, bits=fmt, bucket_size=512, average=True)
                assert_same(y, O.fp8_quantize_dequantize(xi.cpu(), fmt, 512), f"{dtype} {fmt}")
                with cgx.compression(bits=fmt, bucket_size=1024):
                    y = xi.clone()
                    dist.all_reduce(y)
                assert_same(y, O.fp8_quantize_dequantize(xi.cpu(), fmt, 1024), f"{dtype} {fmt} compression()")
                backend = cgx.backend.get_backend(dist.group.WORLD, y.device)
                y = xi.clone()
                with cgx.compression(bits=8):  # max-min in the environment, the format given to the call
                    backend.allreduce_bucket(y, -1, True, fmt).wait()
                torch.cuda.synchronize()
                assert_same(y, O.fp8_quantize_dequantize(xi.cpu(), fmt, 512), f"{dtype} {fmt} bucket")
        with pytest.raises(ValueError, match="round"):
            cgx.all_reduce(x.clone(), bits="e5m2", stochastic=True)
        with pytest.raises(ValueError, match="bits 8 or 32"), cgx.compression(bits=4):
            backend.allreduce_bucket(x.clone(), -1, True, "e4m3")
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_process_group_world1(monkeypatch):
    monkeypatch.setenv("CGX_COMPRESSION_BUCKET_SIZE", "512")
    spawn(_pg_world1, 1)


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(512, 256), torch.nn.LayerNorm(256), torch.nn.GELU(),
                               torch.nn.Linear(256, 10))


def _ddp_world1(rank, world, native):
    from torch.nn.parallel import DistributedDataParallel as DDP

    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        model = DDP(_mlp().cuda(), device_ids=[0])
        ref = _mlp().cuda()
        ref.load_state_dict(model.module.state_dict())
        state = cgx.CGXState(None, compression_params={"bits": "e5m2", "bucket_size": 512})
        handle = cgx.register_cgx_hook(model, state, native=native)
        assert (handle is not None) == native
        for step in range(4):
            x = torch.randn(16, 512, device="cuda")
            model(x).square().mean().backward()
            ref(x).square().mean().backward()
            # world 1: every compressed layer is one e5m2 round trip of its gradient (layers are
            # registered at step 2; before that the bucket goes as the environment says: raw)
            for p, q in zip(model.parameters(), ref.parameters()):
                want = q.grad
                if step >= 2 and q.dim() > 1 and q.numel() >= 1024:
                    want = O.fp8_quantize_dequantize(q.grad.reshape(-1).cpu(), "e5m2", 512).view_as(q).cuda()
                assert_same(p.grad, want, f"step {step} {tuple(p.shape)}")
            model.zero_grad()
            ref.zero_grad()
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("native", [False, True], ids=["python_hook", "native_hook"])
def test_ddp_hooks_world1(native):
    spawn(_ddp_world1, 1, args=(native,))


# ---- several GPUs ----------------------------------------------------------------------------------
def _pg_bitwise(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for dtype in DTYPES:
            for fmt, bucket, n in (("e4m3", 512, 70_001), ("e5m2", 1024, 3_000_001), ("e4m3", 100, 1001)):
                xs = inputs(world, n, dtype, world)
                y = xs[rank].cuda()
                cgx.all_reduce(y, bits=fmt, bucket_size=bucket, average=True)
                table = [(0, n, 8, bucket)]
                peers = [x.reshape(-1) for x in xs]
                want = O.sra_reference(peers, table, fmt=fmt, average=True)
                close = O.oneshot_reference(peers, table, fmt=fmt, average=True)
                # the process group picks SRA or one-shot by size: the result is one of the two, every
                # rank the same
                assert any(torch.equal(y.cpu().view(torch.int8), w[rank].view(torch.int8))
                           for w in (want, close)) or transport == "NCCL", f"{dtype} {fmt} {n}"
                gathered = [torch.empty_like(y) for _ in range(world)]
                dist.all_gather(gathered, y)
                for t in gathered:
                    assert_same(t, y, f"replicas differ {dtype} {fmt} {n}")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
@pytest.mark.parametrize("world", [2, 4])
def test_public_api_on_both_transports(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_bitwise, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport}, timeout=600)


def _ddp_tracks_nccl(rank, world):
    from torch.nn.parallel import DistributedDataParallel as DDP

    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        models = []
        for fp8 in (False, True):
            torch.manual_seed(0)
            m = DDP(_mlp().cuda(), device_ids=[rank])
            if fp8:
                cgx.register_cgx_hook(m, cgx.CGXState(None, compression_params={"bits": "e5m2", "bucket_size": 512}))
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
def test_ddp_mlp_e5m2_tracks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_ddp_tracks_nccl, 2, timeout=600)
