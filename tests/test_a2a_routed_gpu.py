"""The routed all-to-all (a2a_kernel with row indices) on one H100 with W virtual ranks
(C.LocalSraGroup): bitwise equal to the composition index_select -> plain kernel -> index_copy_,
NaN-aware, over dtypes, widths, buckets, worlds, split kinds and index kinds; small slots with many
windows per pair; stochastic rounding; routed and plain calls on one heap; rows of an index outside
its tensor; the public API at world 1 (eager, with rows the kernel cannot route, and in a CUDA graph
whose indices change between replays); and, with >= 2 GPUs, the public API on both transports and
a top-2 MoE layer routed end to end.

Data, outputs and indices are views into sentinel-filled buffers: the elements around each view,
the inputs and the indices must be unchanged afterwards, and the output rows no index names keep
their previous contents."""
import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import DTYPES, counts
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
GUARD_ROWS = 2
SENTINEL = -7.25
IX_SENTINEL = -(1 << 40)
R_BITS = (2, 3, 4, 8, 32)
R_BUCKETS = (64, 512, 1024)
R_WORLDS = (2, 3, 5, 8, 16)
R_SPLITS = ("equal", "uneven", "empty")
R_MODES = ("input", "output", "both")


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20, lanes=None):
    return C.LocalSraGroup(world, lanes or lanes_for(world, dtype), slot, 5000, 256)


def guarded_rows(x, H):
    """x ([rows, H]) copied into the middle of a buffer with GUARD_ROWS sentinel rows on each side"""
    buf = torch.full((x.shape[0] + 2 * GUARD_ROWS, H), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[GUARD_ROWS:GUARD_ROWS + x.shape[0]]
    view.copy_(x)
    return buf, view


def guarded_index(ix):
    buf = torch.full((ix.numel() + 6,), IX_SENTINEL, dtype=torch.long, device=dev())
    view = buf[3:3 + ix.numel()]
    view.copy_(ix)
    return buf, view


class Case:
    """W ranks' routed call: rows[q][r] rows from q to r, rank q's physical input of in_rows[q]
    rows, its input index (or None), rank r's output of out_rows[r] rows and its index (or None)"""

    def __init__(self, W, H, rows, dtype, mode, seed, topk=True):
        g = torch.Generator().manual_seed(seed)
        self.W, self.H, self.rows, self.dtype = W, H, rows, dtype
        self.counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        send = [sum(rows[q]) for q in range(W)]
        recv = [sum(rows[q][r] for q in range(W)) for r in range(W)]
        self.xs, self.ii, self.oi, self.out0 = [], [], [], []
        for q in range(W):
            if mode in ("input", "both"):
                # fewer physical rows than sent rows: top-k style repeats
                n = max(1, send[q] // 2 + 1) if topk else send[q] + 3
                self.ii.append(torch.randint(0, n, (send[q],), generator=g))
            else:
                n = send[q]
                self.ii.append(None)
            self.xs.append((torch.randn(n, H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype))
        for r in range(W):
            if mode in ("output", "both"):
                m = recv[r] + 5
                self.oi.append(torch.randperm(m, generator=g)[:recv[r]])
            else:
                m = recv[r]
                self.oi.append(None)
            self.out0.append(torch.randn(m, H, generator=g).to(dtype))

    def composition(self, g, bits, bucket, **kw):
        """index_select -> the plain kernel -> index_copy_, on the same group"""
        send = [x.to(dev()) if ix is None else x.to(dev()).index_select(0, ix.to(dev()))
                for x, ix in zip(self.xs, self.ii)]
        recv = [torch.empty(sum(self.counts[q][r] for q in range(self.W)) // self.H, self.H, dtype=self.dtype,
                            device=dev()) for r in range(self.W)]
        g.all_to_all([s.reshape(-1) for s in send], [t.reshape(-1) for t in recv], self.counts, bits=bits,
                     bucket_size=bucket, **kw)
        torch.cuda.synchronize()
        g.check()
        outs = []
        for r in range(self.W):
            if self.oi[r] is None:
                outs.append(recv[r].cpu())
            else:
                outs.append(self.out0[r].to(dev()).index_copy_(0, self.oi[r].to(dev()), recv[r]).cpu())
        return outs

    def routed(self, g, bits, bucket, **kw):
        ins = [guarded_rows(x.to(dev()), self.H) for x in self.xs]
        outs = [guarded_rows(o.to(dev()), self.H) for o in self.out0]
        iis = [None if ix is None else guarded_index(ix) for ix in self.ii]
        ois = [None if ix is None else guarded_index(ix) for ix in self.oi]
        g.all_to_all([v.reshape(-1) for _, v in ins], [v.reshape(-1) for _, v in outs], self.counts, bits=bits,
                     bucket_size=bucket, input_index=[None if t is None else t[1] for t in iis],
                     output_index=[None if t is None else t[1] for t in ois], row=self.H, **kw)
        torch.cuda.synchronize()
        g.check()
        for (buf, v), x in zip(ins, self.xs):
            assert_same(v.cpu(), x, "input modified")
            assert (buf[:GUARD_ROWS] == SENTINEL).all() and (buf[-GUARD_ROWS:] == SENTINEL).all()
        for buf, v in outs:
            assert (buf[:GUARD_ROWS] == SENTINEL).all() and (buf[-GUARD_ROWS:] == SENTINEL).all(), "guard written"
        for t, ix in zip(iis + ois, self.ii + self.oi):
            if t is not None:
                assert torch.equal(t[1].cpu(), ix) and (t[0][:3] == IX_SENTINEL).all() and (t[0][-3:] == IX_SENTINEL).all()
        return [v.cpu() for _, v in outs]


def rows_matrix(W, kind, base, seed):
    return counts(W, kind, base, seed)


def check_case(g, case, bits, bucket, what, **kw):
    got = case.routed(g, bits, bucket, **kw)
    want = case.composition(g, bits, bucket, **kw)
    for r in range(case.W):
        assert_same(got[r], want[r], f"{what}: rank {r}")
    if not kw.get("stochastic"):
        ref = O.routed_all_to_all_reference(case.xs, case.counts, case.ii, case.oi, case.H, bits=bits,
                                            bucket_size=bucket, outputs=case.out0)
        for r in range(case.W):
            assert_same(got[r].reshape(-1), ref[r], f"{what}: rank {r} vs reference")


@pytest.mark.parametrize("dtype,bits,bucket", list(itertools.product(DTYPES, R_BITS, R_BUCKETS)))
def test_routed_matches_composition(dtype, bits, bucket):
    i = DTYPES.index(dtype) * 15 + R_BITS.index(bits) * 3 + R_BUCKETS.index(bucket)
    W = R_WORLDS[i % len(R_WORLDS)]
    kind = R_SPLITS[i % len(R_SPLITS)]
    mode = R_MODES[(i // 2) % len(R_MODES)]
    H = (512, 1024, 7168)[i % 3] if bucket != 1024 else (1024, 7168)[i % 2]
    assert C.a2a_rows_fit(H, bits, bucket, DT_CODE[dtype])
    base = 6 if W <= 5 else 2
    case = Case(W, H, rows_matrix(W, kind, base, seed=i), dtype, mode, seed=i)
    check_case(make_group(W, dtype), case, bits, bucket, f"W={W} H={H} {kind} {mode}")


@pytest.mark.parametrize("world", R_WORLDS)
@pytest.mark.parametrize("mode", R_MODES)
def test_routed_every_world_and_mode(world, mode):
    rows = rows_matrix(world, "uneven", 4, seed=world)
    case = Case(world, 1024, rows, torch.bfloat16, mode, seed=world)
    check_case(make_group(world, torch.bfloat16), case, 4, 512, f"W={world} {mode}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_routed_edge_inputs(dtype):
    W, H, bucket = 3, 1024, 64
    n = 6 * H
    xs, _ = edge_inputs(dtype, n * W, bucket, seed=2, world=W, bits=4)
    case = Case(W, H, [[6] * W for _ in range(W)], dtype, "both", seed=5, topk=False)
    # the edge values as the physical inputs, indices a permutation of them
    case.xs = [torch.cat([x.reshape(-1, H), x.reshape(-1, H)[:3]]) for x in xs]
    check_case(make_group(W, dtype), case, 4, bucket, "edge")


def test_rows_that_do_not_fit_are_refused_by_the_kernel():
    W = 2
    for H, bucket in [(100, 1024), (640, 1024)]:
        case = Case(W, H, [[3, 4], [5, 6]], torch.float32, "both", seed=H)
        with pytest.raises(ValueError, match="quantization items"):
            case.routed(make_group(W, torch.float32), 4, bucket)


@pytest.mark.parametrize("bits,bucket", [(8, 512), (4, 1024), (32, 512)])
def test_routed_small_slots_many_windows(bits, bucket):
    W, lanes, dtype, H = 4, 2, torch.bfloat16, 1024
    block = C.a2a_windows(1, bits, bucket, DT_CODE[dtype], 1 << 20, 1)["block_wire"]
    slot = ((2 * lanes * block + 16 * lanes) + 255) // 256 * 256
    g = make_group(W, dtype, slot=slot, lanes=lanes)
    rows = [[0, 9, 70, 120], [8, 0, 1, 0], [50, 0, 33, 17], [0, 200, 5, 7]]
    for q in range(W):
        rows[q][q] = 10 * q
    w = C.a2a_windows(200 * H, bits, bucket, DT_CODE[dtype], slot, lanes)
    assert len(w["lanes"][0]) > 3
    check_case(g, Case(W, H, rows, dtype, "both", seed=7), bits, bucket, "small slots")


def test_routed_stochastic_matches_composition():
    W, dtype = 3, torch.float32
    g = make_group(W, dtype)
    case = Case(W, 512, rows_matrix(W, "uneven", 6, seed=3), dtype, "both", seed=3)
    a = case.routed(g, 3, 64, stochastic=True, seed=11, seq=1)
    want = case.composition(g, 3, 64, stochastic=True, seed=11, seq=1)
    for r in range(W):
        assert_same(a[r], want[r], f"stochastic rank {r}")
    b = case.routed(g, 3, 64, stochastic=True, seed=11, seq=2)
    assert any(not torch.equal(a[r], b[r]) for r in range(W) if a[r].numel())


def test_routed_and_plain_calls_interleaved():
    W, dtype = 4, torch.float16
    g = make_group(W, dtype)
    for it in range(3):
        case = Case(W, 1024, rows_matrix(W, "uneven", 5, seed=it), dtype, R_MODES[it], seed=it)
        check_case(g, case, 4, 512, f"routed {it}")
        plain = Case(W, 1024, rows_matrix(W, "uneven", 5, seed=10 + it), dtype, "none", seed=10 + it)
        check_case(g, plain, 8, 1024, f"plain {it}")


@pytest.mark.parametrize("which,bad", [("input", "past"), ("input", "neg"), ("output", "past"), ("output", "neg")])
@pytest.mark.parametrize("bits", [4, 32])
def test_bad_index_is_reported_and_never_dereferenced(which, bad, bits):
    """An index naming the row just past its view (a guard row of the same allocation) or row -1:
    the call completes, the status names the index, and no guard row is read or written."""
    W, H, dtype = 2, 512, torch.float32
    g = make_group(W, dtype)
    case = Case(W, H, [[3, 4], [5, 6]], dtype, "both", seed=bits)
    pick = case.ii if which == "input" else case.oi
    rows = case.xs[0].shape[0] if which == "input" else case.out0[0].shape[0]
    pick[0] = pick[0].clone()
    pick[0][1] = rows if bad == "past" else -1
    with pytest.raises(RuntimeError, match=f"{which}_index"):
        case.routed(g, bits, 512)
    assert f"{which}_index" in g.status(0) and g.status(1) == ""
    g.clear()


def _bad_index_guards(which, bits):
    W, H, dtype = 2, 512, torch.float32
    g = make_group(W, dtype)
    case = Case(W, H, [[3, 4], [5, 6]], dtype, "both", seed=bits)
    ins = [guarded_rows(x.to(dev()), H) for x in case.xs]
    outs = [guarded_rows(o.to(dev()), H) for o in case.out0]
    ii = [ix.clone().to(dev()) for ix in case.ii]
    oi = [ix.clone().to(dev()) for ix in case.oi]
    if which == "input":
        ii[0][0] = case.xs[0].shape[0]
    else:
        oi[0][0] = case.out0[0].shape[0]
    g.all_to_all([v.reshape(-1) for _, v in ins], [v.reshape(-1) for _, v in outs], case.counts, bits=bits,
                 bucket_size=512, input_index=ii, output_index=oi, row=H)
    torch.cuda.synchronize()
    msg = g.status(0)
    g.clear()
    return ins, outs, msg


@pytest.mark.parametrize("which", ["input", "output"])
def test_bad_index_touches_no_guard_row(which):
    ins, outs, msg = _bad_index_guards(which, 32)
    assert f"{which}_index" in msg
    for buf, v in ins + outs:
        assert (buf[:GUARD_ROWS] == SENTINEL).all() and (buf[-GUARD_ROWS:] == SENTINEL).all(), "guard written"
    for buf, v in outs:
        assert not (v == SENTINEL).any(), "a guard row was read into the output"


# ---- the public API at world 1 ---------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        for dtype, H, bucket in [(torch.bfloat16, 1024, 512), (torch.float32, 7168, 1024), (torch.float16, 100, 1024),
                                 (torch.float32, 640, 1024)]:
            x = torch.randn(40, H, device="cuda", generator=g).to(dtype)
            ii = torch.randint(0, 40, (70,), device="cuda", generator=g)
            oi = torch.randperm(80, device="cuda", generator=g)[:70]
            out = torch.full((80, H), SENTINEL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, x, [70], [70], bits=4, bucket_size=bucket, input_index=ii, output_index=oi)
            recv = torch.empty(70, H, dtype=dtype, device="cuda")
            cgx.all_to_all_single(recv, x.index_select(0, ii), [70], [70], bits=4, bucket_size=bucket)
            want = torch.full_like(out, SENTINEL).index_copy_(0, oi, recv)
            assert_same(out, want, f"{dtype} H={H}")
            # equal splits divide the index entries
            out2 = torch.empty(70, H, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out2, x, bits=4, bucket_size=bucket, input_index=ii)
            assert_same(out2, recv, f"{dtype} H={H} equal splits")
        x = torch.randn(10, 8, device="cuda")
        with pytest.raises(RuntimeError, match="entries"):
            cgx.all_to_all_single(torch.empty(10, 8, device="cuda"), x, [10], [10],
                                  input_index=torch.arange(9, device="cuda"))
        with pytest.raises(RuntimeError, match="int64"):
            cgx.all_to_all_single(torch.empty(10, 8, device="cuda"), x, input_index=torch.arange(10, device="cuda").int())
        with pytest.raises(RuntimeError, match="device"):
            cgx.all_to_all_single(torch.empty(10, 8, device="cuda"), x, input_index=torch.arange(10))
        with pytest.raises(RuntimeError, match="contiguous"):
            cgx.all_to_all_single(torch.empty(10, 8, device="cuda"), x,
                                  output_index=torch.arange(20, device="cuda")[::2])
        # the differentiable form against autograd through the composition
        torch.use_deterministic_algorithms(True)
        try:
            xa = torch.randn(30, 1024, device="cuda", requires_grad=True)
            ii = torch.randint(0, 30, (60,), device="cuda", generator=g)
            oi = torch.randperm(64, device="cuda", generator=g)[:60]
            y = cgx.differentiable_all_to_all_single(xa, [60], [60], bits=8, grad_bits=4, input_index=ii,
                                                     output_index=oi, output_rows=64)
            w = torch.randn(64, 1024, device="cuda", generator=g)
            (y * w).sum().backward()
            xb = xa.detach().clone().requires_grad_()
            mid = cgx.differentiable_all_to_all_single(xb.index_select(0, ii), [60], [60], bits=8, grad_bits=4)
            yb = torch.zeros(64, 1024, device="cuda").index_copy(0, oi, mid)
            (yb * w).sum().backward()
            assert_same(y.detach(), yb.detach(), "differentiable forward")
            assert_same(xa.grad, xb.grad, "differentiable backward")
        finally:
            torch.use_deterministic_algorithms(False)
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def _graph_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        H, n = 1024, 500
        x = torch.randn(300, H, device="cuda")
        ii = torch.randint(0, 300, (n,), device="cuda")
        oi = torch.randperm(n + 10, device="cuda")[:n]
        out = torch.zeros(n + 10, H, device="cuda")
        cgx.all_to_all_single(out, x, [n], [n], bits=4, input_index=ii, output_index=oi)  # initialise
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            cgx.all_to_all_single(out, x, [n], [n], bits=4, input_index=ii, output_index=oi)
        for it in range(3):
            x.copy_(torch.randn(300, H, device="cuda"))
            ii.copy_(torch.randint(0, 300, (n,), device="cuda"))
            oi.copy_(torch.randperm(n + 10, device="cuda")[:n])
            out.zero_()
            graph.replay()
            torch.cuda.synchronize()
            recv = torch.empty(n, H, device="cuda")
            cgx.all_to_all_single(recv, x.index_select(0, ii), [n], [n], bits=4)
            assert_same(out, torch.zeros_like(out).index_copy_(0, oi, recv), f"replay {it}")
    finally:
        dist.destroy_process_group()


def test_cuda_graph_world1():
    spawn(_graph_world1, 1)


# ---- several GPUs ------------------------------------------------------------------------------
def _pg_routed(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for it, (dtype, bits, bucket, H, mode) in enumerate([
                (torch.bfloat16, 8, 512, 1024, "both"), (torch.float32, 4, 1024, 7168, "input"),
                (torch.float16, 3, 64, 512, "output"), (torch.float32, 32, 512, 512, "both"),
                (torch.float32, 4, 1024, 640, "both")]):
            case = Case(world, H, rows_matrix(world, "uneven", 6, seed=it), dtype, mode, seed=it)
            ref = O.routed_all_to_all_reference(case.xs, case.counts, case.ii, case.oi, H, bits=bits,
                                                bucket_size=bucket, outputs=case.out0)[rank]
            out = case.out0[rank].cuda()
            ii, oi = case.ii[rank], case.oi[rank]
            cgx.all_to_all_single(out, case.xs[rank].cuda(), [case.rows[q][rank] for q in range(world)],
                                  case.rows[rank], bits=bits, bucket_size=bucket,
                                  input_index=None if ii is None else ii.cuda(),
                                  output_index=None if oi is None else oi.cuda())
            assert_same(out.cpu().reshape(-1), ref, f"{transport} {dtype} bits={bits} H={H} {mode}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
def test_public_api_routed_matches_reference(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_routed, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport}, timeout=600)


def _moe_top2(rank, world):
    """Top-2 routing, one expert per rank, dispatched and combined with router indices (no manual
    permutation), forward and backward bitwise against autograd through the composition."""
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

        def layer(x, routed):
            if routed:
                tok = cgx.differentiable_all_to_all_single(x, recv, send[rank], bits=8, grad_bits=8, input_index=ii)
                y = tok @ w
                return cgx.differentiable_all_to_all_single(y, send[rank], recv, bits=8, grad_bits=8,
                                                            output_index=oi, output_rows=T * k)
            tok = cgx.differentiable_all_to_all_single(x.index_select(0, ii), recv, send[rank], bits=8, grad_bits=8)
            y = tok @ w
            back = cgx.differentiable_all_to_all_single(y, send[rank], recv, bits=8, grad_bits=8)
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
    finally:
        torch.use_deterministic_algorithms(False)
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_moe_top2_routed_forward_backward():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    spawn(_moe_top2, 2, env={"CUBLAS_WORKSPACE_CONFIG": ":4096:8"}, timeout=600)
