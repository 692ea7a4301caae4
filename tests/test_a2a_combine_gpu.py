"""The weighted top-k combine (DESIGN §2.13d) on one H100 with W virtual ranks (C.LocalSraGroup for
the fused kernel, C.LocalReducerGroup for the composed path), bit for bit against the oracle's
composition, NaN-aware: dtypes x widths x buckets, worlds x k x row lengths, the slots against the
plain routed call, the composed path against the fused one, the edge inputs, stochastic rounding,
small slots with many windows, combine / plain / routed / codes calls on one heap, a repeated slot
and an index out of range; and the public API at world 1 (eager, async, differentiable, and in a
CUDA graph replayed with new indices and gates)."""
import itertools

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
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BITS = (2, 4, 8, 32, "e4m3", "e5m2")


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, 256)


class Case:
    """Each of W ranks combines T tokens of k choices; rows[q][r] of rank r's T * k slots come from
    rank q, rank q sends sum_r rows[q][r] rows, and rank r's output_index is a permutation."""

    def __init__(self, W, T, k, H, dtype, seed, xs=None):
        g = torch.Generator().manual_seed(seed)
        self.W, self.T, self.k, self.H, self.dtype = W, T, k, H, dtype
        rows = [[0] * W for _ in range(W)]
        for r in range(W):
            src = torch.randint(0, W, (T * k,), generator=g)
            for q in range(W):
                rows[q][r] = int((src == q).sum())
        self.counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        self.xs = xs or [(torch.randn(sum(rows[q]), H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype)
                         for q in range(W)]
        self.oi = [torch.randperm(T * k, generator=g) for _ in range(W)]
        self.gates = [torch.rand(T, k, generator=g) * 2 - 0.5 for _ in range(W)]

    def run(self, grp, bits, bucket, reducer=False, **kw):
        """(slots, outputs) of the combine call, flat, on the CPU"""
        slots = [torch.zeros(self.T * self.k * self.H, dtype=self.dtype, device=dev()) for _ in range(self.W)]
        outs = [torch.full((self.T * self.H,), -3.0, dtype=self.dtype, device=dev()) for _ in range(self.W)]
        common = dict(bits=bits, bucket_size=bucket, output_index=[ix.to(dev()) for ix in self.oi], row=self.H,
                      gate=[gt.to(dev()) for gt in self.gates], combine_out=outs, **kw)
        grp.all_to_all([x.to(dev()).reshape(-1) for x in self.xs], slots, self.counts, **common)
        torch.cuda.synchronize()
        if not reducer:
            grp.check()
        return [s.cpu() for s in slots], [o.cpu() for o in outs]

    def reference(self, bits, bucket):
        return O.routed_all_to_all_combine_reference([x.reshape(-1) for x in self.xs], self.counts, self.oi,
                                                     self.gates, self.H, bits=bits, bucket_size=bucket)


def check(case, got, want, what):
    for r in range(case.W):
        assert_same(got[0][r], want[0][r], f"{what} slots rank {r}")
        assert_same(got[1][r], want[1][r], f"{what} output rank {r}")


@pytest.mark.parametrize("dtype,bits,bucket", list(itertools.product(DTYPES, BITS, (512, 1024))))
def test_fused_matches_oracle(dtype, bits, bucket):
    case = Case(8, 6, 8, 7168, dtype, seed=hash((str(dtype), str(bits), bucket)) % 1000)
    check(case, case.run(make_group(8, dtype), bits, bucket), case.reference(bits, bucket), f"{dtype} {bits} {bucket}")


@pytest.mark.parametrize("world,k,H", [(w, k, H) for w, k, H in itertools.product((1, 2, 3, 8), (1, 2, 8), (1024, 7168))
                                       if not (w == 8 and H == 1024 and k == 1)])
def test_fused_worlds_and_k(world, k, H):
    case = Case(world, 10, k, H, torch.bfloat16, seed=world * 100 + k * 10 + H % 7)
    check(case, case.run(make_group(world, torch.bfloat16), 4, 512), case.reference(4, 512), f"W{world} k{k} H{H}")


def test_k32_and_few_tokens():
    case = Case(3, 2, 32, 1024, torch.float16, seed=5)
    check(case, case.run(make_group(3, torch.float16), 8, 1024), case.reference(8, 1024), "k32")


def test_slots_equal_the_routed_call():
    case = Case(4, 12, 4, 2048, torch.bfloat16, seed=11)
    grp = make_group(4, torch.bfloat16)
    slots, _ = case.run(grp, 4, 512)
    plain = [torch.zeros(case.T * case.k * case.H, dtype=case.dtype, device=dev()) for _ in range(4)]
    grp.all_to_all([x.to(dev()).reshape(-1) for x in case.xs], plain, case.counts, bits=4, bucket_size=512,
                   output_index=[ix.to(dev()) for ix in case.oi], row=case.H)
    torch.cuda.synchronize()
    grp.check()
    for r in range(4):
        assert_same(slots[r], plain[r].cpu(), f"rank {r}")


@pytest.mark.parametrize("H,bucket,bits", [(2048, 512, 4), (7168, 1024, "e4m3"), (640, 1024, 4), (1000, 100, 8)])
def test_composed_path_matches(H, bucket, bits):
    # the process group's composed path: the generic reducer, index_copy_ into the slots, combine_rows_kernel
    case = Case(3, 7, 4, H, torch.bfloat16, seed=H)
    red = C.LocalReducerGroup(3, "SRA")
    got = case.run(red, bits, bucket, reducer=True)
    want = case.reference(bits, bucket)
    check(case, got, want, f"composed H={H}")
    if C.a2a_rows_fit(H, bits if isinstance(bits, int) else 8, bucket, DT_CODE[case.dtype]):
        check(case, case.run(make_group(3, torch.bfloat16), bits, bucket), got, f"fused H={H}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_edge_inputs(dtype):
    W, T, k, H = 4, 8, 4, 1024
    probe = Case(W, T, k, H, dtype, seed=3)
    sizes = [sum(probe.counts[q]) for q in range(W)]
    ins, _ = edge_inputs(dtype, max(sizes), 512, seed=4, world=W, bits=4)
    xs = [ins[q][:sizes[q]].reshape(-1, H) for q in range(W)]
    case = Case(W, T, k, H, dtype, seed=3, xs=xs)
    case.gates[0][0, 0] = float("nan")
    case.gates[1][1, :] = -0.0
    case.gates[2][2, 1] = float("inf")
    for bits in (4, 32, "e5m2"):
        check(case, case.run(make_group(W, dtype), bits, 512), case.reference(bits, 512), f"edge {bits}")


def test_stochastic_matches_composition():
    case = Case(4, 9, 2, 1024, torch.bfloat16, seed=21)
    grp = make_group(4, torch.bfloat16)
    kw = dict(stochastic=True, seed=77, seq=5)
    slots, outs = case.run(grp, 3, 512, **kw)
    plain = [torch.zeros(case.T * case.k * case.H, dtype=case.dtype, device=dev()) for _ in range(4)]
    grp.all_to_all([x.to(dev()).reshape(-1) for x in case.xs], plain, case.counts, bits=3, bucket_size=512,
                   output_index=[ix.to(dev()) for ix in case.oi], row=case.H, **kw)
    torch.cuda.synchronize()
    grp.check()
    for r in range(4):
        assert_same(slots[r], plain[r].cpu(), f"slots rank {r}")
        assert_same(outs[r], O.combine_rows_reference(plain[r].cpu().reshape(-1, case.H), case.gates[r]).reshape(-1),
                    f"output rank {r}")


@pytest.mark.parametrize("bits,bucket", [(4, 512), (32, 512), ("e4m3", 1024)])
def test_small_slots_many_windows(bits, bucket):
    case = Case(3, 24, 4, 2048, torch.float16, seed=8)
    grp = C.LocalSraGroup(3, 2, 64 << 10, 5000, 256)
    check(case, case.run(grp, bits, bucket), case.reference(bits, bucket), "small slots")


def test_interleaved_on_one_heap():
    W, dtype = 4, torch.bfloat16
    grp = make_group(W, dtype)
    case = Case(W, 8, 4, 1024, dtype, seed=31)
    want = case.reference(4, 512)
    n = 4096
    xs = [torch.randn(W * n, device=dev()).to(dtype) for _ in range(W)]
    counts = [[n] * W for _ in range(W)]
    for it in range(2):
        check(case, case.run(grp, 4, 512), want, f"combine {it}")
        outs = [torch.empty(W * n, dtype=dtype, device=dev()) for _ in range(W)]
        grp.all_to_all(xs, outs, counts, bits=4, bucket_size=512)
        codes = [torch.empty(W * n, dtype=torch.float8_e4m3fn, device=dev()) for _ in range(W)]
        scales = [torch.empty(W * n // 512, device=dev()) for _ in range(W)]
        grp.all_to_all(xs, codes, counts, bits="e4m3", bucket_size=512, output_scales=scales)
        routed = [torch.empty(W * n, dtype=dtype, device=dev()) for _ in range(W)]
        grp.all_to_all(xs, routed, counts, bits=4, bucket_size=512, row=512,
                       output_index=[torch.randperm(W * n // 512, device=dev()) for _ in range(W)])
        torch.cuda.synchronize()
        grp.check()
        ref = O.all_to_all_reference([x.cpu() for x in xs], counts, bits=4, bucket_size=512)
        for r in range(W):
            assert_same(outs[r].cpu(), ref[r], f"plain {it} rank {r}")


@pytest.mark.parametrize("kind", ("repeat", "range"))
def test_bad_index_is_reported(kind):
    case = Case(2, 4, 2, 1024, torch.float32, seed=41)
    bad = case.oi[1].clone()
    if kind == "repeat":
        bad[1] = bad[0]
    else:
        bad[0] = case.T * case.k
    case.oi[1] = bad
    grp = make_group(2, torch.float32)
    with pytest.raises(RuntimeError, match="output_index"):
        case.run(grp, 4, 512)
    msg = grp.status(1)
    assert "output_index" in msg and (("repeats a slot" in msg) == (kind == "repeat")), msg
    assert grp.status(0) == ""


def test_binding_refusals():
    case = Case(2, 4, 2, 1024, torch.float32, seed=2)
    grp = make_group(2, torch.float32)
    with pytest.raises(ValueError, match="codes output"):
        case.run(grp, "e4m3", 512, output_scales=[torch.empty(8 * 2, device=dev()) for _ in range(2)])
    case.gates = [torch.rand(1, 33) for _ in range(2)]
    with pytest.raises(ValueError, match="1..32"):
        case.run(grp, 4, 512)


# ---- the public API at world 1 -------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        for dtype, H, bucket, bits, k in [(torch.bfloat16, 1024, 512, 4, 2), (torch.float32, 7168, 1024, "e4m3", 8),
                                          (torch.float16, 640, 1024, 4, 3), (torch.bfloat16, 2048, 512, 32, 1)]:
            T = 37
            x = torch.randn(T * k, H, device="cuda", generator=g).to(dtype)
            oi = torch.randperm(T * k, device="cuda", generator=g)
            gate = torch.rand(T, k, device="cuda", generator=g)
            out = torch.empty(T, H, dtype=dtype, device="cuda")
            slots = torch.empty(T * k, H, dtype=dtype, device="cuda")
            cgx.all_to_all_combine(out, x, gate, oi, bits=bits, bucket_size=bucket, slots=slots)
            plain = torch.zeros(T * k, H, dtype=dtype, device="cuda")
            cgx.all_to_all_single(plain, x, bits=bits, bucket_size=bucket, output_index=oi)
            assert_same(slots, plain, f"slots {dtype} H={H}")
            assert_same(out, O.combine_rows_reference(plain.cpu(), gate.cpu()), f"combine {dtype} H={H}")
            out2 = torch.empty_like(out)
            work = cgx.all_to_all_combine(out2, x, gate, oi, bits=bits, bucket_size=bucket, async_op=True)
            work.wait()
            assert_same(out2, out, f"async {dtype} H={H}")
        with pytest.raises(ValueError, match="at most 32"):
            cgx.all_to_all_combine(torch.empty(1, 8, device="cuda"), torch.randn(33, 8, device="cuda"),
                                   torch.rand(1, 33, device="cuda"), torch.arange(33, device="cuda"))
        # the differentiable form against torch on the same slots
        T, k, H = 20, 4, 1024
        xa = torch.randn(T * k, H, device="cuda", generator=g, requires_grad=True)
        ga = torch.rand(T, k, device="cuda", generator=g, requires_grad=True)
        oi = torch.randperm(T * k, device="cuda", generator=g)
        y = cgx.differentiable_all_to_all_combine(xa, ga, oi, bits=8, grad_bits=32)
        w = torch.randn(T, H, device="cuda", generator=g)
        (y * w).sum().backward()
        slots = torch.zeros(T * k, H, device="cuda")
        cgx.all_to_all_single(slots, xa.detach(), bits=8, output_index=oi)
        assert_same(y.detach(), O.combine_rows_reference(slots.cpu(), ga.detach().cpu()).cuda(), "forward")
        want_gx = (w.unsqueeze(1) * ga.detach().unsqueeze(-1)).reshape(T * k, H).index_select(0, oi)
        assert_same(xa.grad, want_gx, "input gradient")
        want_gg = (w.unsqueeze(1) * slots.reshape(T, k, H)).sum(-1)
        assert_same(ga.grad, want_gg, "gate gradient")
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def _graph_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, k, H = 300, 8, 1024
        x = torch.randn(T * k, H, device="cuda", dtype=torch.bfloat16)
        oi = torch.randperm(T * k, device="cuda")
        gate = torch.rand(T, k, device="cuda")
        out = torch.zeros(T, H, device="cuda", dtype=torch.bfloat16)
        cgx.all_to_all_combine(out, x, gate, oi, bits=4)  # initialise
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            cgx.all_to_all_combine(out, x, gate, oi, bits=4)
        for it in range(3):
            x.copy_(torch.randn(T * k, H, device="cuda"))
            oi.copy_(torch.randperm(T * k, device="cuda"))
            gate.copy_(torch.rand(T, k, device="cuda"))
            out.zero_()
            graph.replay()
            torch.cuda.synchronize()
            slots = torch.zeros(T * k, H, device="cuda", dtype=torch.bfloat16)
            cgx.all_to_all_single(slots, x, bits=4, output_index=oi)
            assert_same(out, O.combine_rows_reference(slots.cpu(), gate.cpu()), f"replay {it}")
    finally:
        dist.destroy_process_group()


def test_cuda_graph_world1():
    spawn(_graph_world1, 1)


# ---- several GPUs ------------------------------------------------------------------------------
def _pg_multi(rank, world):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, k, H = 64, 2, 2048
        g = torch.Generator().manual_seed(5)
        xs = [torch.randn(T * k, H, generator=g).to(torch.bfloat16) for _ in range(world)]
        ois = [torch.randperm(T * k, generator=g) for _ in range(world)]
        gates = [torch.rand(T, k, generator=g) for _ in range(world)]
        per = T * k // world
        counts = [[per * H] * world for _ in range(world)]
        out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
        cgx.all_to_all_combine(out, xs[rank].cuda(), gates[rank].cuda(), ois[rank].cuda(), bits=4)
        _, want = O.routed_all_to_all_combine_reference([x.reshape(-1) for x in xs], counts, ois, gates, H, bits=4,
                                                        bucket_size=512)
        assert_same(out.reshape(-1), want[rank].cuda(), f"rank {rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", (2, 4))
def test_public_api_multi_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_multi, world)
