"""The backward of the MoE dispatch (DESIGN §2.13i) on one H100 with W virtual ranks: the unit-gate
combine with the slot index as its output index, through C.LocalSraGroup (the fused kernel) and
C.LocalReducerGroup (the composed path), bit for bit against ``oracle.dispatch_backward_reference``,
NaN-aware: dtypes x widths, worlds x k x row lengths, with and without the forward's output index
(the combine's input_index), the edge inputs, stochastic rounding and a repeated slot; and the
public API at world 1 (forward, backward, determinism, the index_add_ backward, -0, a repeated slot
and a CUDA graph)."""
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
BITS = (2, 4, 8, 32, "e4m3", "e5m2", "e4m3_pow2", "e5m2_sr")
SEED, SEQ = 0x5EED, 7


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, 256)


class Case:
    """The gradient exchange of a dispatch backward: rank r owns T tokens of k choices and its slot
    index is a permutation of [0, T * k); rank q returns rows[q][r] gradient rows to rank r. With
    ``indexed`` rank q's gradient has 3 rows more than it returns and input_index picks them (the
    forward's output_index)."""

    def __init__(self, W, T, k, H, dtype, seed, indexed=False, xs=None):
        g = torch.Generator().manual_seed(seed)
        self.W, self.T, self.k, self.H, self.dtype = W, T, k, H, dtype
        rows = [[0] * W for _ in range(W)]
        for r in range(W):
            src = torch.randint(0, W, (T * k,), generator=g)
            for q in range(W):
                rows[q][r] = int((src == q).sum())
        self.counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        n = [sum(rows[q]) for q in range(W)]
        extra = 3 if indexed else 0
        self.xs = xs or [(torch.randn(n[q] + extra, H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype)
                         for q in range(W)]
        self.ii = [torch.randperm(n[q] + extra, generator=g)[:n[q]] for q in range(W)] if indexed else None
        self.si = [torch.randperm(T * k, generator=g) for _ in range(W)]

    def run(self, grp, bits, bucket, reducer=False, **kw):
        """(slots, gradients) of the unit-gate combine, flat, on the CPU"""
        slots = [torch.zeros(self.T * self.k * self.H, dtype=self.dtype, device=dev()) for _ in range(self.W)]
        outs = [torch.full((self.T * self.H,), -3.0, dtype=self.dtype, device=dev()) for _ in range(self.W)]
        if self.ii is not None:
            kw["input_index"] = [ix.to(dev()) for ix in self.ii]
        grp.all_to_all([x.to(dev()).reshape(-1) for x in self.xs], slots, self.counts, bits=bits, bucket_size=bucket,
                       output_index=[ix.to(dev()) for ix in self.si], row=self.H,
                       gate=[torch.ones(self.T, self.k, device=dev()) for _ in range(self.W)], combine_out=outs, **kw)
        torch.cuda.synchronize()
        if not reducer:
            grp.check()
        return [s.cpu() for s in slots], [o.cpu() for o in outs]

    def reference(self, bits, bucket, seed=0, seq=0):
        return O.dispatch_backward_reference([x.reshape(-1) for x in self.xs], self.counts, self.si, self.k, self.H,
                                             bits=bits, bucket_size=bucket, input_index=self.ii, seed=seed, seq=seq)


def check(case, got, want, what):
    for r in range(case.W):
        assert_same(got[0][r], want[0][r], f"{what} slots rank {r}")
        assert_same(got[1][r], want[1][r], f"{what} gradient rank {r}")


@pytest.mark.parametrize("indexed", (False, True), ids=("plain", "indexed"))
@pytest.mark.parametrize("dtype,bits", list(itertools.product(DTYPES, BITS)))
def test_fused_matches_oracle(dtype, bits, indexed):
    case = Case(8, 6, 8, 7168, dtype, seed=hash((str(dtype), str(bits), indexed)) % 1000, indexed=indexed)
    kw = dict(seed=SEED, seq=SEQ)
    check(case, case.run(make_group(8, dtype), bits, 512, **kw), case.reference(bits, 512, **kw), f"{dtype} {bits}")


# W = 8, H = 1024, k = 1 is left out as in test_a2a_combine_gpu.py
@pytest.mark.parametrize("world,k,H,indexed",
                         [(w, k, H, ix) for w, k, H, ix in itertools.product((1, 2, 3, 8), (1, 2, 8, 32), (1024, 7168),
                                                                             (False, True))
                          if not (w == 8 and H == 1024 and k == 1)])
def test_fused_worlds_and_k(world, k, H, indexed):
    T = 2 if k == 32 else 10
    case = Case(world, T, k, H, torch.bfloat16, seed=world * 100 + k * 10 + H % 7, indexed=indexed)
    check(case, case.run(make_group(world, torch.bfloat16), 4, 512), case.reference(4, 512), f"W{world} k{k} H{H}")


@pytest.mark.parametrize("dtype,bits", list(itertools.product(DTYPES, BITS)))
def test_composed_matches_oracle(dtype, bits):
    # rows of 1000 elements in buckets of 100 do not hold whole quantization items: the composed path
    case = Case(3, 7, 4, 1000, dtype, seed=17, indexed=True)
    kw = dict(seed=SEED, seq=SEQ)
    check(case, case.run(C.LocalReducerGroup(3, "SRA"), bits, 100, reducer=True, **kw),
          case.reference(bits, 100, **kw), f"composed {dtype} {bits}")


@pytest.mark.parametrize("indexed", (False, True), ids=("plain", "indexed"))
@pytest.mark.parametrize("H,bucket,bits,k", [(1024, 512, 4, 2), (7168, 1024, "e4m3", 8), (640, 100, 4, 32),
                                             (1000, 100, 8, 1)])
def test_composed_path_matches(H, bucket, bits, k, indexed):
    case = Case(3, 2 if k == 32 else 7, k, H, torch.bfloat16, seed=H + k, indexed=indexed)
    got = case.run(C.LocalReducerGroup(3, "SRA"), bits, bucket, reducer=True)
    check(case, got, case.reference(bits, bucket), f"composed H={H}")
    if C.a2a_rows_fit(H, bits if isinstance(bits, int) else 8, bucket, DT_CODE[case.dtype]):
        check(case, case.run(make_group(3, torch.bfloat16), bits, bucket), got, f"fused H={H}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_edge_inputs(dtype):
    W, T, k, H = 4, 8, 4, 1024
    probe = Case(W, T, k, H, dtype, seed=3, indexed=True)
    sizes = [x.numel() for x in probe.xs]
    ins, _ = edge_inputs(dtype, max(sizes), 512, seed=4, world=W, bits=4)
    case = Case(W, T, k, H, dtype, seed=3, indexed=True, xs=[ins[q][:sizes[q]].reshape(-1, H) for q in range(W)])
    for bits in (4, 32, "e5m2"):
        fused = case.run(make_group(W, dtype), bits, 512)
        check(case, fused, case.reference(bits, 512), f"edge {bits}")
        check(case, case.run(C.LocalReducerGroup(W, "SRA"), bits, 512, reducer=True), fused, f"edge composed {bits}")


def test_stochastic_matches_composition():
    case = Case(4, 9, 2, 1024, torch.bfloat16, seed=21, indexed=True)
    grp = make_group(4, torch.bfloat16)
    kw = dict(stochastic=True, seed=77, seq=5)
    slots, outs = case.run(grp, 4, 512, **kw)
    plain = [torch.zeros(case.T * case.k * case.H, dtype=case.dtype, device=dev()) for _ in range(4)]
    grp.all_to_all([x.to(dev()).reshape(-1) for x in case.xs], plain, case.counts, bits=4, bucket_size=512,
                   input_index=[ix.to(dev()) for ix in case.ii], output_index=[ix.to(dev()) for ix in case.si],
                   row=case.H, **kw)
    torch.cuda.synchronize()
    grp.check()
    for r in range(4):
        assert_same(slots[r], plain[r].cpu(), f"slots rank {r}")
        assert_same(outs[r], O.dispatch_sum_reference(plain[r].cpu().reshape(-1, case.H), case.k).reshape(-1),
                    f"gradient rank {r}")


def test_repeated_slot_is_reported():
    case = Case(2, 4, 2, 1024, torch.float32, seed=41, indexed=True)
    bad = case.si[1].clone()
    bad[1] = bad[0]
    case.si[1] = bad
    grp = make_group(2, torch.float32)
    with pytest.raises(RuntimeError, match="output_index"):
        case.run(grp, 4, 512)
    assert "repeats a slot" in grp.status(1), grp.status(1)
    assert grp.status(0) == ""


# ---- the public API at world 1 -------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        for dtype, H, bucket, bits, gb, k, indexed in [
                (torch.bfloat16, 1024, 512, 4, "e5m2", 2, False), (torch.float32, 7168, 1024, "e4m3", 8, 8, True),
                (torch.float16, 640, 1024, 4, 4, 3, True), (torch.bfloat16, 2048, 512, 32, 32, 32, False),
                (torch.bfloat16, 1000, 100, 8, 8, 4, True)]:
            T = 3 if k == 32 else 37
            x = torch.randn(T, H, device="cuda", generator=g).to(dtype)
            si = torch.randperm(T * k, device="cuda", generator=g)
            kw = dict(bits=bits, grad_bits=gb, bucket_size=bucket)
            if indexed:
                kw.update(output_index=torch.randperm(T * k + 5, device="cuda", generator=g)[:T * k],
                          output_rows=T * k + 5)
            xa = x.clone().requires_grad_(True)
            y = cgx.differentiable_all_to_all_dispatch(xa, si, **kw)
            xb = x.clone().requires_grad_(True)
            want_y = cgx.differentiable_all_to_all_single(xb, input_index=torch.div(si, k, rounding_mode="floor"), **kw)
            assert_same(y.detach(), want_y.detach(), f"forward {dtype} H={H}")
            w = torch.randn(y.shape, device="cuda", generator=g).to(dtype)
            y.backward(w)
            oi = kw.get("output_index")
            _, want = O.dispatch_backward_reference([w.reshape(-1)], [[T * k * H]], [si], k, H, bits=gb,
                                                    bucket_size=bucket, input_index=None if oi is None else [oi])
            assert_same(xa.grad.reshape(-1), want[0].cuda(), f"backward {dtype} H={H}")
            first = xa.grad.clone()
            xa.grad = None
            cgx.differentiable_all_to_all_dispatch(xa, si, **kw).backward(w)
            assert_same(xa.grad, first, f"second backward {dtype} H={H}")
        # fp32 at 32 bits and k = 2: two adds commute, so the index_add_ backward gives the same bits
        T, k, H = 50, 2, 1024
        x = torch.randn(T, H, device="cuda", generator=g)
        si = torch.randperm(T * k, device="cuda", generator=g)
        w = torch.randn(T * k, H, device="cuda", generator=g)
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        cgx.differentiable_all_to_all_dispatch(xa, si, bits=32).backward(w)
        cgx.differentiable_all_to_all_single(xb, input_index=si // k, bits=32).backward(w)
        assert_same(xa.grad, xb.grad, "index_add_")
        # a token whose k gradients are all -0 gets -0, where index_add_ (from +0) gives +0
        w = torch.randn(T * k, H, device="cuda", generator=g).to(torch.bfloat16)
        w[(si // k) == 0] = -0.0
        xa = x.to(torch.bfloat16).requires_grad_(True)
        cgx.differentiable_all_to_all_dispatch(xa, si, bits=32).backward(w)
        assert torch.equal(xa.grad[0].view(torch.int16), torch.full((H,), -0.0, dtype=torch.bfloat16,
                                                                    device="cuda").view(torch.int16))
        xb = x.to(torch.bfloat16).requires_grad_(True)
        cgx.differentiable_all_to_all_single(xb, input_index=si // k, bits=32).backward(w)
        assert not torch.signbit(xb.grad[0]).any()
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def _repeat_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, k, H = 8, 2, 1024
        si = torch.randperm(T * k, device="cuda")
        si[1] = si[0]
        xa = torch.randn(T, H, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        y = cgx.differentiable_all_to_all_dispatch(xa, si, bits=4)
        # the kernel reports the repeat; the backward's call, or the first call after it, raises
        with pytest.raises(RuntimeError, match="output_index"):
            y.backward(torch.ones_like(y))
            torch.cuda.synchronize()
            cgx.all_to_all_single(torch.empty(4, H, device="cuda"), torch.randn(4, H, device="cuda"), bits=4)
    finally:
        dist.destroy_process_group()


def test_repeated_slot_world1():
    spawn(_repeat_world1, 1)


def _graph_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, k, H = 300, 8, 1024
        x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
        si = torch.randperm(T * k, device="cuda")
        w = torch.randn(T * k, H, device="cuda", dtype=torch.bfloat16)
        grad = torch.zeros(T, H, device="cuda", dtype=torch.bfloat16)

        def step():
            xa = x.detach().requires_grad_(True)
            y = cgx.differentiable_all_to_all_dispatch(xa, si, bits=4, grad_bits=8)
            (gx,) = torch.autograd.grad(y, xa, w)
            grad.copy_(gx)

        step()  # initialise
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            step()
        for it in range(3):
            si.copy_(torch.randperm(T * k, device="cuda"))
            w.copy_(torch.randn(T * k, H, device="cuda"))
            grad.zero_()
            graph.replay()
            torch.cuda.synchronize()
            _, want = O.dispatch_backward_reference([w.reshape(-1)], [[T * k * H]], [si], k, H, bits=8,
                                                    bucket_size=512)
            assert_same(grad.reshape(-1), want[0].cuda(), f"replay {it}")
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
        xs = [torch.randn(T, H, generator=g).to(torch.bfloat16) for _ in range(world)]
        # every rank sends T * k / world rows to every rank, in slot order
        sis = [torch.randperm(T * k, generator=g) for _ in range(world)]
        per = T * k // world
        xa = xs[rank].cuda().requires_grad_(True)
        y = cgx.differentiable_all_to_all_dispatch(xa, sis[rank].cuda(), bits=4, grad_bits="e5m2")
        ws = [torch.randn(T * k, H, generator=g).to(torch.bfloat16) for _ in range(world)]
        y.backward(ws[rank].cuda())
        counts = [[per * H] * world for _ in range(world)]
        _, want = O.dispatch_backward_reference([w.reshape(-1) for w in ws], counts, sis, k, H, bits="e5m2",
                                                bucket_size=512)
        assert_same(xa.grad.reshape(-1), want[rank].cuda(), f"rank {rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", (2, 4))
def test_public_api_multi_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_multi, world)
