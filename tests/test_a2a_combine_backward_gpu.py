"""The combine's backward (DESIGN §2.13e) on one H100 with W virtual ranks (C.LocalSraGroup for the
fused kernel, C.LocalReducerGroup and torch for the composition), bit for bit and NaN-aware: the
scaled routed call against the oracle over dtypes x widths x buckets and worlds x row lengths,
stochastic rounding, edge inputs and edge scales, repeated input rows with an output_index, the
composition against the fused kernel, small slots, inputs and outputs at odd element offsets, calls
interleaved on one heap, a bad index, the gate-gradient kernel against the oracle over dtypes x k (every
KMAX) x H x aligned and offset views; and at world 1 the
public API (composed and fused rows, the refusals of the process group, a CUDA graph replayed with
new indices and scales, and the differentiable combine with both gate_grad options)."""
import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import hooks

from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BITS = (2, 4, 8, 32, "e4m3", "e5m2")
FILL = -5.0


def dev():
    return torch.device("cuda", 0)


def make_group(world, dtype, slot=1 << 20):
    lanes = max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))
    return C.LocalSraGroup(world, lanes, slot, 5000, 256)


class Case:
    """Rank q holds T rows and sends rows[q][r] rows to rank r, gathered by input_index (repeats on
    purpose) and scaled by input_scale; rank r scatters what it receives by a partial permutation
    output_index into nr + 3 rows (the 3 rows nobody names keep FILL)."""

    def __init__(self, W, H, dtype, seed, T=6, xs=None):
        g = torch.Generator().manual_seed(seed)
        self.W, self.H, self.dtype = W, H, dtype
        rows = [[int(v) for v in torch.randint(1, 5, (W,), generator=g)] for _ in range(W)]
        self.counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        self.xs = xs or [(torch.randn(T, H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype) for q in range(W)]
        self.ii = [torch.randint(0, self.xs[q].shape[0], (sum(rows[q]),), generator=g) for q in range(W)]
        self.sc = [torch.randn(sum(rows[q]), generator=g) * 2 for q in range(W)]
        self.nr = [sum(rows[q][r] for q in range(W)) for r in range(W)]
        self.oi = [torch.randperm(self.nr[r] + 3, generator=g)[:self.nr[r]] for r in range(W)]

    def outputs(self):
        return [torch.full(((self.nr[r] + 3) * self.H,), FILL, dtype=self.dtype, device=dev()) for r in range(self.W)]

    def run(self, grp, bits, bucket, **kw):
        outs = self.outputs()
        grp.all_to_all([x.to(dev()).reshape(-1) for x in self.xs], outs, self.counts, bits=bits, bucket_size=bucket,
                       input_index=[ix.to(dev()) for ix in self.ii], output_index=[ix.to(dev()) for ix in self.oi],
                       row=self.H, input_scale=[s.to(dev()) for s in self.sc], **kw)
        torch.cuda.synchronize()
        grp.check()
        return [o.cpu() for o in outs]

    def sent(self):
        """the scaled rows as torch computes them, on the GPU"""
        return [(x.to(dev()).index_select(0, ix.to(dev())).float() * s.to(dev())[:, None]).to(self.dtype)
                for x, ix, s in zip(self.xs, self.ii, self.sc)]

    def reference(self, bits, bucket):
        return O.routed_all_to_all_reference(self.xs, self.counts, self.ii, self.oi, self.H, bits=bits,
                                             bucket_size=bucket, outputs=[o.cpu() for o in self.outputs()],
                                             input_scale=self.sc)


def check(case, got, want, what):
    for r in range(case.W):
        assert_same(got[r], want[r], f"{what} rank {r}")


@pytest.mark.parametrize("dtype,bits,bucket", list(itertools.product(DTYPES, BITS, (512, 1024))))
def test_fused_matches_oracle(dtype, bits, bucket):
    case = Case(8, 7168, dtype, seed=DTYPES.index(dtype) * 100 + BITS.index(bits) * 10 + bucket // 512)
    check(case, case.run(make_group(8, dtype), bits, bucket), case.reference(bits, bucket), f"{dtype} {bits} {bucket}")


@pytest.mark.parametrize("world,H", list(itertools.product((1, 2, 3, 8), (1024, 7168))))
def test_fused_worlds(world, H):
    case = Case(world, H, torch.bfloat16, seed=world * 10 + H % 7, T=9)
    check(case, case.run(make_group(world, torch.bfloat16), 4, 512), case.reference(4, 512), f"W{world} H{H}")


def test_stochastic_matches_unscaled_call_on_scaled_rows():
    case = Case(4, 2048, torch.bfloat16, seed=21)
    grp = make_group(4, torch.bfloat16)
    kw = dict(stochastic=True, seed=77, seq=5)
    got = case.run(grp, 3, 512, **kw)
    outs = case.outputs()
    grp.all_to_all([s.reshape(-1) for s in case.sent()], outs, case.counts, bits=3, bucket_size=512,
                   output_index=[ix.to(dev()) for ix in case.oi], row=case.H, **kw)
    torch.cuda.synchronize()
    grp.check()
    check(case, got, [o.cpu() for o in outs], "stochastic")


@pytest.mark.parametrize("dtype", DTYPES)
def test_edge_inputs_and_scales(dtype):
    W, H, T = 4, 1024, 8
    ins, _ = edge_inputs(dtype, T * H, 512, seed=4, world=W, bits=4)
    case = Case(W, H, dtype, seed=3, T=T, xs=[i.reshape(T, H).cpu() for i in ins])
    special = torch.tensor([0.0, -0.0, -1.5, float("inf"), float("-inf"), float("nan"), 1e5, 3e38])
    for q in range(W):
        n = case.sc[q].numel()
        case.sc[q][:min(n, special.numel())] = special[:n]
    for bits in (4, 32, "e5m2"):
        check(case, case.run(make_group(W, dtype), bits, 512), case.reference(bits, 512), f"edge {bits}")


@pytest.mark.parametrize("H,bucket,bits", [(2048, 512, 4), (7168, 1024, "e4m3"), (640, 1024, 4), (1000, 100, 8)])
def test_composition_matches_fused(H, bucket, bits):
    # index_select, the scale in torch, the generic reducer's plain call, index_copy_: what the process
    # group's composed path computes; the fused kernel where it can route the rows
    case = Case(3, H, torch.bfloat16, seed=H)
    red = C.LocalReducerGroup(3, "SRA")
    sent = [s.reshape(-1) for s in case.sent()]
    recv = [torch.empty(case.nr[r] * H, dtype=case.dtype, device=dev()) for r in range(3)]
    red.all_to_all(sent, recv, case.counts, bits=bits, bucket_size=bucket)
    outs = case.outputs()
    for r in range(3):
        outs[r].view(-1, H).index_copy_(0, case.oi[r].to(dev()), recv[r].view(-1, H))
    torch.cuda.synchronize()
    composed = [o.cpu() for o in outs]
    check(case, composed, case.reference(bits, bucket), f"composed H={H}")
    if C.a2a_rows_fit(H, bits if isinstance(bits, int) else 8, bucket, DT_CODE[case.dtype]):
        check(case, case.run(make_group(3, torch.bfloat16), bits, bucket), composed, f"fused H={H}")


@pytest.mark.parametrize("bits,bucket", [(4, 512), (32, 512), ("e4m3", 1024)])
def test_small_slots_many_windows(bits, bucket):
    case = Case(3, 2048, torch.float16, seed=8, T=40)
    case.ii = [torch.randint(0, 40, (ix.numel() * 8,)) for ix in case.ii]
    case.sc = [torch.randn(ix.numel()) for ix in case.ii]
    case.counts = [[c * 8 for c in row] for row in case.counts]
    case.nr = [n * 8 for n in case.nr]
    g = torch.Generator().manual_seed(1)
    case.oi = [torch.randperm(n + 3, generator=g)[:n] for n in case.nr]
    grp = C.LocalSraGroup(3, 2, 64 << 10, 5000, 256)
    check(case, case.run(grp, bits, bucket), case.reference(bits, bucket), "small slots")


def test_interleaved_on_one_heap():
    W, dtype, H = 4, torch.bfloat16, 1024
    grp = make_group(W, dtype)
    case = Case(W, H, dtype, seed=31)
    want = case.reference(4, 512)
    n = 4096
    xs = [torch.randn(W * n, device=dev()).to(dtype) for _ in range(W)]
    counts = [[n] * W for _ in range(W)]
    T, k = 8, 4
    ccounts = [[T * k // W * H] * W for _ in range(W)]
    cx = [torch.randn(T * k * H, device=dev()).to(dtype) for _ in range(W)]
    gates = [torch.rand(T, k, device=dev()) for _ in range(W)]
    coi = [torch.randperm(T * k, device=dev()) for _ in range(W)]
    for it in range(2):
        check(case, case.run(grp, 4, 512), want, f"scaled {it}")
        routed = [torch.empty(W * n, dtype=dtype, device=dev()) for _ in range(W)]
        rix = [torch.randperm(W * n // 512, device=dev()) for _ in range(W)]
        grp.all_to_all(xs, routed, counts, bits=4, bucket_size=512, row=512, input_index=rix)
        codes = [torch.empty(W * n, dtype=torch.float8_e4m3fn, device=dev()) for _ in range(W)]
        scales = [torch.empty(W * n // 512, device=dev()) for _ in range(W)]
        grp.all_to_all(xs, codes, counts, bits="e4m3", bucket_size=512, output_scales=scales)
        slots = [torch.empty(T * k * H, dtype=dtype, device=dev()) for _ in range(W)]
        comb = [torch.empty(T * H, dtype=dtype, device=dev()) for _ in range(W)]
        grp.all_to_all(cx, slots, ccounts, bits=4, bucket_size=512, output_index=coi, row=H, gate=gates,
                       combine_out=comb)
        torch.cuda.synchronize()
        grp.check()
        ref = O.routed_all_to_all_reference([x.cpu() for x in xs], counts, [i.cpu() for i in rix], [None] * W, 512,
                                            bits=4, bucket_size=512)
        cref = O.routed_all_to_all_combine_reference([x.cpu() for x in cx], ccounts, [i.cpu() for i in coi],
                                                     [g.cpu() for g in gates], H, bits=4, bucket_size=512)[1]
        for r in range(W):
            assert_same(routed[r].cpu(), ref[r], f"routed {it} rank {r}")
            assert_same(comb[r].cpu(), cref[r], f"combine {it} rank {r}")


def test_bad_index_is_reported():
    case = Case(2, 1024, torch.float32, seed=41)
    case.ii[1][0] = case.xs[1].shape[0]
    grp = make_group(2, torch.float32)
    with pytest.raises(RuntimeError, match="input_index"):
        case.run(grp, 4, 512)
    assert "input_index" in grp.status(1)
    assert grp.status(0) == ""


def test_binding_refusals():
    case = Case(2, 1024, torch.float32, seed=2)
    grp = make_group(2, torch.float32)
    case.sc = [s[:-1] for s in case.sc]
    with pytest.raises(ValueError, match="input_scale"):
        case.run(grp, 4, 512)


SENTINEL, GUARD = -7.0, 64


def _guarded(x, offset):
    buf = torch.full((offset + x.numel() + GUARD,), SENTINEL, dtype=x.dtype, device=dev())
    view = buf[offset:offset + x.numel()]
    view.copy_(x)
    return buf, view


@pytest.mark.parametrize("dtype,bits,offset", list(itertools.product((torch.bfloat16, torch.float32),
                                                                     (4, 32, "e4m3"), (1, 3))))
def test_unaligned_views(dtype, bits, offset):
    # inputs and outputs at an odd element offset: every scaled send takes its element-at-a-time path
    # (unaligned full items, the raw items' scalar loop, the own rows' scalar copy)
    case = Case(3, 2048, dtype, seed=offset * 7 + len(str(bits)))
    ins = [_guarded(x.to(dev()).reshape(-1), offset) for x in case.xs]
    outs = [_guarded(o, offset) for o in case.outputs()]
    grp = make_group(3, dtype)
    grp.all_to_all([v for _, v in ins], [v for _, v in outs], case.counts, bits=bits, bucket_size=512,
                   input_index=[ix.to(dev()) for ix in case.ii], output_index=[ix.to(dev()) for ix in case.oi],
                   row=case.H, input_scale=[s.to(dev()) for s in case.sc])
    torch.cuda.synchronize()
    grp.check()
    for (_, v), x in zip(ins, case.xs):
        assert_same(v.cpu(), x.reshape(-1), "input modified")
    for buf, v in ins + outs:
        n = v.numel()
        assert (buf[:offset] == SENTINEL).all() and (buf[offset + n:] == SENTINEL).all(), "sentinel overwritten"
    check(case, [v.cpu() for _, v in outs], case.reference(bits, 512), f"offset {offset} {bits}")


# ---- the gate-gradient kernel ------------------------------------------------------------------------
# (grad_out, slots) element offsets: (0, 0) is the 16-byte path wherever H is a multiple of 16 bytes' worth
# of elements (640, 1024, 7168), the other pairs and the ragged H the element-at-a-time path; k covers every
# KMAX (1, 2, 4, 8, 16, 32)
@pytest.mark.parametrize("dtype,k,H,offs", list(itertools.product(DTYPES, (1, 2, 3, 8, 16, 32), (1, 7, 640, 1024, 7168),
                                                                  ((0, 0), (0, 1), (1, 0)))))
def test_gate_grad_kernel_matches_oracle(dtype, k, H, offs):
    g = torch.Generator().manual_seed(k * 100 + H + 10 * offs[0] + offs[1])
    T = 5
    go_buf = torch.randn(T * H + 1, generator=g).to(dtype).to(dev())
    x_buf = (torch.randn(T * k * H + 1, generator=g) * 3).to(dtype).to(dev())
    go = go_buf[offs[0]:offs[0] + T * H].view(T, H)
    x = x_buf[offs[1]:offs[1] + T * k * H].view(T * k, H)
    got = C.combine_gate_grad(go, x, k)
    torch.cuda.synchronize()
    assert got.shape == (T, k) and got.dtype == torch.float32
    assert_same(got.cpu(), O.combine_gate_grad_reference(go.cpu(), x.cpu()), f"{dtype} k{k} H{H} offsets {offs}")


@pytest.mark.parametrize("H", (1030, 1032))  # fp32 rows of 4120 bytes (element at a time), 4128 bytes (16-byte)
def test_gate_grad_kernel_edge_values(H):
    T, k = 4, 3
    go = torch.randn(T, H, device=dev())
    x = torch.randn(T * k, H, device=dev())
    go[0, 5] = float("nan")
    x[4, 0], x[4, 9] = float("inf"), float("-inf")
    x[7] = -0.0
    x[11, 100] = 3e38
    go[3, 100] = 3e38
    assert_same(C.combine_gate_grad(go, x, k).cpu(), O.combine_gate_grad_reference(go.cpu(), x.cpu()), "edge")


# ---- the public API at world 1 -------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        # H 640 with bucket 1024: the composed path; the others run in the fused kernel
        for dtype, H, bucket, bits in [(torch.bfloat16, 1024, 512, 4), (torch.float32, 7168, 1024, "e4m3"),
                                       (torch.float16, 640, 1024, 4), (torch.bfloat16, 2048, 512, 32)]:
            T, n = 37, 50
            x = torch.randn(T, H, device="cuda", generator=g).to(dtype)
            ii = torch.randint(0, T, (n,), device="cuda", generator=g)
            sc = torch.randn(n, device="cuda", generator=g)
            sc[:3] = torch.tensor([0.0, float("inf"), -2.0])
            oi = torch.randperm(n + 4, device="cuda", generator=g)[:n]
            out = torch.full((n + 4, H), FILL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, x, bits=bits, bucket_size=bucket, input_index=ii, output_index=oi,
                                  input_scale=sc)
            want = O.routed_all_to_all_reference([x.cpu()], [[n * H]], [ii.cpu()], [oi.cpu()], H, bits=bits,
                                                 bucket_size=bucket, outputs=[torch.full(((n + 4) * H,), FILL,
                                                                                         dtype=dtype)],
                                                 input_scale=[sc.cpu()])[0]
            assert_same(out.reshape(-1), want.cuda(), f"scaled {dtype} H={H}")
        # the process group repeats the Python checks
        pg = hooks._native_backend(dist.group.WORLD, x)
        x = torch.randn(8, 512, device="cuda")
        ix = torch.arange(8, device="cuda")
        with pytest.raises(ValueError, match="no combine"):
            pg.all_to_all_compressed(torch.empty(8, 512, device="cuda"), x, [], [], 8, 512, False, -1, ix, ix, None,
                                     torch.rand(4, 2, device="cuda"), torch.empty(4, 512, device="cuda"),
                                     torch.ones(8, device="cuda"))
        with pytest.raises(ValueError, match="needs an input_index"):
            pg.all_to_all_compressed(torch.empty(8, 512, device="cuda"), x, [], [], 8, 512, False, -1, None, None,
                                     None, None, None, torch.ones(8, device="cuda"))
        out = torch.empty(8, 512, device="cuda")
        with pytest.raises(ValueError, match="overlaps the output"):
            pg.all_to_all_compressed(out, x, [], [], 8, 512, False, -1, ix, None, None, None, None,
                                     out.reshape(-1)[:8])
        # the differentiable combine: the input gradient is today's, bit for bit, whichever gate_grad
        T, k, H = 20, 4, 1024
        for dtype in (torch.float32, torch.bfloat16):
            xa = torch.randn(T * k, H, device="cuda", generator=g).to(dtype).requires_grad_()
            oi = torch.randperm(T * k, device="cuda", generator=g)
            w = torch.randn(T, H, device="cuda", generator=g).to(dtype)
            grads = {}
            for mode in ("torch", "fused"):
                ga = torch.rand(T, k, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1),
                                requires_grad=True)
                xa.grad = None
                y = cgx.differentiable_all_to_all_combine(xa, ga, oi, bits=8, grad_bits=4, gate_grad=mode)
                y.backward(w)
                grads[mode] = (xa.grad.clone(), ga.grad.clone())
            slots = torch.zeros(T * k, H, device="cuda", dtype=dtype)
            cgx.all_to_all_single(slots, xa.detach(), bits=8, output_index=oi)
            gslots = (w.reshape(T, 1, H) * ga.detach().unsqueeze(-1)).to(dtype).reshape(T * k, H)
            want_gx = torch.empty_like(xa)
            cgx.all_to_all_single(want_gx, gslots, bits=4, input_index=oi)
            assert_same(grads["torch"][0], want_gx, f"input gradient torch {dtype}")
            assert_same(grads["fused"][0], want_gx, f"input gradient fused {dtype}")
            assert_same(grads["torch"][1], (w.reshape(T, 1, H).float() * slots.reshape(T, k, H).float()).sum(-1),
                        f"gate gradient torch {dtype}")
            assert_same(grads["fused"][1], O.combine_gate_grad_reference(w.cpu(), slots.cpu()).cuda(),
                        f"gate gradient fused {dtype}")
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def _graph_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, n, H = 300, 600, 1024
        x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
        ii = torch.randint(0, T, (n,), device="cuda")
        sc = torch.randn(n, device="cuda")
        oi = torch.randperm(n, device="cuda")
        out = torch.zeros(n, H, device="cuda", dtype=torch.bfloat16)
        cgx.all_to_all_single(out, x, bits=4, input_index=ii, output_index=oi, input_scale=sc)  # initialise
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            cgx.all_to_all_single(out, x, bits=4, input_index=ii, output_index=oi, input_scale=sc)
        for it in range(3):
            x.copy_(torch.randn(T, H, device="cuda"))
            ii.copy_(torch.randint(0, T, (n,), device="cuda"))
            sc.copy_(torch.randn(n, device="cuda"))
            oi.copy_(torch.randperm(n, device="cuda"))
            out.zero_()
            graph.replay()
            torch.cuda.synchronize()
            want = O.routed_all_to_all_reference([x.cpu()], [[n * H]], [ii.cpu()], [oi.cpu()], H, bits=4,
                                                 bucket_size=512, outputs=[torch.zeros(n * H, dtype=x.dtype)],
                                                 input_scale=[sc.cpu()])[0]
            assert_same(out.reshape(-1), want.cuda(), f"replay {it}")
    finally:
        dist.destroy_process_group()


def test_cuda_graph_world1():
    spawn(_graph_world1, 1)


# ---- several GPUs: a top-2 MoE layer's combine, forward and backward -----------------------------------
def _moe_multi(rank, world):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        T, k, H = 64, 2, 2048
        g = torch.Generator().manual_seed(5)
        xs = [torch.randn(T * k, H, generator=g).to(torch.bfloat16) for _ in range(world)]
        ois = [torch.randperm(T * k, generator=g) for _ in range(world)]
        gates = [torch.rand(T, k, generator=g) for _ in range(world)]
        ws = [torch.randn(T, H, generator=g).to(torch.bfloat16) for _ in range(world)]
        per = T * k // world
        counts = [[per * H] * world for _ in range(world)]
        x = xs[rank].cuda().requires_grad_()
        gate = gates[rank].cuda().requires_grad_()
        y = cgx.differentiable_all_to_all_combine(x, gate, ois[rank].cuda(), bits=4, grad_bits=8, gate_grad="fused")
        y.backward(ws[rank].cuda())
        slots, _ = O.routed_all_to_all_combine_reference([v.reshape(-1) for v in xs], counts, ois, gates, H, bits=4,
                                                         bucket_size=512)
        back = O.routed_all_to_all_reference(ws, counts, [ix // k for ix in ois], [None] * world, H, bits=8,
                                             bucket_size=512, input_scale=[gt.reshape(-1)[ix] for gt, ix in
                                                                           zip(gates, ois)])
        assert_same(x.grad.reshape(-1), back[rank].cuda(), f"input gradient rank {rank}")
        assert_same(gate.grad, O.combine_gate_grad_reference(ws[rank], slots[rank].reshape(T * k, H)).cuda(),
                    f"gate gradient rank {rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", (2, 4))
def test_moe_layer_multi_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_moe_multi, world)
