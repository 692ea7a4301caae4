"""Power-of-two FP8 scales ("e4m3_pow2" / "e5m2_pow2") on one H100: the fused kernels at virtual ranks
(C.LocalSraGroup: all-to-all plain, routed, scaled, combine and codes output; reduce-scatter; all-gather
and its codes output; SRA and one-shot), the generic reducers' device kernels (C.LocalReducerGroup)
and the engine (C.LocalEngineGroup, local_size < world included), each bitwise equal, NaN-aware, to
the CPU simulator and the oracle; the public API at world 1; and row-wise torch._scaled_mm on the
codes output."""
from __future__ import annotations

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import counts, inputs, outputs
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs
from _engine_cases import TIMEOUT_MS, assert_results, clean_environment  # noqa: F401

pytestmark = pytest.mark.gpu
C = cgx._C
FMTS = ("e4m3_pow2", "e5m2_pow2")
TDT = {"e4m3_pow2": torch.float8_e4m3fn, "e5m2_pow2": torch.float8_e5m2}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
WORLDS = (2, 3, 8)
BUCKETS = (7, 128, 512, 1024, 8192)
MIN_LANE = 256
MIXED = [(0, 37, 32, 512), (37, 30_000, 8, 1024), (30_037, 301, 32, 512), (30_338, 4501, 8, 100),
         (34_839, 9000, 8, 512)]
S_MIXED = 43_839


@pytest.fixture(autouse=True)
def no_format_in_environment(monkeypatch):
    monkeypatch.delenv("CGX_COMPRESSION_FORMAT", raising=False)


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 21):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, MIN_LANE)


def cuda(ts):
    return [t.to(dev()) for t in ts]


def cpu(ts):
    return [t.cpu() for t in ts]


def assert_codes(got, ref, what):
    got, ref = got.cpu().reshape(-1), ref.cpu().reshape(-1)
    gn, rn = torch.isnan(got.float()), torch.isnan(ref.float())
    assert torch.equal(gn, rn), f"{what}: NaN codes differ"
    assert torch.equal(got.view(torch.uint8)[~gn], ref.view(torch.uint8)[~rn]), f"{what}: codes differ"


def a2a_case(world, dtype, bucket, seed):
    c = counts(world, "uneven", max(300, bucket + bucket // 3 + 5), seed)
    return c, inputs(c, dtype, seed)


def a2a_sim(xs, c, fmt, bucket):
    sim = outputs(c, xs[0].dtype)
    C.all_to_all_simulate(xs, sim, c, bits=fmt, bucket_size=bucket)
    return sim


# ---- the all-to-all ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_a2a_fused_and_generic(bucket, fmt, dtype):
    for W in WORLDS:
        c, xs = a2a_case(W, dtype, bucket, W * 31 + bucket)
        sim = a2a_sim(xs, c, fmt, bucket)
        ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=bucket)
        outs = cuda(outputs(c, dtype))
        g = make_group(W, dtype)
        g.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=bucket)
        torch.cuda.synchronize()
        g.check()
        gen = cuda(outputs(c, dtype))
        C.LocalReducerGroup(W, "SRA", 5000).all_to_all(cuda(xs), gen, c, bits=fmt, bucket_size=bucket)
        torch.cuda.synchronize()
        for r in range(W):
            assert_same(outs[r].cpu(), sim[r], f"W={W} fused rank {r}")
            assert_same(gen[r].cpu(), sim[r], f"W={W} generic rank {r}")
            assert_same(sim[r], ref[r], f"W={W} simulator rank {r}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
def test_a2a_edge_inputs(fmt, dtype):
    W, n, bucket = 3, 12 * 512, 64
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=2, world=W, bits=8)
    assert planted
    c = [[n] * W for _ in range(W)]
    outs = cuda(outputs(c, dtype))
    g = make_group(W, dtype)
    g.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=bucket)
    torch.cuda.synchronize()
    g.check()
    sim = a2a_sim(xs, c, fmt, bucket)
    for r in range(W):
        assert_same(outs[r].cpu(), sim[r], f"rank {r}")


class Routed:
    """rank q sends rows gathered by an index with repeats, scaled per row; rank r scatters them by a
    permutation into a larger output"""

    def __init__(self, W, H, dtype, seed):
        g = torch.Generator().manual_seed(seed)
        rows = counts(W, "uneven", 4, seed=seed)
        self.W, self.H, self.dtype = W, H, dtype
        self.c = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        send = [sum(rows[q]) for q in range(W)]
        self.recv = [sum(rows[q][r] for q in range(W)) for r in range(W)]
        self.xs = [(torch.randn(max(1, s // 2 + 1), H, generator=g) * (q + 1)).to(dtype) for q, s in enumerate(send)]
        self.ii = [torch.randint(0, x.shape[0], (s,), generator=g) for x, s in zip(self.xs, send)]
        self.oi = [torch.randperm(m + 5, generator=g)[:m] for m in self.recv]
        self.out0 = [torch.randn(m + 5, H, generator=g).to(dtype) for m in self.recv]
        self.sc = [torch.rand(s, generator=g) * 2 for s in send]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("scaled", (False, True), ids=("routed", "scaled"))
def test_a2a_routed_and_scaled(scaled, fmt, dtype):
    for W, H, bucket in ((2, 1024, 512), (3, 7168, 1024), (8, 2048, 128)):
        k = Routed(W, H, dtype, W + H)
        outs = [o.reshape(-1).to(dev()) for o in k.out0]
        kw = dict(input_scale=cuda(k.sc)) if scaled else {}
        g = make_group(W, dtype)
        g.all_to_all([x.reshape(-1).to(dev()) for x in k.xs], outs, k.c, bits=fmt, bucket_size=bucket,
                     input_index=cuda(k.ii), output_index=cuda(k.oi), row=H, **kw)
        torch.cuda.synchronize()
        g.check()
        ref = O.routed_all_to_all_reference(k.xs, k.c, k.ii, k.oi, H, bits=fmt, bucket_size=bucket,
                                            outputs=k.out0, input_scale=k.sc if scaled else None)
        for r in range(W):
            assert_same(outs[r].cpu(), ref[r], f"W={W} rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_a2a_combine(dtype, fmt):
    W, T, k, H, bucket = 4, 24, 4, 2048, 512
    g = torch.Generator().manual_seed(9)
    rows = [[0] * W for _ in range(W)]
    for r in range(W):
        src = torch.randint(0, W, (T * k,), generator=g)
        for q in range(W):
            rows[q][r] = int((src == q).sum())
    c = [[rows[q][r] * H for r in range(W)] for q in range(W)]
    xs = [(torch.randn(sum(rows[q]), H, generator=g) * (q + 1)).to(dtype) for q in range(W)]
    oi = [torch.randperm(T * k, generator=g) for _ in range(W)]
    gates = [torch.rand(T, k, generator=g) * 2 - 0.5 for _ in range(W)]
    slots = [torch.zeros(T * k * H, dtype=dtype, device=dev()) for _ in range(W)]
    outs = [torch.full((T * H,), -3.0, dtype=dtype, device=dev()) for _ in range(W)]
    grp = make_group(W, dtype)
    grp.all_to_all([x.reshape(-1).to(dev()) for x in xs], slots, c, bits=fmt, bucket_size=bucket,
                   output_index=cuda(oi), row=H, gate=cuda(gates), combine_out=outs)
    torch.cuda.synchronize()
    grp.check()
    ref_s, ref_o = O.routed_all_to_all_combine_reference([x.reshape(-1) for x in xs], c, oi, gates, H, bits=fmt,
                                                         bucket_size=bucket)
    for r in range(W):
        assert_same(slots[r].cpu(), ref_s[r], f"slots rank {r}")
        assert_same(outs[r].cpu(), ref_o[r], f"combine rank {r}")


def codes_buffers(c, B, fmt):
    W = len(c)
    outs, scales = [], []
    for r in range(W):
        n = sum(c[q][r] for q in range(W))
        outs.append(torch.full((n,), 0x55, dtype=torch.uint8, device=dev()).view(TDT[fmt]))
        scales.append(torch.full((n // B,), float("nan"), device=dev()))
    return outs, scales


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", (128, 512, 1024, "H"))
def test_a2a_codes_output(bucket, fmt, dtype):
    H = 7168 if bucket == "H" else 2048
    B = H if bucket == "H" else bucket
    for W in WORLDS:
        c = [[v * H for v in row] for row in counts(W, "uneven", 2, W + B)]
        xs = inputs(c, dtype, B)
        rc, rs = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=B)
        for which, grp in (("fused", make_group(W, dtype)), ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            outs, scales = codes_buffers(c, B, fmt)
            grp.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=B, output_scales=scales)
            torch.cuda.synchronize()
            for r in range(W):
                assert_codes(outs[r], rc[r], f"{which} W={W} rank {r}")
                assert_same(scales[r].cpu(), rs[r], f"{which} W={W} rank {r} scales")
                s = scales[r][torch.isfinite(scales[r])]
                assert torch.equal(s.to(torch.float8_e8m0fnu).float(), s)


# ---- reduce-scatter, all-gather, allreduce -----------------------------------------------------------------
def full_inputs(world, S, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(world * S, generator=g) * (r + 1)).to(dtype) for r in range(world)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_sharded_fused_and_generic(bucket, fmt, dtype):
    for W in WORLDS:
        S = 3 * 8192 + 37
        table = [(0, S, 8, bucket)]
        full = full_inputs(W, S, dtype, W + bucket)
        own = [full[r][r * S:(r + 1) * S].clone() for r in range(W)]
        rs_ref = O.reduce_scatter_reference(full, table, average=True, fmt=fmt)
        ag_ref = O.all_gather_reference(own, table, fmt)
        sim = [torch.empty(S, dtype=dtype) for _ in range(W)]
        C.reduce_scatter_simulate(full, sim, table, average=True, bits=fmt)
        assert_results(sim, rs_ref, "rs simulator")
        for which, grp in (("fused", make_group(W, dtype, 1 << 22)), ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            outs = [torch.empty(S, dtype=dtype, device=dev()) for _ in range(W)]
            grp.reduce_scatter(cuda(full), outs, table, True, bits=fmt)
            gathered = [torch.empty(W * S, dtype=dtype, device=dev()) for _ in range(W)]
            grp.all_gather(cuda(own), gathered, table, bits=fmt)
            torch.cuda.synchronize()
            assert_results(cpu(outs), rs_ref, f"{which} rs W={W}")
            assert_results(cpu(gathered), [ag_ref] * W, f"{which} ag W={W}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", (128, 1024, 8192, 7168))
def test_all_gather_codes_output(bucket, fmt):
    for W in WORLDS:
        S = 2 * max(bucket, 1024)
        g = torch.Generator().manual_seed(W + bucket)
        xs = [torch.randn(S, generator=g) * torch.exp(torch.randn(S, generator=g) * 2) for _ in range(W)]
        rc, rs = O.all_gather_codes_reference(xs, fmt, bucket)
        for which, grp in (("fused", make_group(W, torch.float32, 1 << 22)),
                           ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            codes = [torch.full((W * S,), 0x55, dtype=torch.uint8, device=dev()).view(TDT[fmt]) for _ in range(W)]
            scales = [torch.full((W * S // bucket,), float("nan"), device=dev()) for _ in range(W)]
            grp.all_gather(cuda(xs), codes, [(0, S, 8, bucket)], bits=fmt, output_scales=scales)
            torch.cuda.synchronize()
            for r in range(W):
                assert_codes(codes[r], rc, f"{which} W={W} rank {r}")
                assert_same(scales[r].cpu(), rs, f"{which} W={W} rank {r} scales")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_allreduce_fused_and_generic(bucket, fmt, dtype):
    for W in WORLDS:
        table = [(0, 37, 32, 512), (37, 24 * 1024 + 3, 8, bucket), (24 * 1024 + 40, 301, 32, 512)]
        n = 24 * 1024 + 350
        g = torch.Generator().manual_seed(W * 7 + bucket)
        xs = [(torch.randn(n, generator=g) * (r + 1)).to(dtype) for r in range(W)]
        lanes = lanes_for(W, dtype)
        grp = make_group(W, dtype, 1 << 22)
        for oneshot in (False, True):
            got = cuda(xs)
            (grp.allreduce_oneshot if oneshot else grp.allreduce)(got, table, True, bits=fmt)
            torch.cuda.synchronize()
            grp.check()
            sim = [x.clone() for x in xs]
            (C.oneshot_simulate if oneshot else C.sra_simulate)(sim, table, lanes, True, min_lane_elems=MIN_LANE,
                                                                bits=fmt)
            assert_results(cpu(got), sim, f"{'oneshot' if oneshot else 'sra'} W={W}")
        ref = O.sra_reference(xs, table, lanes=lanes, min_lane_elems=MIN_LANE, average=True, fmt=fmt)
        C.sra_simulate(xs_sim := [x.clone() for x in xs], table, lanes, True, min_lane_elems=MIN_LANE, bits=fmt)
        assert_results(xs_sim, ref, f"sra reference W={W}")
        for kind, kref in (("SRA", O.sra_reference), ("RING", O.ring_reference)):
            got = cuda(xs)
            C.LocalReducerGroup(W, kind, 5000).allreduce(got, table, average=True, bits=fmt)
            torch.cuda.synchronize()
            kw = dict(lanes=1, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS) if kind == "SRA" else {}
            assert_results(cpu(got), kref(xs, table, average=True, fmt=fmt, **kw), f"generic {kind} W={W}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_allreduce_edge_inputs_and_broadcast(dtype, fmt):
    W, bucket, n = 3, 64, 64 * 90
    table = [(0, n, 8, bucket)]
    lanes = lanes_for(W, dtype)
    owners = O.block_owners(table, n, W, lanes, dtype, False, MIN_LANE)
    xs, planted = edge_inputs(dtype, n, bucket, 5, world=W, bits=8, owners=owners, where="peer")
    assert planted
    got = cuda(xs)
    grp = make_group(W, dtype)
    grp.allreduce(got, table, False, bits=fmt)
    torch.cuda.synchronize()
    grp.check()
    sim = [x.clone() for x in xs]
    C.sra_simulate(sim, table, lanes, False, min_lane_elems=MIN_LANE, bits=fmt)
    assert_results(cpu(got), sim, "edge sra")
    for root in (0, W - 1):
        got = cuda(xs)
        C.LocalReducerGroup(W, "SRA", 5000).broadcast_compressed(got, table, root, bits=fmt)
        torch.cuda.synchronize()
        assert_results(cpu(got), O.broadcast_compressed_reference(xs, table, root=root, fmt=fmt), f"bcast {root}")


# ---- the engine, one node and several ------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,local", [(4, 4), (4, 2), (6, 3), (8, 2)])
@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_engine(fused, world, local, fmt):
    dtype = torch.bfloat16
    g = C.LocalEngineGroup(world, local, dict(p2p=fused), 1, 1 << 22, TIMEOUT_MS)
    full = full_inputs(world, S_MIXED, dtype, world + local)
    own = [full[r][r * S_MIXED:(r + 1) * S_MIXED].clone() for r in range(world)]
    outs = [torch.empty(world * S_MIXED, dtype=dtype, device=dev()) for _ in range(world)]
    g.all_gather(cuda(own), outs, MIXED, bits=fmt)
    torch.cuda.synchronize()
    assert_results(cpu(outs), [O.all_gather_reference(own, MIXED, fmt)] * world, "ag")
    outs = [torch.empty(S_MIXED, dtype=dtype, device=dev()) for _ in range(world)]
    g.reduce_scatter(cuda(full), outs, True, MIXED, bits=fmt)
    torch.cuda.synchronize()
    want = O.reduce_scatter_hier_reference(full, MIXED, local_size=local, average=True, fmt=fmt)
    assert_results(cpu(outs), want, "rs")
    c = counts(world, "uneven", 3000, seed=world)
    xs = inputs(c, dtype, local)
    outs = cuda(outputs(c, dtype))
    g.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=512)
    torch.cuda.synchronize()
    ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=512)
    for r in range(world):
        assert_same(outs[r].cpu(), ref[r], f"a2a rank {r}")
    H = 1024
    c = [[v * H for v in row] for row in counts(world, "uneven", 2, world)]
    xs = inputs(c, dtype, 3)
    codes, scales = codes_buffers(c, H, fmt)
    g.all_to_all(cuda(xs), codes, c, bits=fmt, bucket_size=H, output_scales=scales)
    torch.cuda.synchronize()
    rc, rs = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=H)
    for r in range(world):
        assert_codes(codes[r], rc[r], f"a2a codes rank {r}")
        assert_same(scales[r].cpu(), rs[r], f"a2a scales rank {r}")


# ---- the public API at world 1 ---------------------------------------------------------------------------
def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(512, 256), torch.nn.GELU(), torch.nn.Linear(256, 10))


def _pg_world1(rank, world):
    from torch.nn.parallel import DistributedDataParallel as DDP

    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for fmt in FMTS:
            x = torch.randn(64, 1024, device="cuda", dtype=torch.bfloat16)
            out = torch.empty_like(x)
            cgx.all_to_all_single(out, x, bits=fmt)
            assert_same(out, x, f"{fmt}: the own chunk is a copy")
            codes = torch.empty(64, 1024, dtype=TDT[fmt], device="cuda")
            scales = torch.empty(64, 1, device="cuda")
            cgx.all_to_all_single(codes, x, bits=fmt, bucket_size=1024, output_scales=scales)
            rc, rs = O.fp8_quantize(x.reshape(-1).cpu(), fmt, 1024)
            assert_codes(codes, rc, f"{fmt} a2a codes")
            assert_same(scales.reshape(-1).cpu(), rs, f"{fmt} a2a scales")
            g = torch.empty(64 * 1024, dtype=TDT[fmt], device="cuda")
            gs = torch.empty(64, device="cuda")
            cgx.all_gather_into_tensor(g, x.reshape(-1), bits=fmt, bucket_size=1024, output_scales=gs)
            assert_codes(g, rc, f"{fmt} ag codes")
            assert_same(gs.cpu(), rs, f"{fmt} ag scales")
            y = x.reshape(-1).float().clone()
            cgx.all_reduce(y, bits=fmt, bucket_size=512)
            assert torch.isfinite(y).all()
        torch.manual_seed(0)
        model = DDP(_mlp().cuda(), device_ids=[0])
        ref = _mlp().cuda()
        ref.load_state_dict(model.module.state_dict())
        cgx.register_cgx_hook(model, cgx.CGXState(None, compression_params={"bits": "e4m3_pow2", "bucket_size": 512}))
        for step in range(4):
            x = torch.randn(16, 512, device="cuda")
            model(x).square().mean().backward()
            ref(x).square().mean().backward()
            # world 1: every compressed layer is one e4m3_pow2 round trip of its gradient from step 2 on
            for p, q in zip(model.parameters(), ref.parameters()):
                want = q.grad
                if step >= 2 and q.dim() > 1 and q.numel() >= 1024:
                    want = O.fp8_quantize_dequantize(q.grad.reshape(-1).cpu(), "e4m3_pow2", 512).view_as(q).cuda()
                assert_same(p.grad, want, f"step {step} {tuple(p.shape)}")
            model.zero_grad()
            ref.zero_grad()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


def test_rowwise_scaled_mm_with_pow2_scales():
    """bucket = H: one power-of-two scale per row. The gathered codes feed torch._scaled_mm row-wise;
    the product equals the oracle codes' product bit for bit and is close to an fp32 GEMM of the
    decoded values. The scales survive a trip through float8_e8m0fnu unchanged."""
    W, H, N, dtype, fmt = 2, 7168, 256, torch.bfloat16, "e4m3_pow2"
    g = torch.Generator().manual_seed(4)
    acts = [torch.randn(64 * H, generator=g).to(dtype) for _ in range(W)]
    wts = [(torch.randn(N // W * H, generator=g) * 0.05).to(dtype) for _ in range(W)]
    grp = make_group(W, dtype, 1 << 23)
    got = []
    for xs in (acts, wts):
        S = xs[0].numel()
        codes = [torch.empty(W * S, dtype=TDT[fmt], device=dev()) for _ in range(W)]
        scales = [torch.empty(W * S // H, device=dev()) for _ in range(W)]
        grp.all_gather(cuda(xs), codes, [(0, S, 8, H)], bits=fmt, output_scales=scales)
        torch.cuda.synchronize()
        grp.check()
        got.append((codes, scales))
    ra_c, ra_s = O.all_gather_codes_reference(acts, fmt, H)
    rb_c, rb_s = O.all_gather_codes_reference(wts, fmt, H)
    ref = torch._scaled_mm(ra_c.reshape(-1, H).to(dev()), rb_c.reshape(N, H).to(dev()).t(),
                           scale_a=ra_s.reshape(-1, 1).to(dev()), scale_b=rb_s.reshape(1, N).to(dev()),
                           out_dtype=torch.bfloat16)
    (a_c, a_s), (b_c, b_s) = got
    for r in range(W):
        sa, sb = a_s[r].reshape(-1, 1), b_s[r].reshape(1, N)
        assert torch.equal(sa.to(torch.float8_e8m0fnu).float(), sa) and torch.equal(sb.to(torch.float8_e8m0fnu).float(), sb)
        a, b = a_c[r].reshape(-1, H), b_c[r].reshape(N, H).t()
        out = torch._scaled_mm(a, b, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
        assert_same(out.cpu(), ref.cpu(), f"rank {r}")
        exact = (a.float() * sa) @ (b.float() * sb)
        torch.testing.assert_close(out.float(), exact, rtol=2e-2, atol=2e-2 * exact.abs().max().item())
