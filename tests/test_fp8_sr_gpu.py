"""Stochastic FP8 rounding ("e4m3_sr" / "e5m2_sr", DESIGN §2.13h) on one H100: the fused kernels at
virtual ranks (C.LocalSraGroup: all-to-all plain, routed, scaled, combine and codes output;
reduce-scatter; all-gather and its codes output; SRA and one-shot), the generic reducers' device item
kernels (C.LocalReducerGroup), the cross-node all-to-all's pack and unpack on virtual nodes and the
engine (C.LocalEngineGroup), each bitwise equal, NaN-aware, to the CPU simulator or the oracle for
the same seed and sequence; a CUDA graph whose replays advance the random stream; and the public API
at world 1. The `multigpu` cases run the public API at world 2 and 4; they have not been run on
several GPUs."""
from __future__ import annotations

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import counts, inputs, outputs
from _bitwise import assert_same
from _dist_utils import spawn
from _engine_cases import TIMEOUT_MS, assert_results, clean_environment  # noqa: F401

pytestmark = pytest.mark.gpu
C = cgx._C
FMTS = ("e4m3_sr", "e5m2_sr")
BASE = {"e4m3_sr": "e4m3", "e5m2_sr": "e5m2"}
TDT = {"e4m3_sr": torch.float8_e4m3fn, "e5m2_sr": torch.float8_e5m2}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
WORLDS = (2, 3, 8)
BUCKETS = (7, 128, 512, 1024, 8192)
MIN_LANE = 256
SEED, SEQ = 0x1234_5678_9ABC, 21


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


def offset_views(ts, dtype, off):
    """copies of ts that start `off` elements into their storage (unaligned for off odd)"""
    out = []
    for t in ts:
        buf = torch.empty(t.numel() + off, dtype=dtype, device=dev())
        v = buf[off:]
        v.copy_(t.reshape(-1))
        out.append(v)
    return out


# ---- the all-to-all ----------------------------------------------------------------------------------
@pytest.mark.parametrize("off", (0, 1), ids=("aligned", "unaligned"))
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_a2a_fused_and_generic(bucket, fmt, dtype, off):
    for W in WORLDS:
        c = counts(W, "uneven", max(300, bucket + bucket // 3 + 5), W * 31 + bucket)
        xs = inputs(c, dtype, W * 31 + bucket)
        sim = outputs(c, dtype)
        C.all_to_all_simulate(xs, sim, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ)
        ref = O.all_to_all_reference(xs, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ)
        outs = offset_views(outputs(c, dtype), dtype, off)
        g = make_group(W, dtype)
        g.all_to_all(offset_views(xs, dtype, off), outs, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ,
                     stochastic=bool(W % 2))
        torch.cuda.synchronize()
        g.check()
        gen = cuda(outputs(c, dtype))
        C.LocalReducerGroup(W, "SRA", 5000).all_to_all(cuda(xs), gen, c, bits=fmt, bucket_size=bucket, seed=SEED,
                                                       seq=SEQ)
        torch.cuda.synchronize()
        for r in range(W):
            assert_same(sim[r], ref[r], f"W={W} simulator rank {r}")
            assert_same(outs[r].cpu(), sim[r], f"W={W} fused rank {r}")
            assert_same(gen[r].cpu(), sim[r], f"W={W} generic rank {r}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("scaled", (False, True), ids=("routed", "scaled"))
def test_a2a_routed_and_scaled(scaled, fmt, dtype):
    """the routed (and scaled) fused call is the plain call on the gathered (and scaled) rows,
    scattered by the output index, with the same random bits"""
    for W, H, bucket in ((2, 1024, 512), (3, 7168, 1024), (8, 2048, 128)):
        g = torch.Generator().manual_seed(W + H)
        rows = counts(W, "uneven", 4, seed=W + H)
        c = [[rows[q][r] * H for r in range(W)] for q in range(W)]
        send = [sum(rows[q]) for q in range(W)]
        recv = [sum(rows[q][r] for q in range(W)) for r in range(W)]
        xs = [(torch.randn(max(1, s // 2 + 1), H, generator=g) * (q + 1)).to(dtype) for q, s in enumerate(send)]
        ii = [torch.randint(0, x.shape[0], (s,), generator=g) for x, s in zip(xs, send)]
        oi = [torch.randperm(m + 5, generator=g)[:m] for m in recv]
        out0 = [torch.randn(m + 5, H, generator=g).to(dtype) for m in recv]
        sc = [torch.rand(s, generator=g) * 2 for s in send]
        sent = [x[i] for x, i in zip(xs, ii)]
        if scaled:
            sent = [(s_.float() * k[:, None]).to(dtype) for s_, k in zip(sent, sc)]
        plain = outputs(c, dtype)
        C.all_to_all_simulate([s_.reshape(-1) for s_ in sent], plain, c, bits=fmt, bucket_size=bucket, seed=SEED,
                              seq=SEQ)
        outs = [o.reshape(-1).to(dev()) for o in out0]
        kw = dict(input_scale=cuda(sc)) if scaled else {}
        grp = make_group(W, dtype)
        grp.all_to_all([x.reshape(-1).to(dev()) for x in xs], outs, c, bits=fmt, bucket_size=bucket, seed=SEED,
                       seq=SEQ, input_index=cuda(ii), output_index=cuda(oi), row=H, **kw)
        torch.cuda.synchronize()
        grp.check()
        for r in range(W):
            want = out0[r].clone()
            want.index_copy_(0, oi[r], plain[r].view(-1, H))
            assert_same(outs[r].cpu(), want.reshape(-1), f"W={W} rank {r}")


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
    grp.all_to_all([x.reshape(-1).to(dev()) for x in xs], slots, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ,
                   output_index=cuda(oi), row=H, gate=cuda(gates), combine_out=outs)
    torch.cuda.synchronize()
    grp.check()
    plain = outputs(c, dtype)
    C.all_to_all_simulate([x.reshape(-1) for x in xs], plain, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ)
    for r in range(W):
        want = torch.zeros(T * k, H, dtype=dtype)
        want.index_copy_(0, oi[r], plain[r].view(-1, H))
        assert_same(slots[r].cpu(), want.reshape(-1), f"slots rank {r}")
        assert_same(outs[r].cpu(), O.combine_rows_reference(want, gates[r]).reshape(-1), f"combine rank {r}")


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
@pytest.mark.parametrize("bucket", (128, 1024, "H"))
def test_a2a_codes_output(bucket, fmt, dtype):
    H = 7168 if bucket == "H" else 2048
    B = H if bucket == "H" else bucket
    for W in WORLDS:
        c = [[v * H for v in row] for row in counts(W, "uneven", 2, W + B)]
        xs = inputs(c, dtype, B)
        rc, rs = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=B, seed=SEED, seq=SEQ)
        for which, grp in (("fused", make_group(W, dtype)), ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            outs, scales = codes_buffers(c, B, fmt)
            grp.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=B, seed=SEED, seq=SEQ, output_scales=scales)
            torch.cuda.synchronize()
            for r in range(W):
                assert_codes(outs[r], rc[r], f"{which} W={W} rank {r}")
                assert_same(scales[r].cpu(), rs[r], f"{which} W={W} rank {r} scales")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("nodes,local", [(2, 2), (3, 2), (2, 4)])
def test_a2a_across_virtual_nodes(nodes, local, fmt):
    """pack and unpack across nodes: the engine at N x L ranks gives the one-node all-to-all of its
    W ranks, bit for bit, and both equal the simulator at the engine's sequence"""
    W, dtype = nodes * local, torch.bfloat16
    c = counts(W, "uneven", 3000, seed=W)
    xs = inputs(c, dtype, local)
    res = {}
    for L in (local, W):
        for p2p in (True, False):
            g = C.LocalEngineGroup(W, L, dict(p2p=p2p), 1, 1 << 22, TIMEOUT_MS)
            outs = cuda(outputs(c, dtype))
            g.all_to_all(cuda(xs), outs, c, bits=fmt, bucket_size=512)
            torch.cuda.synchronize()
            res[(L, p2p)] = cpu(outs)
    for key, outs in res.items():
        for r in range(W):
            assert_same(outs[r], res[(W, True)][r], f"L={key[0]} p2p={key[1]} rank {r}")
    assert not all(torch.equal(a, b) for a, b in zip(res[(W, True)], O.all_to_all_reference(
        xs, c, bits=BASE[fmt], bucket_size=512)))


# ---- reduce-scatter, all-gather, allreduce -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", BUCKETS)
def test_sharded_fused_and_generic(bucket, fmt, dtype):
    for W in WORLDS:
        S = 3 * 8192 + 37
        table = [(0, S, 8, bucket)]
        g = torch.Generator().manual_seed(W + bucket)
        full = [(torch.randn(W * S, generator=g) * (r + 1)).to(dtype) for r in range(W)]
        own = [full[r][r * S:(r + 1) * S].clone() for r in range(W)]
        rs_sim = [torch.empty(S, dtype=dtype) for _ in range(W)]
        C.reduce_scatter_simulate(full, rs_sim, table, average=True, seed=SEED, seq=SEQ, bits=fmt)
        ag_ref = O.all_gather_reference(own, table, fmt, seed=SEED, seq=SEQ)
        for which, grp in (("fused", make_group(W, dtype, 1 << 22)), ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            outs = [torch.empty(S, dtype=dtype, device=dev()) for _ in range(W)]
            grp.reduce_scatter(cuda(full), outs, table, True, seed=SEED, seq=SEQ, bits=fmt)
            gathered = [torch.empty(W * S, dtype=dtype, device=dev()) for _ in range(W)]
            grp.all_gather(cuda(own), gathered, table, seed=SEED, seq=SEQ, bits=fmt)
            torch.cuda.synchronize()
            assert_results(cpu(outs), rs_sim, f"{which} rs W={W}")
            assert_results(cpu(gathered), [ag_ref] * W, f"{which} ag W={W}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", (128, 1024, 8192))
def test_all_gather_codes_output(bucket, fmt):
    for W in WORLDS:
        S = 2 * max(bucket, 1024)
        g = torch.Generator().manual_seed(W + bucket)
        xs = [torch.randn(S, generator=g) * torch.exp(torch.randn(S, generator=g) * 2) for _ in range(W)]
        rc, rs = O.all_gather_codes_reference(xs, fmt, bucket, seed=SEED, seq=SEQ)
        for which, grp in (("fused", make_group(W, torch.float32, 1 << 22)),
                           ("generic", C.LocalReducerGroup(W, "SRA", 5000))):
            codes = [torch.full((W * S,), 0x55, dtype=torch.uint8, device=dev()).view(TDT[fmt]) for _ in range(W)]
            scales = [torch.full((W * S // bucket,), float("nan"), device=dev()) for _ in range(W)]
            grp.all_gather(cuda(xs), codes, [(0, S, 8, bucket)], seed=SEED, seq=SEQ, bits=fmt, output_scales=scales)
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
            (grp.allreduce_oneshot if oneshot else grp.allreduce)(got, table, True, seed=SEED, seq=SEQ, bits=fmt)
            torch.cuda.synchronize()
            grp.check()
            sim = [x.clone() for x in xs]
            (C.oneshot_simulate if oneshot else C.sra_simulate)(sim, table, lanes, True, seed=SEED, seq=SEQ,
                                                                min_lane_elems=MIN_LANE, bits=fmt)
            assert_results(cpu(got), sim, f"{'oneshot' if oneshot else 'sra'} W={W}")
        assert_results(sim, O.oneshot_reference(xs, table, average=True, fmt=fmt, seed=SEED, seq=SEQ),
                       f"oneshot reference W={W}")
        got = cuda(xs)
        C.LocalReducerGroup(W, "SRA", 5000).allreduce(got, table, average=True, seed=SEED, seq=SEQ, bits=fmt)
        torch.cuda.synchronize()
        sim = [x.clone() for x in xs]
        C.sra_simulate(sim, table, 1, True, seed=SEED, seq=SEQ, min_lane_elems=O.GENERIC_MIN_LANE_ELEMS, bits=fmt)
        assert_results(cpu(got), sim, f"generic SRA W={W}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("world,local", [(4, 4), (4, 2), (8, 2)])
@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_engine(fused, world, local, fmt):
    """the engine at world > 1: every rank ends with the same bytes, a fresh group given the same
    calls repeats them bit for bit, a second call draws new bits, and the average stays within the
    format's error of the exact one. (The fused and generic paths key their calls differently, as
    for integer stochastic rounding, so they are not compared bitwise.)"""
    dtype = torch.bfloat16
    layers = [(0, 37, 32, 512), (37, 30_000, 8, 1024), (30_037, 4501, 8, 100)]
    n = 34_538
    g = torch.Generator().manual_seed(world + local)
    xs = [(torch.randn(n, generator=g) * (1 + 0.1 * r)).to(dtype) for r in range(world)]
    runs = []
    for _ in range(2):
        eg = C.LocalEngineGroup(world, local, dict(p2p=fused), 1, 1 << 22, TIMEOUT_MS)
        first = cuda(xs)
        eg.allreduce_layers(first, layers, True, bits=fmt)
        second = cuda(xs)
        eg.allreduce_layers(second, layers, True, bits=fmt)
        torch.cuda.synchronize()
        runs.append((cpu(first), cpu(second)))
    for r in range(world):
        assert_same(runs[0][0][r], runs[0][0][0], f"rank {r} vs rank 0")
        assert_same(runs[1][0][r], runs[0][0][r], f"repeat, rank {r}")
        assert_same(runs[1][1][r], runs[0][1][r], f"repeat of the second call, rank {r}")
    assert not torch.equal(runs[0][0][0], runs[0][1][0])
    exact = torch.stack([x.double() for x in xs]).mean(0)
    rel = float((runs[0][0][0].double() - exact).norm() / exact.norm())
    assert rel < (0.08 if fmt == "e4m3_sr" else 0.16), rel


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph_replays_advance_the_stream(fmt):
    """a captured all-to-all: replay k draws the bits of sequence SEQ + k (the capture's launch
    counts as the call after the warm-up's), as integer stochastic rounding does"""
    W, dtype, bucket = 4, torch.float32, 512
    g = make_group(W, dtype, 1 << 22)
    c = [[1000, 7000, 0, 9000], [8192, 500, 4000, 1], [0, 33, 2000, 10000], [6500, 0, 5, 300]]
    ins = [torch.empty(sum(row), device=dev(), dtype=dtype) for row in c]
    outs = [torch.empty(sum(c[q][r] for q in range(W)), device=dev(), dtype=dtype) for r in range(W)]
    xs = inputs(c, dtype, 0)
    for t, x in zip(ins, xs):
        t.copy_(x)
    g.all_to_all(ins, outs, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        g.all_to_all(ins, outs, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ)
    torch.cuda.synchronize()
    for it in range(3):
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        sim = outputs(c, dtype)
        C.all_to_all_simulate(xs, sim, c, bits=fmt, bucket_size=bucket, seed=SEED, seq=SEQ + it)
        for r in range(W):
            assert_same(outs[r].cpu(), sim[r], f"replay {it} rank {r}")


# ---- the public API ----------------------------------------------------------------------------------------
def _pg_api(rank, world):
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        for fmt in FMTS:
            x = torch.randn(64 * world, 1024, device="cuda", dtype=torch.bfloat16) * (rank + 1)
            out = torch.empty_like(x)
            cgx.all_to_all_single(out, x, bits=fmt)
            codes = torch.empty(64 * world, 1024, dtype=TDT[fmt], device="cuda")
            scales = torch.empty(64 * world, 1, device="cuda")
            cgx.all_to_all_single(codes, x, bits=fmt, bucket_size=1024, output_scales=scales)
            assert torch.isfinite(scales).all()
            dec = (codes.float() * scales).to(x.dtype)
            if world == 1:
                assert_same(out, x, f"{fmt}: the own chunk is a copy")
                # the own chunk's codes: stream a2a_rng_stream(0, 0)
                assert torch.allclose(dec.float(), x.float(), rtol=0.25, atol=1e-2)
            sh = x.reshape(-1)[: 65536].contiguous()
            gathered = torch.empty(world * sh.numel(), dtype=sh.dtype, device="cuda")
            cgx.all_gather_into_tensor(gathered, sh, bits=fmt, bucket_size=1024)
            y = x.reshape(-1).float().clone()
            cgx.all_reduce(y, bits=fmt, bucket_size=512)
            assert torch.isfinite(y).all()
            rs_out = torch.empty(y.numel() // world, device="cuda")
            cgx.reduce_scatter_tensor(rs_out, y, bits=fmt, stochastic=True)
            assert torch.isfinite(rs_out).all()
        with pytest.raises(ValueError, match="round"):
            cgx.all_reduce(torch.ones(64, device="cuda"), bits="e5m2", stochastic=True)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_api, 1)


@pytest.mark.multigpu
@pytest.mark.parametrize("world", (2, 4))
def test_public_api_multigpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_api, world)
