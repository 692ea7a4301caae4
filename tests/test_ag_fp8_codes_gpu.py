"""The FP8 all-gather's codes output on the GPU: the fused ag_kernel against the simulator and the
oracle byte for byte (NaN-aware), on guarded unaligned views with shards that are not multiples of
16; small slots with many windows (the scale address across windows); codes, decoded, reduce-scatter,
allreduce and all-to-all codes calls interleaved on one heap; a CUDA graph replayed with new inputs;
the device generic path against the fused and the host paths; the multi-node refusal; the public
API at world 1; and the row-wise ``torch._scaled_mm`` contract. With >= 2 GPUs, the public API on
both transports."""
from __future__ import annotations

import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import DTYPES
from _ag_codes_cases import (BUCKET_SHARDS, FMTS, TDT, assert_codes, codes_buffers, decode, shards, simulate_codes,
                             table)
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
GUARD = 64
SENT_F = -7.25
SENT_B = 0x5A
MIN_LANE = 256
FUSED_WORLDS = (2, 3, 8)


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def slot_for(tab, world, S, dtype):
    rep = [(c * S + o, n, b, k) for c in range(world) for (o, n, b, k) in tab]
    wire = C.build_plan(rep, world=world, lanes=lanes_for(world, dtype), dtype=DT_CODE[dtype],
                        skip_incomplete=False, min_lane_elems=MIN_LANE)["max_chunk_wire"]
    return (wire + 255) // 256 * 256 + 256


def make_group(world, dtype, slot):
    return C.LocalSraGroup(world, lanes_for(world, dtype), slot, 5000, MIN_LANE)


def guarded(n, offset, dtype, fill):
    buf = torch.full((offset + n + GUARD,), fill, dtype=dtype, device=dev())
    return buf, buf[offset:offset + n]


def check_guards(pairs, offset, fill):
    for buf, v in pairs:
        n = v.numel()
        assert (buf[:offset] == fill).all() and (buf[offset + n:] == fill).all(), "sentinel overwritten"


def run_fused(g, xs, fmt, bucket, offset=0):
    """the codes call on guarded views (codes and scales at `offset` elements); returns host codes and scales"""
    W, S = len(xs), xs[0].numel()
    ins = []
    for x in xs:
        buf, v = guarded(S, offset, x.dtype, SENT_F)
        v.copy_(x.to(dev()))
        ins.append((buf, v))
    cods = [guarded(W * S, offset, torch.uint8, SENT_B) for _ in range(W)]
    scs = [guarded(W * S // bucket, offset, torch.float32, SENT_F) for _ in range(W)]
    g.all_gather([v for _, v in ins], [v.view(TDT[fmt]) for _, v in cods], table(S, bucket), bits=fmt,
                 output_scales=[v for _, v in scs])
    torch.cuda.synchronize()
    g.check()
    for (_, v), x in zip(ins, xs):
        assert_same(v.cpu(), x, "input modified")
    check_guards(ins + scs, offset, SENT_F)
    check_guards(cods, offset, SENT_B)
    return [v.cpu().view(TDT[fmt]) for _, v in cods], [v.cpu() for _, v in scs]


def check(got, xs, fmt, bucket, what):
    sim_c, sim_s = simulate_codes(xs, fmt, bucket)
    ref_c, ref_s = O.all_gather_codes_reference(xs, fmt, bucket)
    for r in range(len(xs)):
        assert_codes(got[0][r], sim_c[r], f"{what}: rank {r} codes vs simulator")
        assert_same(got[1][r], sim_s[r], f"{what}: rank {r} scales vs simulator")
        assert_codes(got[0][r], ref_c, f"{what}: rank {r} codes vs oracle")
        assert_same(got[1][r], ref_s, f"{what}: rank {r} scales vs oracle")


# ---- the fused kernel against the simulator and the oracle --------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, BUCKET_SHARDS)))
def test_fused_matches_simulator(dtype, fmt, bucket):
    i = DTYPES.index(dtype) * 7 + FMTS.index(fmt) * 3 + list(BUCKET_SHARDS).index(bucket)
    W = FUSED_WORLDS[i % len(FUSED_WORLDS)]
    S = BUCKET_SHARDS[bucket]
    xs = shards(W, S, dtype, i)
    g = make_group(W, dtype, slot_for(table(S, bucket), W, S, dtype))
    offset = (0, 3, 5)[i % 3]
    check(run_fused(g, xs, fmt, bucket, offset=offset), xs, fmt, bucket, f"W={W} S={S} B={bucket} off={offset}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [64, 512])
def test_fused_edge_inputs(dtype, fmt, bucket):
    W = 3
    S = 40 * bucket
    xs, planted = edge_inputs(dtype, S, bucket, seed=7, world=W, bits=8)
    assert planted
    g = make_group(W, dtype, slot_for(table(S, bucket), W, S, dtype))
    got = run_fused(g, xs, fmt, bucket, offset=1)
    check(got, xs, fmt, bucket, "edge")
    dec = [torch.empty(W * S, dtype=dtype, device=dev()) for _ in range(W)]
    g.all_gather([x.to(dev()) for x in xs], dec, table(S, bucket), bits=fmt)
    torch.cuda.synchronize()
    for r in range(W):
        assert_same(decode(got[0][r], got[1][r], bucket, dtype), dec[r].cpu(), f"decode identity rank {r}")


@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", 8192),
                                        ("e4m3", 7168)])
def test_small_slots_many_windows(fmt, bucket):
    W, dtype = 4, torch.bfloat16
    S = bucket * (24 * 8192 // bucket)
    slot = 8192 if bucket <= 1024 else 3 * 8192
    assert len(C.reduce_scatter_windows(table(S, bucket), W, lanes_for(W, dtype), DT_CODE[dtype], False, MIN_LANE,
                                        slot)) > 3
    xs = shards(W, S, dtype, bucket)
    got = run_fused(make_group(W, dtype, slot), xs, fmt, bucket, offset=7)
    check(got, xs, fmt, bucket, "small slots")


def test_codes_decoded_rs_allreduce_and_a2a_interleaved_on_one_heap():
    W, dtype, S, B = 4, torch.float16, 12_000, 400
    tab = table(S, B)
    g = make_group(W, dtype, max(slot_for(tab, W, S, dtype), 1 << 20))
    for it, fmt in enumerate(["e4m3", "e5m2", "e4m3"]):
        xs = shards(W, S, dtype, it)
        check(run_fused(g, xs, fmt, B, offset=(1, 3, 5)[it]), xs, fmt, B, f"call {it} codes")
        dec = [torch.empty(W * S, dtype=dtype, device=dev()) for _ in range(W)]
        g.all_gather([x.to(dev()) for x in xs], dec, tab, bits=fmt)
        full = [torch.cat(xs).to(dev()) for _ in range(W)]
        rs = [torch.empty(S, dtype=dtype, device=dev()) for _ in range(W)]
        g.reduce_scatter(full, rs, tab, bits=fmt)
        ar = [torch.cat(xs).to(dev()) for _ in range(W)]
        g.allreduce(ar, [(0, W * S, 8, 512)], bits=fmt)
        c = [[2 * 1024] * W for _ in range(W)]
        a2a_in = [x[:2 * 1024 * W].contiguous() for x in xs]
        a2a_c = [torch.zeros(2 * 1024 * W, dtype=torch.uint8, device=dev()).view(TDT[fmt]) for _ in range(W)]
        a2a_s = [torch.zeros(2 * 1024 * W // 128, device=dev()) for _ in range(W)]
        g.all_to_all([x.to(dev()) for x in a2a_in], a2a_c, c, bits=fmt, bucket_size=128, output_scales=a2a_s)
        torch.cuda.synchronize()
        g.check()
        ref_dec = O.all_gather_reference(xs, tab, fmt=fmt)
        codes, scales = simulate_codes(xs, fmt, B)
        ref_rs = O.reduce_scatter_reference([f.cpu() for f in full], tab, fmt=fmt)
        ref_ar = O.sra_reference([torch.cat(xs)] * W, [(0, W * S, 8, 512)], lanes=lanes_for(W, dtype),
                                 min_lane_elems=MIN_LANE, fmt=fmt)
        for r in range(W):
            assert_same(dec[r].cpu(), ref_dec, f"call {it} decoded rank {r}")
            assert_same(dec[r].cpu(), decode(codes[r], scales[r], B, dtype), f"call {it} decode identity rank {r}")
            assert_same(rs[r].cpu(), ref_rs[r], f"call {it} reduce-scatter rank {r}")
            assert_same(ar[r].cpu(), ref_ar[r], f"call {it} allreduce rank {r}")
        ref_c, ref_s = O.all_to_all_codes_reference(a2a_in, c, fmt=fmt, bucket_size=128)
        for r in range(W):
            assert_codes(a2a_c[r].cpu(), ref_c[r], f"call {it} a2a codes rank {r}")
            assert_same(a2a_s[r].cpu(), ref_s[r], f"call {it} a2a scales rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph_replayed_with_new_inputs(fmt):
    W, dtype, S, B = 4, torch.bfloat16, 6 * 1024, 128
    g = make_group(W, dtype, 8192)  # several windows: several launches in the graph
    ins = [torch.zeros(S, dtype=dtype, device=dev()) for _ in range(W)]
    codes, scales = codes_buffers(W, S, B, fmt, device=dev())

    def call():
        g.all_gather(ins, codes, table(S, B), bits=fmt, output_scales=scales)

    call()  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        call()
    torch.cuda.synchronize()
    for it in range(3):
        xs = shards(W, S, dtype, 100 + it)
        for t, x in zip(ins, xs):
            t.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        check(([c.cpu() for c in codes], [t.cpu() for t in scales]), xs, fmt, B, f"replay {it}")


# ---- the generic reducer (NCCL transport's path) ---------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", 7168)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_path_equals_fused_and_host(fmt, bucket, dtype):
    W, S = 3, BUCKET_SHARDS[bucket]
    xs = shards(W, S, dtype, bucket)
    fused = run_fused(make_group(W, dtype, slot_for(table(S, bucket), W, S, dtype)), xs, fmt, bucket, offset=3)
    got = {}
    for where in ("cpu", "cuda"):
        red = C.LocalReducerGroup(W, "SRA", 5000)
        cods, scs = codes_buffers(W, S, bucket, fmt, device=where)
        red.all_gather([x.to(where) for x in xs], cods, table(S, bucket), bits=fmt, output_scales=scs)
        torch.cuda.synchronize()
        got[where] = ([t.cpu() for t in cods], [t.cpu() for t in scs])
    for r in range(W):
        assert_codes(got["cuda"][0][r], fused[0][r], f"device generic vs fused rank {r}")
        assert_same(got["cuda"][1][r], fused[1][r], f"device generic vs fused rank {r}")
        assert_codes(got["cuda"][0][r], got["cpu"][0][r], f"device vs host rank {r}")
        assert_same(got["cuda"][1][r], got["cpu"][1][r], f"device vs host rank {r}")


# ---- several nodes: refused on every rank before anything runs -------------------------------------------
@pytest.mark.parametrize("p2p", [True, False])
def test_multinode_refused_on_every_rank(p2p):
    W, L, S, B = 4, 2, 4096, 128
    g = C.LocalEngineGroup(W, L, dict(p2p=p2p, min_lane_elems=MIN_LANE), 2, 1 << 20, 20000)
    xs = [x.to(dev()) for x in shards(W, S, torch.bfloat16, 1)]
    codes, scales = codes_buffers(W, S, B, "e4m3", device=dev())
    with pytest.raises(RuntimeError, match="one node"):
        g.all_gather(xs, codes, shard_layers=table(S, B), bits="e4m3", output_scales=scales)
    torch.cuda.synchronize()
    for r in range(W):
        st = g.stats(r)
        assert st["calls"] == 0 and st["kernel_launches"] == 0 and st["wire_bytes"] == 0, f"rank {r}: {st}"
        assert (codes[r].view(torch.uint8) == 0x55).all() and scales[r].isnan().all(), f"rank {r} output written"


# ---- the public API at world 1 ---------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        gen = torch.Generator(device="cuda").manual_seed(0)
        for dtype, fmt, shape, B in [(torch.bfloat16, "e4m3", (16, 4096), 128), (torch.float32, "e5m2", (8, 7168), 7168),
                                     (torch.float16, "e4m3", (2500,), 100), (torch.bfloat16, "e5m2", (3, 8192), 8192)]:
            x = torch.randn(shape, device="cuda", generator=gen).to(dtype)
            codes = torch.empty(shape, dtype=TDT[fmt], device="cuda")
            scales = torch.empty(x.numel() // B, device="cuda")
            if len(shape) == 2:
                scales = scales.view(shape[0], -1)  # [rows, H / B] works: any shape of the right size
            work = cgx.all_gather_into_tensor(codes, x, bits=fmt, bucket_size=B, output_scales=scales, async_op=True)
            work.wait()
            torch.cuda.synchronize()
            rc, rs = O.fp8_quantize(x.reshape(-1).cpu(), fmt, B)
            assert_codes(codes.cpu(), rc, f"{dtype} {fmt} {shape}")
            assert_same(scales.cpu().reshape(-1), rs)
            dec = torch.empty_like(x)
            cgx.all_gather_into_tensor(dec, x, bits=fmt, bucket_size=B)
            assert_same(decode(codes.cpu(), scales.cpu(), B, dtype).view(shape), dec.cpu(), f"decode identity {shape}")
        # below CGX_COMPRESSION_MINIMAL_SIZE the decoded call copies; the codes call still encodes
        x = torch.randn(256, device="cuda")
        codes = torch.empty(256, dtype=torch.float8_e4m3fn, device="cuda")
        scales = torch.empty(2, device="cuda")
        cgx.all_gather_into_tensor(codes, x, bits="e4m3", bucket_size=128, output_scales=scales)
        rc, rs = O.fp8_quantize(x.cpu(), "e4m3", 128)
        assert_codes(codes.cpu(), rc, "small")
        assert_same(scales.cpu(), rs)
        # the refusals on CUDA tensors
        x = torch.randn(8, 512, device="cuda")
        codes = torch.empty(8, 512, dtype=torch.float8_e4m3fn, device="cuda")
        good = torch.empty(8, 4, device="cuda")
        for bad in (good.double(), good[:, :2], torch.empty(4, 8, device="cuda").t(), good.cpu(),
                    torch.empty(7, 4, device="cuda")):
            with pytest.raises(ValueError, match="output_scales"):
                cgx.all_gather_into_tensor(codes, x, bits="e4m3", bucket_size=128, output_scales=bad)
        for kw in (dict(bits=8), dict(bits="e5m2"), dict(bits="e4m3", stochastic=True),
                   dict(bits="e4m3", bucket_size=3), dict(bits="e4m3", bucket_size=16384),
                   dict(bits="e4m3", layers=[(0, 4096, 8, 128)])):
            kw.setdefault("bucket_size", 128)
            with pytest.raises(ValueError):
                cgx.all_gather_into_tensor(codes, x, output_scales=good, **kw)
        flat = torch.empty(8 * 512 + 64, device="cuda")
        with pytest.raises((ValueError, RuntimeError), match="overlap"):
            cgx.all_gather_into_tensor(codes, flat[:4096].view(8, 512), bits="e4m3", bucket_size=128,
                                       output_scales=flat[8:40].view(8, 4))
        raw = torch.empty(8 * 512, dtype=torch.uint8, device="cuda")
        with pytest.raises((ValueError, RuntimeError), match="overlap"):
            cgx.all_gather_into_tensor(raw.view(torch.float8_e4m3fn), x, bits="e4m3", bucket_size=128,
                                       output_scales=raw[64:192].view(torch.float32))
        with pytest.raises(RuntimeError):  # codes of the wrong size
            cgx.all_gather_into_tensor(codes[:4], x, bits="e4m3", bucket_size=128, output_scales=good[:4])
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


# ---- the GEMM contract --------------------------------------------------------------------------------
def test_rowwise_scaled_mm_contract():
    """bucket = H: one scale per row, the row-wise scaling torch._scaled_mm takes. Gathered activations
    [M, H] are `a` with scale_a [M, 1]; a gathered weight [N, K] is `b` = codes.view(N, K).t() with
    scale_b [1, N]. The product equals the oracle's codes' product bit for bit and is close to an fp32
    GEMM of the decoded values."""
    W, H, N, dtype = 2, 7168, 256, torch.bfloat16
    g = torch.Generator().manual_seed(4)
    acts = [torch.randn(64 * H, generator=g).to(dtype) for _ in range(W)]      # [T/W, H] per rank
    wts = [(torch.randn(N // W * H, generator=g) * 0.05).to(dtype) for _ in range(W)]  # [N/W, K] per rank
    grp = make_group(W, dtype, slot_for(table(64 * H, H), W, 64 * H, dtype))
    a_c, a_s = run_fused(grp, acts, "e4m3", H)
    b_c, b_s = run_fused(grp, wts, "e4m3", H)
    ra_c, ra_s = O.all_gather_codes_reference(acts, "e4m3", H)
    rb_c, rb_s = O.all_gather_codes_reference(wts, "e4m3", H)
    ref = torch._scaled_mm(ra_c.reshape(-1, H).to(dev()), rb_c.reshape(N, H).to(dev()).t(),
                           scale_a=ra_s.reshape(-1, 1).to(dev()), scale_b=rb_s.reshape(1, N).to(dev()),
                           out_dtype=torch.bfloat16)
    for r in range(W):
        a = a_c[r].reshape(-1, H).to(dev())
        b = b_c[r].reshape(N, H).to(dev()).t()
        sa, sb = a_s[r].reshape(-1, 1).to(dev()), b_s[r].reshape(1, N).to(dev())
        out = torch._scaled_mm(a, b, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
        assert_same(out.cpu(), ref.cpu(), f"rank {r}")
        exact = (a.float() * sa) @ (b.float() * sb)
        torch.testing.assert_close(out.float(), exact, rtol=2e-2, atol=2e-2 * exact.abs().max().item())


# ---- several GPUs -----------------------------------------------------------------------------------------
def _pg_codes(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        S, B, fmt = 4096, 128, "e4m3"
        xs = shards(world, S, torch.bfloat16, 0)
        ref_c, ref_s = O.all_gather_codes_reference(xs, fmt, B)
        codes = torch.empty(world * S, dtype=TDT[fmt], device="cuda")
        scales = torch.empty(world * S // B, device="cuda")
        cgx.all_gather_into_tensor(codes, xs[rank].cuda(), bits=fmt, bucket_size=B, output_scales=scales)
        assert_codes(codes.cpu(), ref_c, f"rank {rank}")
        assert_same(scales.cpu(), ref_s, f"rank {rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
def test_public_api_codes_multigpu(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_codes, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport})
