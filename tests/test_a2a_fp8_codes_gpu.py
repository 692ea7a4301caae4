"""The FP8 all-to-all's codes output (a2a_kernel with CODES) on one H100 with W virtual ranks
(C.LocalSraGroup): codes and scales byte for byte, NaN-aware, equal to the CPU simulator and the
oracle over dtypes, both formats, buckets, worlds and splits; the routed form against the
composition; small slots with many windows; codes, decoded FP8, max-min and raw calls on one heap; a
CUDA graph whose indices change between replays; the generic reducer's device path against the fused
kernel and the host backend; a bad index; the public API at world 1, its refusals and its routed
composition; and the GEMM contract through ``torch._scaled_mm``. With >= 2 GPUs, the public API on
both transports.

Inputs and outputs are views at element offsets 1, 3 and 5 into sentinel-filled buffers: the
elements around each view and the inputs must be unchanged afterwards."""
import itertools

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _a2a_cases import DTYPES, counts, inputs, outputs
from _bitwise import assert_same
from _dist_utils import spawn
from _edge_inputs import edge_inputs
from test_a2a_fp8_codes_cpu import BUCKET_ROWS, FMTS, TDT, assert_codes, row_counts, simulate_codes

pytestmark = pytest.mark.gpu
C = cgx._C
DT_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
GUARD = 64
SENT_F = -7.25
SENT_B = 0x5A


def dev():
    return torch.device("cuda", 0)


def lanes_for(world, dtype):
    return max(1, min(4, C.max_resident_ctas(DT_CODE[dtype]) // 2 // world))


def make_group(world, dtype, slot=1 << 20, lanes=None):
    return C.LocalSraGroup(world, lanes or lanes_for(world, dtype), slot, 5000, 256)


def small_slot(bucket, dtype, lanes):
    block = C.a2a_windows(1, 8, bucket, DT_CODE[dtype], 1 << 20, 1)["block_wire"]
    return ((2 * lanes * block + 16 * lanes) + 255) // 256 * 256


def guarded(n, offset, dtype, fill):
    buf = torch.full((offset + n + GUARD,), fill, dtype=dtype, device=dev())
    return buf, buf[offset:offset + n]


def guarded_codes(n, offset, fmt):
    buf, v = guarded(n, offset, torch.uint8, SENT_B)
    return buf, v.view(TDT[fmt])


def check_guards(pairs, offset, fill):
    for buf, v in pairs:
        n = v.numel()
        b = buf.view(torch.uint8) if buf.dtype == torch.uint8 else buf
        assert (b[:offset] == fill).all() and (b[offset + n:] == fill).all(), "sentinel overwritten"


def run_fused(g, xs, c, fmt, bucket, offset=0):
    """the codes call on guarded views; returns host codes and scales"""
    W = len(xs)
    ins = []
    for x in xs:
        buf, v = guarded(x.numel(), offset, x.dtype, SENT_F)
        v.copy_(x.to(dev()))
        ins.append((buf, v))
    ncol = [sum(c[q][r] for q in range(W)) for r in range(W)]
    cods = [guarded_codes(n, offset, fmt) for n in ncol]
    scs = [guarded(n // bucket, offset, torch.float32, SENT_F) for n in ncol]
    g.all_to_all([v for _, v in ins], [v for _, v in cods], c, bits=fmt, bucket_size=bucket,
                 output_scales=[v for _, v in scs])
    torch.cuda.synchronize()
    g.check()
    for (_, v), x in zip(ins, xs):
        assert_same(v.cpu(), x, "input modified")
    check_guards(ins + scs, offset, SENT_F)
    check_guards(cods, offset, SENT_B)
    return [v.cpu() for _, v in cods], [v.cpu() for _, v in scs]


def check(got, xs, c, fmt, bucket, what):
    sim_c, sim_s = simulate_codes(xs, c, fmt, bucket)
    ref_c, ref_s = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=bucket)
    for r in range(len(xs)):
        assert_codes(got[0][r], sim_c[r], f"{what}: rank {r} codes vs simulator")
        assert_same(got[1][r], sim_s[r], f"{what}: rank {r} scales vs simulator")
        assert_codes(got[0][r], ref_c[r], f"{what}: rank {r} codes vs oracle")
        assert_same(got[1][r], ref_s[r], f"{what}: rank {r} scales vs oracle")


def _bucket(b):
    return BUCKET_ROWS["H"] if b == "H" else b


# ---- the fused kernel against the simulator and the oracle --------------------------------------
@pytest.mark.parametrize("dtype,fmt,bucket", list(itertools.product(DTYPES, FMTS, BUCKET_ROWS)))
def test_fused_matches_simulator(dtype, fmt, bucket):
    H, B = BUCKET_ROWS[bucket], _bucket(bucket)
    i = DTYPES.index(dtype) * 12 + FMTS.index(fmt) * 6 + list(BUCKET_ROWS).index(bucket)
    for j, W in enumerate((2, 3, 8, 16)):
        kind = ("equal", "uneven", "empty")[(i + j) % 3]
        c = row_counts(W, kind, 3 if W <= 3 else 1, H, seed=i * 7 + j)
        xs = inputs(c, dtype, i * 7 + j)
        got = run_fused(make_group(W, dtype), xs, c, fmt, B, offset=(1, 3, 5)[(i + j) % 3])
        check(got, xs, c, fmt, B, f"W={W} {kind} H={H}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("bucket", [64, 512])
def test_fused_edge_inputs(dtype, fmt, bucket):
    W, n = 3, 12 * 512
    xs, planted = edge_inputs(dtype, n * W, bucket, seed=2, world=W, bits=8)
    assert planted
    c = [[n] * W for _ in range(W)]
    check(run_fused(make_group(W, dtype), xs, c, fmt, bucket, offset=1), xs, c, fmt, bucket, "edge")


# ---- the routed form -----------------------------------------------------------------------------
def _routed_case(W, H, dtype, seed, mode):
    """top-k style: rank q sends rows gathered by an index with repeats, rank r scatters what it
    receives by a permutation into a larger output; `mode` says which indices are used"""
    g = torch.Generator().manual_seed(seed)
    rows = counts(W, "uneven", 4, seed=seed)
    c = [[rows[q][r] * H for r in range(W)] for q in range(W)]
    send = [sum(rows[q]) for q in range(W)]
    recv = [sum(rows[q][r] for q in range(W)) for r in range(W)]
    if mode == "output":
        xs = [(torch.randn(s, H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype) for q, s in enumerate(send)]
    else:
        xs = [(torch.randn(max(1, s // 2 + 1), H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype)
              for q, s in enumerate(send)]
    ii = [None if mode == "output" else torch.randint(0, x.shape[0], (s,), generator=g) for x, s in zip(xs, send)]
    oi = [None if mode == "input" else torch.randperm(m + 5, generator=g)[:m] for m in recv]
    rows_out = [m if mode == "input" else m + 5 for m in recv]
    return c, xs, ii, oi, rows_out


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H,bucket", [(512, 128), (1024, 1024), (7168, 128), (7168, 7168)])
@pytest.mark.parametrize("mode", ["input", "output", "both"])
def test_routed_matches_composition(fmt, H, bucket, mode):
    W = 4
    dtype = DTYPES[(H + bucket + len(mode)) % 3]
    assert C.a2a_rows_fit(H, 8, bucket, DT_CODE[dtype])
    c, xs, ii, oi, rows_out = _routed_case(W, H, dtype, H + bucket + len(mode), mode)
    base_c = [torch.randint(0, 256, (m * H,), dtype=torch.uint8).view(TDT[fmt]) for m in rows_out]
    base_s = [torch.randn(m * H // bucket) for m in rows_out]
    g = make_group(W, dtype)
    codes = [b.to(dev()) for b in base_c]
    scales = [s.to(dev()) for s in base_s]
    g.all_to_all([x.to(dev()).reshape(-1) for x in xs], codes, c, bits=fmt, bucket_size=bucket,
                 input_index=[None if ix is None else ix.to(dev()) for ix in ii],
                 output_index=[None if ix is None else ix.to(dev()) for ix in oi], row=H, output_scales=scales)
    torch.cuda.synchronize()
    g.check()
    ref_c, ref_s = O.routed_all_to_all_codes_reference(xs, c, ii, oi, H, fmt=fmt, bucket_size=bucket,
                                                       outputs=base_c, output_scales=base_s)
    for r in range(W):
        assert_codes(codes[r].cpu(), ref_c[r], f"rank {r} codes")
        assert_same(scales[r].cpu(), ref_s[r], f"rank {r} scales")


def test_bad_index_is_reported():
    W, H, B, dtype = 2, 512, 128, torch.float32
    g = make_group(W, dtype)
    c = [[3 * H, 4 * H], [5 * H, 6 * H]]
    xs = [torch.randn(7, H, device=dev()), torch.randn(11, H, device=dev())]
    for which in ("input", "output"):
        ii = [torch.arange(7, device=dev()), torch.arange(11, device=dev())]
        oi = [torch.arange(8, device=dev()), torch.arange(10, device=dev())]
        (ii if which == "input" else oi)[0][1] = -1
        codes = [torch.zeros(n * H, dtype=torch.uint8, device=dev()) for n in (8, 10)]
        scales = [torch.zeros(n * H // B, device=dev()) for n in (8, 10)]
        with pytest.raises(RuntimeError, match=f"{which}_index"):
            g.all_to_all([x.reshape(-1) for x in xs], codes, c, bits="e4m3", bucket_size=B, input_index=ii,
                         output_index=oi, row=H, output_scales=scales)
            torch.cuda.synchronize()
            g.check()
        assert f"{which}_index" in g.status(0)
        g.clear()


# ---- windows, heap sharing, graphs -----------------------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", 8192)])
def test_small_slots_many_windows(fmt, bucket):
    W, lanes, dtype = 4, 2, torch.bfloat16
    slot = small_slot(bucket, dtype, lanes)
    g = make_group(W, dtype, slot=slot, lanes=lanes)
    rows = [[0, 9, 70, 123], [8, 0, 1, 0], [50, 0, 3, 16], [0, 200, 5, 7]]
    for q in range(W):
        rows[q][q] = 3 * q
    H = bucket * (8192 // bucket)  # rows of whole buckets, about one block each
    c = [[v * H for v in row] for row in rows]
    assert len(C.a2a_windows(200 * H, 8, bucket, DT_CODE[dtype], slot, lanes)["lanes"][0]) > 3
    xs = inputs(c, dtype, 7)
    check(run_fused(g, xs, c, fmt, bucket, offset=5), xs, c, fmt, bucket, "small slots")


def test_codes_decoded_max_min_and_raw_interleaved_on_one_heap():
    W, dtype, B = 4, torch.float16, 512
    g = make_group(W, dtype)
    for it, (bits, codes) in enumerate([("e4m3", True), ("e4m3", False), (8, False), ("e5m2", True), (32, False),
                                        (4, False), ("e5m2", True)]):
        c = row_counts(W, "uneven", 2, 1024, seed=it)
        xs = inputs(c, dtype, it)
        if codes:
            check(run_fused(g, xs, c, bits, B, offset=(1, 3, 5)[it % 3]), xs, c, bits, B, f"call {it} codes")
            continue
        outs = outputs(c, dtype, device=dev())
        g.all_to_all([x.to(dev()) for x in xs], outs, c, bits=bits, bucket_size=B)
        torch.cuda.synchronize()
        ref = O.all_to_all_reference(xs, c, bits=bits, bucket_size=B)
        for r in range(W):
            assert_same(outs[r].cpu(), ref[r], f"call {it} bits={bits} rank {r}")


@pytest.mark.parametrize("fmt", FMTS)
def test_cuda_graph_indices_change_between_replays(fmt):
    """one routed codes call of W = 4 virtual ranks with small slots, captured once and replayed with
    new data and new indices written into the captured index tensors"""
    W, lanes, dtype, H, B = 4, 2, torch.bfloat16, 1024, 128
    g = make_group(W, dtype, slot=small_slot(B, dtype, lanes), lanes=lanes)
    c, xs, ii, oi, rows_out = _routed_case(W, H, dtype, 3, "both")
    ins = [x.to(dev()).reshape(-1) for x in xs]
    iis = [ix.to(dev()) for ix in ii]
    ois = [ix.to(dev()) for ix in oi]
    codes = [torch.zeros(m * H, dtype=torch.uint8, device=dev()).view(TDT[fmt]) for m in rows_out]
    scales = [torch.zeros(m * H // B, device=dev()) for m in rows_out]

    def call():
        g.all_to_all(ins, codes, c, bits=fmt, bucket_size=B, input_index=iis, output_index=ois, row=H,
                     output_scales=scales)

    call()  # warm up outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        call()
    torch.cuda.synchronize()
    gen = torch.Generator().manual_seed(9)
    for it in range(3):
        new_x = [(torch.randn(x.shape, generator=gen) * (it + 1)).to(dtype) for x in xs]
        new_ii = [torch.randint(0, x.shape[0], (ix.numel(),), generator=gen) for x, ix in zip(xs, ii)]
        new_oi = [torch.randperm(m, generator=gen)[:ix.numel()] for m, ix in zip(rows_out, oi)]
        for t, v in zip(ins + iis + ois, [x.reshape(-1) for x in new_x] + new_ii + new_oi):
            t.copy_(v)
        before_c = [t.cpu() for t in codes]
        before_s = [t.cpu() for t in scales]
        graph.replay()
        torch.cuda.synchronize()
        g.check()
        ref_c, ref_s = O.routed_all_to_all_codes_reference(new_x, c, new_ii, new_oi, H, fmt=fmt, bucket_size=B,
                                                           outputs=before_c, output_scales=before_s)
        for r in range(W):
            assert_codes(codes[r].cpu(), ref_c[r], f"replay {it} rank {r} codes")
            assert_same(scales[r].cpu(), ref_s[r], f"replay {it} rank {r} scales")


# ---- the generic reducer (NCCL transport's path) ---------------------------------------------------
@pytest.mark.parametrize("fmt,bucket", [("e4m3", 128), ("e5m2", 1024), ("e4m3", 100), ("e5m2", "H")])
@pytest.mark.parametrize("dtype", DTYPES)
def test_generic_path_equals_fused_and_host(fmt, bucket, dtype):
    H, B = BUCKET_ROWS[bucket], _bucket(bucket)
    W = 3
    c = row_counts(W, "uneven", 3, H, seed=B)
    xs = inputs(c, dtype, B)
    fused = run_fused(make_group(W, dtype), xs, c, fmt, B, offset=3)
    got = {}
    for where in ("cpu", "cuda"):
        red = C.LocalReducerGroup(W, "SRA", 5000)
        ncol = [sum(c[q][r] for q in range(W)) for r in range(W)]
        cods = [torch.zeros(n, dtype=torch.uint8, device=where).view(TDT[fmt]) for n in ncol]
        scs = [torch.zeros(n // B, device=where) for n in ncol]
        red.all_to_all([x.to(where) for x in xs], cods, c, bits=fmt, bucket_size=B, output_scales=scs)
        torch.cuda.synchronize()
        got[where] = ([t.cpu() for t in cods], [t.cpu() for t in scs])
    for r in range(W):
        assert_codes(got["cuda"][0][r], fused[0][r], f"device generic vs fused rank {r}")
        assert_same(got["cuda"][1][r], fused[1][r], f"device generic vs fused rank {r}")
        assert_codes(got["cuda"][0][r], got["cpu"][0][r], f"device vs host rank {r}")
        assert_same(got["cuda"][1][r], got["cpu"][1][r], f"device vs host rank {r}")


# ---- the public API at world 1 ---------------------------------------------------------------------
def _pg_world1(rank, world):
    torch.cuda.set_device(0)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        gen = torch.Generator(device="cuda").manual_seed(0)
        # plain, routed in the kernel when the rows fit, composed otherwise (640: rows of 512-element
        # slices do not fit)
        for dtype, fmt, H, B in [(torch.bfloat16, "e4m3", 1024, 128), (torch.float32, "e5m2", 7168, 7168),
                                 (torch.float16, "e4m3", 640, 128), (torch.bfloat16, "e5m2", 7168, 128)]:
            x = torch.randn(40, H, device="cuda", generator=gen).to(dtype)
            codes = torch.empty(40, H, dtype=TDT[fmt], device="cuda")
            scales = torch.empty(40, H // B, device="cuda")
            cgx.all_to_all_single(codes, x, bits=fmt, bucket_size=B, output_scales=scales)
            rc, rs = O.fp8_quantize(x.reshape(-1).cpu(), fmt, B)
            assert_codes(codes.cpu(), rc, f"{dtype} {fmt} H={H}")
            assert_same(scales.cpu().reshape(-1), rs)
            ii = torch.randint(0, 40, (70,), device="cuda", generator=gen)
            oi = torch.randperm(80, device="cuda", generator=gen)[:70]
            codes = torch.full((80, H), SENT_B, dtype=torch.uint8, device="cuda").view(TDT[fmt])
            scales = torch.full((80, H // B), SENT_F, device="cuda")
            c0, s0 = codes.cpu(), scales.cpu()
            cgx.all_to_all_single(codes, x, [70], [70], bits=fmt, bucket_size=B, output_scales=scales,
                                  input_index=ii, output_index=oi)
            ref_c, ref_s = O.routed_all_to_all_codes_reference([x.cpu()], [[70 * H]], [ii.cpu()], [oi.cpu()], H,
                                                               fmt=fmt, bucket_size=B, outputs=[c0],
                                                               output_scales=[s0])
            assert_codes(codes.cpu(), ref_c[0], f"routed {dtype} {fmt} H={H}")
            assert_same(scales.cpu().reshape(-1), ref_s[0], f"routed {dtype} {fmt} H={H}")
        # the refusals on CUDA tensors
        x = torch.randn(8, 512, device="cuda")
        codes = torch.empty(8, 512, dtype=torch.float8_e4m3fn, device="cuda")
        good = torch.empty(8, 4, device="cuda")
        for bad in (good.double(), good[:, :2], torch.empty(4, 8, device="cuda").t(), good.cpu(),
                    torch.empty(7, 4, device="cuda")):
            with pytest.raises(ValueError, match="output_scales"):
                cgx.all_to_all_single(codes, x, bits="e4m3", bucket_size=128, output_scales=bad)
        for kw in (dict(bits=8), dict(bits="e5m2"), dict(bits="e4m3", stochastic=True), dict(bits="e4m3", bucket_size=100)):
            kw.setdefault("bucket_size", 128)
            with pytest.raises(ValueError):
                cgx.all_to_all_single(codes, x, output_scales=good, **kw)
        flat = torch.empty(8 * 512 + 64, device="cuda")
        with pytest.raises((ValueError, RuntimeError), match="overlap"):
            cgx.all_to_all_single(codes, flat[:4096].view(8, 512), bits="e4m3", bucket_size=128,
                                  output_scales=flat[8:40].view(8, 4))
        # index_copy_ on float8, which the codes composition avoids by moving bytes
        t = torch.zeros(4, 3, dtype=torch.float8_e4m3fn, device="cuda")
        try:
            t.index_copy_(0, torch.tensor([1], device="cuda"), torch.ones(1, 3, device="cuda").to(t.dtype))
            print("index_copy_ on float8_e4m3fn (cuda): supported")
        except RuntimeError as e:
            print(f"index_copy_ on float8_e4m3fn (cuda): {str(e).splitlines()[0]}")
    finally:
        dist.destroy_process_group()


def test_public_api_world1():
    spawn(_pg_world1, 1)


# ---- the GEMM contract --------------------------------------------------------------------------------
def test_rowwise_scaled_mm_contract():
    """bucket = H: one scale per row, what torch._scaled_mm takes as row-wise scaling. The call's codes
    and scales and the oracle's give the same bf16 product, close to an fp32 matmul of the decoded
    values."""
    W, H, N, dtype = 2, 7168, 256, torch.bfloat16
    g = torch.Generator().manual_seed(4)
    c = [[64 * H, 64 * H], [64 * H, 64 * H]]
    xs = [torch.randn(128 * H, generator=g).to(dtype) for _ in range(W)]
    codes, scales = run_fused(make_group(W, dtype), xs, c, "e4m3", H)
    ref_c, ref_s = O.all_to_all_codes_reference(xs, c, fmt="e4m3", bucket_size=H)
    w = torch.randn(N, H, generator=g) * 0.05
    w_scale = w.abs().amax(dim=1, keepdim=True) / 448.0
    w8 = (w / w_scale).to(torch.float8_e4m3fn).to(dev())
    for r in range(W):
        a = codes[r].reshape(-1, H).to(dev())
        sa = scales[r].reshape(-1, 1).to(dev())
        out = torch._scaled_mm(a, w8.t(), scale_a=sa, scale_b=w_scale.reshape(1, -1).to(dev()),
                               out_dtype=torch.bfloat16)
        out_ref = torch._scaled_mm(ref_c[r].reshape(-1, H).to(dev()), w8.t(), scale_a=ref_s[r].reshape(-1, 1).to(dev()),
                                   scale_b=w_scale.reshape(1, -1).to(dev()), out_dtype=torch.bfloat16)
        assert_same(out.cpu(), out_ref.cpu(), f"rank {r}")
        exact = (a.float() * sa) @ (w8.float() * w_scale.to(dev())).t()
        torch.testing.assert_close(out.float(), exact, rtol=2e-2, atol=2e-2 * exact.abs().max().item())


# ---- several GPUs -----------------------------------------------------------------------------------------
def _pg_codes(rank, world, transport):
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        H, B, fmt = 1024, 128, "e4m3"
        rows = [[(q + 2 * r) % 5 + 1 for r in range(world)] for q in range(world)]
        g = torch.Generator().manual_seed(0)
        xs = [torch.randn(sum(rows[q]) * H, generator=g).to(torch.bfloat16) for q in range(world)]
        c = [[v * H for v in row] for row in rows]
        ref_c, ref_s = O.all_to_all_codes_reference(xs, c, fmt=fmt, bucket_size=B)
        recv = sum(rows[q][rank] for q in range(world))
        codes = torch.empty(recv, H, dtype=TDT[fmt], device="cuda")
        scales = torch.empty(recv, H // B, device="cuda")
        cgx.all_to_all_single(codes, xs[rank].reshape(-1, H).cuda(), [rows[q][rank] for q in range(world)], rows[rank],
                              bits=fmt, bucket_size=B, output_scales=scales)
        assert_codes(codes.cpu(), ref_c[rank], f"rank {rank}")
        assert_same(scales.cpu().reshape(-1), ref_s[rank], f"rank {rank}")
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("transport", ["P2P", "NCCL"])
def test_public_api_codes_multigpu(world, transport):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_codes, world, args=(transport,), env={"CGX_INNER_COMMUNICATOR_TYPE": transport})
