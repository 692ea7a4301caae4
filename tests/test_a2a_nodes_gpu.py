"""The compressed all-to-all over several nodes on one GPU: C.LocalEngineGroup runs W real engines
as N virtual nodes of L ranks, with the node-local stage on heaps (the fused kernel) or through the
generic reducer, and the cross-node chunks through the pack and unpack kernels and a loopback
exchange. Every result is the one-node all-to-all of W ranks, bit for bit. The routed, scaled,
combine and indexed-codes forms run through a2a_compose, the composition the process group uses
over several nodes. With several GPUs (``-m multigpu``, CGX_LOCAL_SIZE=2): the public API, the
differentiable dispatch and the combine against the references."""
from __future__ import annotations

import os

import pytest
import torch
import torch.distributed as dist

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same
from _dist_utils import spawn
from _engine_cases import C, TIMEOUT_MS, clean_environment  # noqa: F401

pytestmark = pytest.mark.gpu

TOPOLOGIES = ((2, 1), (2, 2), (2, 4), (3, 2), (4, 4), (2, 8), (3, 8))
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BITS = (2, 4, 8, 32, "e4m3", "e5m2")
DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def row_counts(world, H, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "equal":
        rows = [[3] * world for _ in range(world)]
    elif kind == "skewed":
        rows = torch.randint(0, 6, (world, world), generator=g).tolist()
        rows[0] = [9] * world
    else:  # zero: some pairs and one whole rank send nothing
        rows = torch.randint(0, 3, (world, world), generator=g).tolist()
        rows[world - 1] = [0] * world
        for q in range(world):
            rows[q][0] = 0
    return [[n * H for n in row] for row in rows]


def make_inputs(c, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(sum(row), generator=g) * (q + 1)).to(dtype).cuda() for q, row in enumerate(c)]


def make_outputs(c, dtype):
    W = len(c)
    return [torch.full((sum(c[q][r] for q in range(W)),), float("nan"), dtype=dtype, device="cuda")
            for r in range(W)]


def group(N, L, fused):
    return C.LocalEngineGroup(N * L, L, dict(p2p=fused), 1, 1 << 20, TIMEOUT_MS)


def run_and_check(g, c, dtype, bits, bucket, seed=0):
    ins, outs = make_inputs(c, dtype, seed), make_outputs(c, dtype)
    g.all_to_all(ins, outs, c, bits=bits, bucket_size=bucket)
    ref = O.all_to_all_reference([x.cpu() for x in ins], c, bits=bits, bucket_size=bucket)
    for r in range(len(c)):
        assert_same(outs[r].cpu(), ref[r], f"rank {r}")
    return ins, outs


@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
@pytest.mark.parametrize("N,L", TOPOLOGIES)
def test_topologies(N, L, fused):
    g = group(N, L, fused)
    for i, (dtype, bits) in enumerate(((torch.bfloat16, 4), (torch.float16, "e4m3"), (torch.float32, 32))):
        run_and_check(g, row_counts(N * L, 1024, "skewed", seed=i), dtype, bits, 512, seed=i)
    log = g.log(0)
    assert [e["kind"] for e in log] == ["a2a_intra", "a2a_cross"]


@pytest.mark.parametrize("bucket", (128, 512, 1024))
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_dtypes_bits_buckets(dtype, bits, bucket):
    run_and_check(group(2, 4, True), row_counts(8, 640, "skewed", seed=7), dtype, bits, bucket)


@pytest.mark.parametrize("kind", ("equal", "skewed", "zero"))
@pytest.mark.parametrize("H", (7168, 1024, 640, 7))
@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_rows_and_splits(H, kind, fused):
    c = row_counts(6, H, kind, seed=H)
    if H == 7168 and kind != "zero":
        c = [[min(n, 2 * H) for n in row] for row in c]
    run_and_check(group(3, 2, fused), c, torch.bfloat16, 4, 512)


@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_stochastic_matches_the_simulator(fused, monkeypatch):
    N, L = 3, 8  # W = 24: pairs whose ranks agree mod 16 get distinct streams
    g = group(N, L, fused)
    c = row_counts(N * L, 512, "skewed", seed=3)
    ins, outs = make_inputs(c, torch.float32, 1), make_outputs(c, torch.float32)
    g.all_to_all(ins, outs, c, bits=3, bucket_size=128, stochastic=True, seed=11)
    seq = g.log(0)[0]["seq"]
    assert all(g.log(r)[0]["seq"] == seq for r in range(N * L))
    sim_out = [o.cpu().clone() for o in make_outputs(c, torch.float32)]
    C.all_to_all_simulate([x.cpu() for x in ins], sim_out, c, bits=3, bucket_size=128, stochastic=True, seed=11,
                          seq=seq)
    for r in range(N * L):
        assert_same(outs[r].cpu(), sim_out[r], f"rank {r}")


@pytest.mark.parametrize("fmt", ("e4m3", "e5m2"))
@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_codes_output(fmt, fused):
    N, L, H, B = 2, 2, 1024, 128
    g = group(N, L, fused)
    c = row_counts(N * L, H, "skewed", seed=5)
    ins = make_inputs(c, torch.bfloat16, 2)
    W = N * L
    codes = [torch.full((sum(c[q][r] for q in range(W)),), 0x7F, dtype=torch.uint8, device="cuda")
             .view(O.FP8_FORMATS[fmt][0]) for r in range(W)]
    scales = [torch.full((x.numel() // H, H // B), float("nan"), device="cuda") for x in codes]
    g.all_to_all(ins, codes, c, bits=fmt, bucket_size=B, output_scales=scales)
    ref_c, ref_s = O.all_to_all_codes_reference([x.cpu() for x in ins], c, fmt=fmt, bucket_size=B)
    for r in range(W):
        assert torch.equal(codes[r].cpu().view(torch.uint8), ref_c[r].view(torch.uint8)), f"rank {r} codes"
        assert_same(scales[r].cpu().reshape(-1), ref_s[r], f"rank {r} scales")


@pytest.mark.parametrize("bits", (2, 4, 8, 5))
@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16))
def test_pack_matches_the_generic_records(dtype, bits):
    """Every region of the send buffer holds the bytes the generic reducer's quantizer writes for the
    chunk (a one-layer plan of it), at even and odd chunk offsets."""
    W, L, rank = 6, 2, 2
    counts = [1031, 0, 517, 64, 3001, 77]  # the remote chunks start at elements 0, 1612 and 4613
    x = torch.randn(sum(counts), device="cuda").to(dtype)
    buf = C.a2a_pack(x, counts, rank, L, bits, 128)
    wire, region, _ = C.a2a_remote_wire(counts, rank, L, bits, 128, DTYPE_CODE[dtype])
    off = 0
    for q, n in enumerate(counts):
        if wire[q]:
            ref = C.quantize(x[off:off + n].contiguous(), [(0, n, bits, 128)])
            assert torch.equal(buf[region[q]:region[q] + wire[q]].cpu(), ref.view(-1)[:wire[q]].cpu()), q
        off += n


@pytest.mark.parametrize("bits", (4, "e4m3"))
@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16))
def test_unpack_at_odd_offsets_keeps_the_guards(dtype, bits):
    """Pack from and unpack into views at an odd element offset inside sentinel-filled buffers."""
    W, L, rank = 4, 2, 0
    counts = [3, 0, 1029, 515]
    n = sum(counts)
    x = torch.randn(n + 2, device="cuda").to(dtype)[1:1 + n]
    buf = C.a2a_pack(x, counts, rank, L, bits, 128)
    big = torch.full((n + 34,), 7.0, dtype=dtype, device="cuda")
    out = big[17:17 + n]
    C.a2a_unpack(buf, out, counts, rank, L, bits, 128)
    torch.cuda.synchronize()
    assert torch.all(big[:17] == 7.0) and torch.all(big[17 + n:] == 7.0)
    off = 0
    for q, c in enumerate(counts):
        if q // L != rank // L and c:
            want = (O.fp8_quantize_dequantize(x[off:off + c].cpu(), bits, 128) if isinstance(bits, str)
                    else O.quantize_dequantize_layers(x[off:off + c].cpu(), [(0, c, bits, 128)]))
            assert_same(out[off:off + c].cpu(), want, f"chunk {q}")
        else:
            assert torch.all(out[off:off + c] == 7.0)
        off += c


# ---- the routed forms over several nodes, through the process group's composition -------------------
FILL = -7.0


def routed_case(W, H, seed):
    """Per rank: T input rows, the rows it sends by input_index, fp32 input_scale, and an output of
    received rows + 4 written through a partial permutation output_index. 2 rows per pair."""
    g = torch.Generator().manual_seed(seed)
    rows = [[2] * W for _ in range(W)]
    c = [[n * H for n in row] for row in rows]
    T = 5
    xs, iis, scs, ois, outs = [], [], [], [], []
    for r in range(W):
        nsend, nrecv = sum(rows[r]), sum(rows[q][r] for q in range(W))
        xs.append(torch.randn(T, H, generator=g))
        iis.append(torch.randint(0, T, (nsend,), generator=g))
        scs.append(torch.randn(nsend, generator=g))
        ois.append(torch.randperm(nrecv + 4, generator=g)[:nrecv])
        outs.append(nrecv + 4)
    return c, xs, iis, scs, ois, outs


@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
@pytest.mark.parametrize("N,L", ((2, 2), (3, 8)))
def test_routed_and_scaled_forms(N, L, fused):
    W, H = N * L, 1024
    g = group(N, L, fused)
    for dtype, bits, scaled in ((torch.bfloat16, 4, False), (torch.float16, "e4m3", True), (torch.float32, 8, True)):
        c, xs, iis, scs, ois, nout = routed_case(W, H, seed=W)
        ins = [x.to(dtype).cuda() for x in xs]
        outs = [torch.full((n, H), FILL, dtype=dtype, device="cuda") for n in nout]
        g.all_to_all(ins, outs, c, bits=bits, bucket_size=512, input_index=[i.cuda() for i in iis],
                     output_index=[o.cuda() for o in ois], input_scale=[s.cuda() for s in scs] if scaled else [],
                     row=H)
        ref = O.routed_all_to_all_reference([x.cpu() for x in ins], c, iis, ois, H, bits=bits, bucket_size=512,
                                            outputs=[torch.full((n, H), FILL, dtype=dtype) for n in nout],
                                            input_scale=scs if scaled else None)
        for r in range(W):
            assert_same(outs[r].cpu().reshape(-1), ref[r], f"{dtype} {bits} rank {r}")


@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
def test_routed_codes_output(fused):
    N, L, H, B, fmt = 2, 2, 1024, 128, "e5m2"
    W = N * L
    g = group(N, L, fused)
    c, xs, iis, _, ois, nout = routed_case(W, H, seed=1)
    ins = [x.to(torch.bfloat16).cuda() for x in xs]
    f8 = O.FP8_FORMATS[fmt][0]
    codes = [torch.full((n, H), 0x55, dtype=torch.uint8, device="cuda").view(f8) for n in nout]
    scales = [torch.full((n, H // B), 3.0, device="cuda") for n in nout]
    g.all_to_all(ins, codes, c, bits=fmt, bucket_size=B, output_scales=scales, input_index=[i.cuda() for i in iis],
                 output_index=[o.cuda() for o in ois], row=H)
    ref_c, ref_s = O.routed_all_to_all_codes_reference(
        [x.cpu() for x in ins], c, iis, ois, H, fmt=fmt, bucket_size=B,
        outputs=[torch.full((n, H), 0x55, dtype=torch.uint8).view(f8) for n in nout],
        output_scales=[torch.full((n, H // B), 3.0) for n in nout])
    for r in range(W):
        assert torch.equal(codes[r].cpu().view(torch.uint8).reshape(-1), ref_c[r].view(torch.uint8)), f"rank {r}"
        assert_same(scales[r].cpu().reshape(-1), ref_s[r], f"rank {r} scales")


@pytest.mark.parametrize("fused", (True, False), ids=("fused", "generic"))
@pytest.mark.parametrize("N,L", ((2, 2), (3, 8)))
def test_combine_form(N, L, fused):
    W, H, k = N * L, 1024, 2
    g = group(N, L, fused)
    gen = torch.Generator().manual_seed(3)
    rows = [[2] * W for _ in range(W)]  # every rank receives 2 W = T k slot rows
    c = [[n * H for n in row] for row in rows]
    T = 2 * W // k
    for dtype, bits in ((torch.bfloat16, 4), (torch.float32, "e4m3")):
        ins = [torch.randn(2 * W, H, generator=gen).to(dtype).cuda() for _ in range(W)]
        ois = [torch.randperm(T * k, generator=gen) for _ in range(W)]
        gates = [torch.rand(T, k, generator=gen) for _ in range(W)]
        slots = [torch.full((T * k, H), FILL, dtype=dtype, device="cuda") for _ in range(W)]
        outs = [torch.full((T, H), FILL, dtype=dtype, device="cuda") for _ in range(W)]
        g.all_to_all(ins, slots, c, bits=bits, bucket_size=512, output_index=[o.cuda() for o in ois],
                     gate=[x.cuda() for x in gates], combine_out=outs, row=H)
        ref_slots, ref_out = O.routed_all_to_all_combine_reference([x.cpu() for x in ins], c, ois, gates, H, bits=bits,
                                                                   bucket_size=512)
        for r in range(W):
            assert_same(slots[r].cpu().reshape(-1), ref_slots[r], f"{dtype} slots rank {r}")
            assert_same(outs[r].cpu().reshape(-1), ref_out[r], f"{dtype} combine rank {r}")


# ---- several GPUs, CGX_LOCAL_SIZE nodes ------------------------------------------------------------------
def _pg_nodes(rank, world):
    local = int(os.environ["CGX_LOCAL_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        assert cgx.get_backend().local_size() == local
        H = 1024
        c, xs, iis, scs, ois, nout = routed_case(world, H, seed=world)  # the same on every rank
        rows = [n // H for n in c[rank]]
        recv_rows = [c[q][rank] // H for q in range(world)]
        for dtype, bits in ((torch.bfloat16, 4), (torch.float16, "e4m3"), (torch.float32, 32)):
            ins = [x.to(dtype) for x in xs]
            # plain: every input row in destination order
            plain_in = [x.index_select(0, i) for x, i in zip(ins, iis)]
            out = torch.full((sum(recv_rows), H), FILL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, plain_in[rank].cuda(), recv_rows, rows, bits=bits, bucket_size=512)
            ref = O.all_to_all_reference([x.reshape(-1) for x in plain_in], c, bits=bits, bucket_size=512)
            assert_same(out.cpu().reshape(-1), ref[rank], f"plain {dtype} {bits}")
            # routed and scaled
            out = torch.full((nout[rank], H), FILL, dtype=dtype, device="cuda")
            cgx.all_to_all_single(out, ins[rank].cuda(), recv_rows, rows, bits=bits, bucket_size=512,
                                  input_index=iis[rank].cuda(), output_index=ois[rank].cuda(),
                                  input_scale=scs[rank].cuda())
            ref = O.routed_all_to_all_reference(ins, c, iis, ois, H, bits=bits, bucket_size=512,
                                                outputs=[torch.full((n, H), FILL, dtype=dtype) for n in nout],
                                                input_scale=scs)
            assert_same(out.cpu().reshape(-1), ref[rank], f"routed {dtype} {bits}")
            # the differentiable dispatch: forward, and the gradient sent back with the splits swapped
            x = plain_in[rank].cuda().requires_grad_()
            y = cgx.differentiable_all_to_all_single(x, recv_rows, rows, bits=bits, bucket_size=512)
            ref = O.all_to_all_reference([p.reshape(-1) for p in plain_in], c, bits=bits, bucket_size=512)
            assert_same(y.detach().cpu().reshape(-1), ref[rank], f"dispatch {dtype} {bits}")
            grads = [torch.randn(sum(c[q][r] for q in range(world)) // H, H,
                                 generator=torch.Generator().manual_seed(100 + r)).to(dtype) for r in range(world)]
            y.backward(grads[rank].cuda())
            back = O.all_to_all_reference([gr.reshape(-1) for gr in grads], [list(col) for col in zip(*c)], bits=bits,
                                          bucket_size=512)
            assert_same(x.grad.cpu().reshape(-1), back[rank], f"dispatch grad {dtype} {bits}")
        # the codes output
        fmt, B = "e4m3", 128
        src = [x.to(torch.bfloat16).index_select(0, i) for x, i in zip(xs, iis)]
        codes = torch.empty(sum(recv_rows), H, dtype=O.FP8_FORMATS[fmt][0], device="cuda")
        scales = torch.empty(sum(recv_rows), H // B, device="cuda")
        cgx.all_to_all_single(codes, src[rank].cuda(), recv_rows, rows, bits=fmt, bucket_size=B, output_scales=scales)
        ref_c, ref_s = O.all_to_all_codes_reference([s.reshape(-1) for s in src], c, fmt=fmt, bucket_size=B)
        assert torch.equal(codes.cpu().view(torch.uint8).reshape(-1), ref_c[rank].view(torch.uint8)), "codes"
        assert_same(scales.cpu().reshape(-1), ref_s[rank], "scales")
        # the combine and its differentiable form (forward)
        k = 2
        T = sum(recv_rows) // k
        gen = torch.Generator().manual_seed(7)
        sl_in = [torch.randn(sum(c[q]) // H, H, generator=gen) for q in range(world)]
        perms = [torch.randperm(T * k, generator=gen) for _ in range(world)]
        gates = [torch.rand(T, k, generator=gen) for _ in range(world)]
        ref_slots, ref_out = O.routed_all_to_all_combine_reference(sl_in, c, perms, gates, H, bits=4, bucket_size=512)
        out = torch.full((T, H), FILL, device="cuda")
        cgx.all_to_all_combine(out, sl_in[rank].cuda(), gates[rank].cuda(), perms[rank].cuda(), recv_rows, rows,
                               bits=4, bucket_size=512)
        assert_same(out.cpu().reshape(-1), ref_out[rank], "combine")
        y = cgx.differentiable_all_to_all_combine(sl_in[rank].cuda(), gates[rank].cuda(), perms[rank].cuda(),
                                                  recv_rows, rows, bits=4, bucket_size=512)
        assert_same(y.detach().cpu().reshape(-1), ref_out[rank], "differentiable combine")
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_public_api_across_nodes():
    world, local = 4, 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    spawn(_pg_nodes, world, env={"CGX_LOCAL_SIZE": str(local)}, timeout=600)
