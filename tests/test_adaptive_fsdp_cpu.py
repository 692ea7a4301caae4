"""Adaptive FSDP2 widths without a GPU: the sharded mode of the CPU quantization-error estimator
against per-chunk calls and the quantize -> dequantize round trip, and AdaptiveFSDPState at world 2
on the cgx CPU path (CGX_COMPRESS_CPU=1), driven through its estimate and pre-forward entry points
with CPU buffers."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from _dist_utils import spawn

CANDS = (2, 3, 4, 5, 6, 7, 8)
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def _shard_table(S):
    """Layers of one shard at unaligned offsets, buckets of 13 (tail), 100, 512 and 20000 (clamped)."""
    layers, off = [], 3
    for n, b in ((777, 13), (1000, 100), (1500, 512), (S - 3300, 20000)):
        layers.append((off, n, 4, b))
        off += n + 3
    assert off <= S
    return layers


def _inputs(chunks, S, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    scale = torch.tensor([0.01 * 10 ** (c % 4) for c in range(chunks)])  # chunks of different ranges
    x = torch.randn(chunks, S, generator=g) * scale[:, None]
    return x.reshape(-1).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("chunks", [2, 3, 8])
@pytest.mark.parametrize("mode", ["nearest", "skip_incomplete", "stochastic"])
def test_sharded_rows_are_per_chunk_sums(dtype, chunks, mode):
    from torch_cgx_b200.ops import quantization_error

    S = 4400
    layers = _shard_table(S)
    t = _inputs(chunks, S, dtype)
    kw = dict(stochastic=mode == "stochastic", skip_incomplete=mode == "skip_incomplete", prescale=1.0 / chunks)
    per = [quantization_error(t[c * S:(c + 1) * S], layers, CANDS, **kw).numpy() for c in range(chunks)]
    for skip in range(-1, chunks):
        got = quantization_error(t, layers, CANDS, chunks=chunks, skip_chunk=skip, **kw).numpy()
        want = sum(p for c, p in enumerate(per) if c != skip)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=f"skip_chunk {skip}")


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("chunks", [2, 3, 8])
def test_sharded_rows_match_round_trip(dtype, chunks):
    from torch_cgx_b200.ops import oracle as O
    from torch_cgx_b200.ops import quantization_error

    S = 4400
    layers = _shard_table(S)
    t = _inputs(chunks, S, dtype, seed=1)
    ps = float(np.float32(1) / np.float32(chunks))
    for skip in (-1, chunks - 1, 0):
        want = np.zeros((len(layers), len(CANDS)))
        for c in range(chunks):
            if c == skip:
                continue
            x = t[c * S:(c + 1) * S].float() * ps  # the prescaled fp32 values the encoder sees
            for k, bits in enumerate(CANDS):
                table = [(o, n, bits, b) for (o, n, _, b) in layers]
                rt = O.quantize_dequantize_layers(x, table).double()  # fp32 round trip
                for l, (o, n, _, _) in enumerate(layers):
                    want[l, k] += ((rt[o:o + n] - x[o:o + n].double()) ** 2).sum().item()
        got = quantization_error(t, layers, CANDS, prescale=ps, chunks=chunks, skip_chunk=skip).numpy()
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=0, err_msg=f"skip_chunk {skip}")


def test_sharded_non_finite_bucket_poisons_only_its_layer():
    from torch_cgx_b200.ops import quantization_error

    S, chunks = 4400, 4
    layers = _shard_table(S)
    t = _inputs(chunks, S, torch.float32)
    t[2 * S + layers[1][0] + 5] = float("nan")
    t[2 * S + layers[2][0] + 600] = float("inf")
    for skip in range(-1, chunks):
        e = quantization_error(t, layers, CANDS, chunks=chunks, skip_chunk=skip)
        bad = torch.isnan(e).all(dim=1).tolist()
        assert bad == ([False] * 4 if skip == 2 else [False, True, True, False]), (skip, bad)
        assert torch.isfinite(e[[0, 3]]).all()


def test_sharded_estimator_rejects_bad_arguments():
    from torch_cgx_b200.ops import quantization_error

    t = torch.randn(1000)
    with pytest.raises(RuntimeError, match="chunks"):
        quantization_error(t, [(0, 100, 4, 64)], chunks=3)  # 1000 is not divisible by 3
    with pytest.raises(RuntimeError, match="chunk of 250"):
        quantization_error(t, [(200, 100, 4, 64)], chunks=4)  # reaches past S = 250
    for skip in (-2, 4):
        with pytest.raises(RuntimeError, match="skip_chunk"):
            quantization_error(t, [(0, 100, 4, 64)], chunks=4, skip_chunk=skip)
    with pytest.raises(RuntimeError, match="chunks"):
        quantization_error(t, [(0, 100, 4, 64)], chunks=0)
    # chunks=1 is the plain table; skipping the only chunk leaves nothing
    a = quantization_error(t, [(0, 1000, 4, 64)])
    assert torch.equal(quantization_error(t, [(0, 1000, 4, 64)], chunks=1, skip_chunk=-1), a)
    assert torch.equal(quantization_error(t, [(0, 1000, 4, 64)], chunks=1, skip_chunk=0), torch.zeros_like(a))


# ---- AdaptiveFSDPState at world 2 ----------------------------------------------------------------
S_MOD = 2560
SCALES = (0.01, 3.0, 0.2, 50.0)


def _module_table(bits):
    """One module's shard table: four weights of very different scales and a raw bias."""
    from torch_cgx_b200 import fsdp_shard_table

    return fsdp_shard_table([((32, 16), 512), ((8,), 8), ((32, 16), 512), ((64, 12), 768), ((24, 32), 760)],
                            bits, 64)


NAMES = ["m.w0", "m.b", "m.w1", "m.w2", "m.w3"]


def _shard(rank, step, table):
    g = torch.Generator().manual_seed(100 * step + rank)
    x = torch.zeros(sum(l[1] for l in table))
    for (o, n, b, _), s in zip([l for l in table if l[2] <= 8], SCALES):
        x[o:o + n] = torch.randn(n, generator=g) * s
    return x


def _world2_state(rank, world):
    import torch_cgx_b200 as cgx
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes

    dist.init_process_group("cgx", init_method="env://", rank=rank, world_size=world)
    try:
        group = dist.group.WORLD
        st = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=6, bucket_size=64, period=3)
        ag = cgx.CGXAllGather(6, 64, _module_table(6), "m")
        rs = cgx.CGXReduceScatter(4, 64, False, _module_table(4), "m")
        st.register(ag, "all_gather", NAMES)
        st.register(rs, "reduce_scatter", NAMES)
        assert st.rows("all_gather") == ["m.w0", "m.w1", "m.w2", "m.w3"]
        assert ag.adaptive is st and rs.adaptive is st
        uniform = {("all_gather", n): 6 for n in st.rows("all_gather")}
        uniform.update({("reduce_scatter", n): 4 for n in st.rows("reduce_scatter")})
        assert st.assignment == uniform

        changed_at, widths = [], [(list(ag.layers), list(rs.layers))]
        # the reduce-scatter runs on steps 0, 1, 4, 5 (gradient accumulation: no sync at steps 2 and 3)
        rs_steps = {0, 1, 4, 5}
        for step in range(7):
            st.pre_forward()
            now = (list(ag.layers), list(rs.layers))
            if now != widths[-1]:
                changed_at.append(step)
            widths.append(now)
            shard = _shard(rank, step, ag.layers)
            st.maybe_estimate(ag, shard, group, average=False)
            if step in rs_steps:
                full = torch.cat([_shard(rank, 10 + step, rs.layers) * (q + 1) for q in range(world)])
                st.maybe_estimate(rs, full, group, average=True)
            assert (list(ag.layers), list(rs.layers)) == widths[-1]  # widths change only in pre_forward
            if step == 3:
                # the all-gather estimated in this round, the reduce-scatter did not: still open
                assert st._round_open and id(rs) not in st._tables
        # round 1 opens at step 0 and is decided at step 1; round 2 opens at step 3, the
        # reduce-scatter estimates at step 4, the decision runs at step 5; round 3 opens at step 6
        assert st.step == 7 and st._round_open
        assert set(changed_at) <= {1, 5}, changed_at
        assert 1 in changed_at
        for kind, comm, target in (("all_gather", ag, 6), ("reduce_scatter", rs, 4)):
            adapted = [l for l in comm.layers if l[2] <= 8]
            assert len({l[2] for l in adapted}) > 1, comm.layers
            assert sum(layer_wire_bytes(l[1], l[2], 64) for l in adapted) <= \
                sum(layer_wire_bytes(l[1], target, 64) for l in adapted)
            assert comm.layers[1][2] == 32  # the bias stays raw
            assert st.last_errors[kind].shape == (4, len(CANDS)) and st.last_errors[kind].dtype == torch.float64
            for (_, n, bits, _), name in zip(adapted, st.rows(kind)):
                assert st.assignment[(kind, name)] == bits
        # the largest scale gets the most bits
        ag_bits = [l[2] for l in ag.layers if l[2] <= 8]
        assert ag_bits[3] == max(ag_bits) and ag_bits[0] == min(ag_bits)
        both = [None] * world
        dist.all_gather_object(both, sorted(st.assignment.items()))
        assert both[0] == both[1]

        # a single candidate keeps the uniform table
        one = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=4, bucket_size=64,
                                    candidate_bits=(4,), period=1)
        ag1 = cgx.CGXAllGather(4, 64, _module_table(4), "m")
        one.register(ag1, "all_gather", NAMES)
        before = list(ag1.layers)
        for step in range(3):
            one.pre_forward()
            one.maybe_estimate(ag1, _shard(rank, step, ag1.layers), group, average=False)
        assert one.last_errors["all_gather"].shape == (4, 1) and ag1.layers == before

        # checkpoint: a fresh state loaded before install applies the widths at install
        sd = st.state_dict()
        assert sd["step"] == 7 and set(sd["assignment"]) == {"all_gather", "reduce_scatter"}
        st2 = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=6, bucket_size=64, period=3)
        st2.load_state_dict(sd)
        ag2 = cgx.CGXAllGather(6, 64, _module_table(6), "m")
        rs2 = cgx.CGXReduceScatter(4, 64, False, _module_table(4), "m")
        st2.register(ag2, "all_gather", NAMES)
        st2.register(rs2, "reduce_scatter", NAMES)
        assert ag2.layers == ag.layers and rs2.layers == rs.layers
        assert st2.state_dict() == sd
        # and after install, at once
        st3 = cgx.AdaptiveFSDPState(reduce_scatter_bits=4, all_gather_bits=6, bucket_size=64)
        ag3 = cgx.CGXAllGather(6, 64, _module_table(6), "m")
        st3.register(ag3, "all_gather", NAMES)
        st3.load_state_dict({"assignment": {"all_gather": sd["assignment"]["all_gather"]}, "step": 7})
        assert ag3.layers == ag.layers
        for bad in ({"assignment": {"broadcast": {}}},
                    {"assignment": {"all_gather": {"m.w0": 9}}},
                    {"assignment": {"all_gather": {"m.w0": 0}}},
                    {"assignment": {"all_gather": {"nope": 4}}}):
            with pytest.raises(ValueError):
                st3.load_state_dict(bad)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_adaptive_fsdp_state_world2_cpu():
    spawn(_world2_state, 2, env={"CGX_COMPRESS_CPU": "1"})


def test_adaptive_fsdp_state_rejects_bad_arguments():
    import torch_cgx_b200 as cgx

    for kw in ({"reduce_scatter_bits": 9}, {"all_gather_bits": 0}, {"candidate_bits": ()},
               {"candidate_bits": (2, 9)}, {"period": 0}, {"bucket_size": 0},
               {"reduce_scatter_bits": None, "all_gather_bits": None}):
        with pytest.raises(ValueError):
            cgx.AdaptiveFSDPState(**kw)
    st = cgx.AdaptiveFSDPState()
    with pytest.raises(ValueError):
        st.register(cgx.CGXAllGather(6, 64, _module_table(6)), "broadcast", NAMES)
    with pytest.raises(ValueError):
        st.register(cgx.CGXAllGather(6, 64, _module_table(6)), "all_gather", NAMES[:2])
    with pytest.raises(ValueError, match="FSDP root"):
        cgx.set_cgx_adaptive(torch.nn.Linear(4, 4), st)
