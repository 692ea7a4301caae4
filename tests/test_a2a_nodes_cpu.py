"""The compressed all-to-all over several nodes, without a GPU: the random stream keys of every pair
of world ranks, the simulator past 16 ranks against the oracle, the record bytes each remote chunk
travels as, and the refusals that need no device."""
from __future__ import annotations

import pytest
import torch

from torch_cgx_b200.ops import oracle as O

import _a2a_cases as A
from _bitwise import assert_same
from _engine_cases import C, TIMEOUT_MS, clean_environment  # noqa: F401

MAX_WORLD = 256


def test_stream_keys_below_16_ranks_are_unchanged():
    for s in range(16):
        for d in range(16):
            assert C.a2a_rng_stream(s, d) == 2 * (s * 16 + d)


def test_stream_keys_are_distinct_up_to_the_world_limit():
    assert C.A2A_MAX_WORLD == MAX_WORLD
    words = {C.a2a_rng_stream(s, d) for s in range(MAX_WORLD) for d in range(MAX_WORLD)}
    assert len(words) == MAX_WORLD * MAX_WORLD
    for w in words:
        # even (phase 0), below 2^17: the low parts in bits 0..8, the high parts in bits 9..16
        assert w % 2 == 0 and w < (1 << 17)
    # the key multiplies the word by an odd constant: distinct words are distinct keys
    assert len({(w * 0x9E3779B9) & 0xFFFFFFFF for w in words}) == len(words)


@pytest.mark.parametrize("world", (17, 24, 33))
@pytest.mark.parametrize("bits", (2, 4, 8, 32, "e4m3", "e5m2"))
@pytest.mark.parametrize("dtype", A.DTYPES)
def test_simulator_past_16_ranks_matches_the_oracle(world, bits, dtype):
    c = A.counts(world, "uneven", 70, seed=world)
    ins = A.inputs(c, dtype, seed=3)
    outs = A.outputs(c, dtype)
    C.all_to_all_simulate(ins, outs, c, bits=bits, bucket_size=64)
    ref = O.all_to_all_reference(ins, c, bits=bits, bucket_size=64)
    for r in range(world):
        assert_same(outs[r], ref[r], f"rank {r}")


def test_stochastic_simulator_past_16_ranks_keys_every_pair():
    """Two pairs whose ranks agree mod 16 get different rounding: the high parts reach the key."""
    world, n = 34, 4096
    c = [[n] * world for _ in range(world)]
    x = torch.randn(n, generator=torch.Generator().manual_seed(0))
    ins = [x.repeat(world) for _ in range(world)]
    outs = A.outputs(c, torch.float32)
    C.all_to_all_simulate(ins, outs, c, bits=2, bucket_size=128, stochastic=True, seed=5, seq=16)
    chunk = lambda r, q: outs[r][q * n:(q + 1) * n]  # noqa: E731
    assert not torch.equal(chunk(1, 0), chunk(1, 16))   # sources 0 and 16, same destination
    assert not torch.equal(chunk(1, 2), chunk(17, 2))   # destinations 1 and 17, same source
    # below 16 ranks the streams are those of a world of 16
    c16 = [[n] * 16 for _ in range(16)]
    outs16 = A.outputs(c16, torch.float32)
    C.all_to_all_simulate([x.repeat(16) for _ in range(16)], outs16, c16, bits=2, bucket_size=128, stochastic=True,
                          seed=5, seq=16)
    assert_same(chunk(3, 5), outs16[3][5 * n:6 * n], "pair (5, 3)")


@pytest.mark.parametrize("bits", (2, 4, 8, "e4m3", 32))
@pytest.mark.parametrize("local", (1, 2, 8))
def test_wire_bytes_per_destination(bits, local):
    world = 3 * local
    counts = [(q * 997) % 5000 for q in range(world)]
    counts[1] = 0
    rank = local  # node 1
    dt = 2
    wire, region, total = C.a2a_remote_wire(counts, rank, local, bits, 512, dt)
    off = 0
    for q, n in enumerate(counts):
        if q // local == rank // local or n == 0:
            assert wire[q] == 0
            continue
        if bits == 32:
            assert wire[q] == 2 * n
            continue
        b = 8 if isinstance(bits, str) else bits
        plan = C.build_plan([(0, n, b, 512)], 1, 1, dt, False)
        assert wire[q] == plan["total_wire"], q
        assert region[q] == off and region[q] % 256 == 0
        off += (wire[q] + 255) // 256 * 256
    assert total == (0 if bits == 32 else off)


def test_refusals_without_a_device():
    with pytest.raises(RuntimeError, match="world must be 1..256"):
        C.LocalEngineGroup(257, 1, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    g = C.LocalEngineGroup(4, 2, dict(p2p=False), 1, 1 << 16, TIMEOUT_MS)
    c = A.counts(4, "uneven", 50, seed=1)
    ins, outs = A.inputs(c, torch.float32, seed=0), A.outputs(c, torch.float32)
    with pytest.raises(RuntimeError, match="over several nodes needs device memory"):
        g.all_to_all(ins, outs, c, bits=4, bucket_size=64)
    bad = [row[:] for row in c]
    bad[0][1] += 1  # rank 0's input no longer matches its row
    with pytest.raises(RuntimeError, match="do not match its row and column"):
        g.all_to_all(ins, outs, bad, bits=4, bucket_size=64)
    with pytest.raises(RuntimeError, match="a multiple of local_size"):
        C.a2a_remote_wire([1, 2, 3], 0, 2, 4, 64)
    with pytest.raises(RuntimeError):
        C.a2a_remote_wire([1] * 257, 0, 1, 4, 64)
