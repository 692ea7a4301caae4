"""The backward of the MoE dispatch without a GPU: the oracle's fp32 sum in choice order against the
unit-gate combine reference (every width, dtype, world and k, and the edge inputs), the arithmetic
it pins (one rounding, -0, NaN, Inf), a reversed-order perturbation that the comparison catches, and
every refusal of ``cgx.differentiable_all_to_all_dispatch`` that fires before anything needs a device."""
from __future__ import annotations

import math

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same, mismatch
from _edge_inputs import edge_inputs

DTYPES = (torch.float32, torch.float16, torch.bfloat16)
BITS = (2, 4, 8, 32, "e4m3", "e5m2", "e4m3_pow2", "e5m2_sr")
SEED, SEQ = 0x5EED, 3


def routed_case(W, T, k, H, dtype, seed, xs=None):
    """(grads, counts, slot_index): rank q returns rows[q][r] slot rows to rank r, whose T * k slots
    are a random permutation"""
    g = torch.Generator().manual_seed(seed)
    rows = [[0] * W for _ in range(W)]
    for r in range(W):
        src = torch.randint(0, W, (T * k,), generator=g)
        for q in range(W):
            rows[q][r] = int((src == q).sum())
    counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
    if xs is None:
        xs = [(torch.randn(sum(rows[q]), H, generator=g, dtype=torch.float64) * (q + 1)).to(dtype).reshape(-1)
              for q in range(W)]
    si = [torch.randperm(T * k, generator=g) for _ in range(W)]
    return xs, counts, si


def unit_gates(si, k):
    return [torch.ones(ix.numel() // k, k) for ix in si]


@pytest.mark.parametrize("k", (1, 2, 8, 32))
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_oracle_is_the_unit_gate_combine(dtype, bits, k):
    H, B = 64, 32
    for W in range(1, 9):
        T = 2 if k == 32 else 5
        xs, counts, si = routed_case(W, T, k, H, dtype, seed=W * 100 + k)
        slots, outs = O.dispatch_backward_reference(xs, counts, si, k, H, bits=bits, bucket_size=B, seed=SEED,
                                                    seq=SEQ)
        cs, co = O.routed_all_to_all_combine_reference(xs, counts, si, unit_gates(si, k), H, bits=bits,
                                                       bucket_size=B, seed=SEED, seq=SEQ)
        for r in range(W):
            assert_same(slots[r], cs[r], f"W={W} slots rank {r}")
            assert_same(outs[r], co[r], f"W={W} rank {r}")


@pytest.mark.parametrize("bits", (4, 32, "e5m2"))
@pytest.mark.parametrize("dtype", DTYPES)
def test_oracle_edge_inputs(dtype, bits):
    W, T, k, H, B = 4, 8, 4, 512, 64
    _, counts, _ = routed_case(W, T, k, H, dtype, seed=3)
    sizes = [sum(counts[q]) for q in range(W)]
    ins, _ = edge_inputs(dtype, max(sizes), B, seed=4, world=W, bits=4)
    xs, counts, si = routed_case(W, T, k, H, dtype, seed=3, xs=[ins[q][:sizes[q]] for q in range(W)])
    _, outs = O.dispatch_backward_reference(xs, counts, si, k, H, bits=bits, bucket_size=B)
    _, co = O.routed_all_to_all_combine_reference(xs, counts, si, unit_gates(si, k), H, bits=bits, bucket_size=B)
    for r in range(W):
        assert_same(outs[r], co[r], f"edge rank {r}")


def test_oracle_input_index_gathers_first():
    W, T, k, H = 3, 4, 2, 64
    xs, counts, si = routed_case(W, T, k, H, torch.bfloat16, seed=9)
    g = torch.Generator().manual_seed(10)
    rows = [x.numel() // H for x in xs]
    big = [torch.randn(n + 3, H, generator=g).to(torch.bfloat16) for n in rows]
    ii = [torch.randperm(n + 3, generator=g)[:n] for n in rows]
    got = O.dispatch_backward_reference([b.reshape(-1) for b in big], counts, si, k, H, bits=4, bucket_size=32,
                                        input_index=ii)
    want = O.dispatch_backward_reference([b[i].reshape(-1) for b, i in zip(big, ii)], counts, si, k, H, bits=4,
                                         bucket_size=32)
    for r in range(W):
        assert_same(got[1][r], want[1][r], f"rank {r}")


def test_sum_rounds_once_in_fp32():
    # bf16 1 + 2^-8 + 2^-8: fp32 keeps 1 + 2^-7, which bf16 holds; rounding after every add (index_add_
    # in bf16) loses each 2^-8 to a tie to even and gives 1
    x = torch.tensor([[1.0], [2.0 ** -8], [2.0 ** -8]], dtype=torch.bfloat16)
    assert O.dispatch_sum_reference(x, 3).item() == 1.0 + 2.0 ** -7
    acc = torch.zeros(1, 1, dtype=torch.bfloat16)
    for c in range(3):
        acc += x[c]
    assert acc.item() == 1.0


def test_nan_inf_and_signed_zero():
    inf, nan = math.inf, math.nan
    x = torch.tensor([[-0.0], [-0.0],   # -0 + -0 = -0 (index_add_ from +0 gives +0)
                      [0.0], [-0.0],    # +0 + -0 = +0
                      [inf], [-inf],    # NaN
                      [nan], [1.0],     # NaN
                      [inf], [1.0]])    # Inf
    out = O.dispatch_sum_reference(x, 2).reshape(-1)
    assert out[0].item() == 0.0 and math.copysign(1.0, out[0].item()) < 0
    assert out[1].item() == 0.0 and math.copysign(1.0, out[1].item()) > 0
    assert math.isnan(out[2]) and math.isnan(out[3])
    assert out[4].item() == inf
    via_index_add = torch.zeros(5, 1).index_add_(0, torch.arange(10) // 2, x)
    assert math.copysign(1.0, via_index_add[0].item()) > 0


def _reversed_sum(slots, k):
    T = slots.shape[0] // k
    return O.dispatch_sum_reference(slots.reshape(T, k, -1).flip(1).reshape(slots.shape), k)


def test_reverse_order_is_caught():
    # choice order 1, 2^-24, 2^-24: each small term is lost to a tie to even and the sum stays 1;
    # reversed, the small terms meet first, sum to 2^-23 exactly and survive
    x = torch.tensor([[1.0], [2.0 ** -24], [2.0 ** -24]])
    want = O.combine_rows_reference(x, torch.ones(1, 3))
    assert_same(O.dispatch_sum_reference(x, 3), want)
    assert want.item() == 1.0
    assert mismatch(_reversed_sum(x, 3), want), "a reversed sum must differ on the named case"


# ---- refusals before anything is sent (CPU tensors: the device check comes last) -------------------
def _tokens(T=4, H=16):
    return torch.zeros(T, H, dtype=torch.bfloat16)


@pytest.mark.parametrize("case,match", [
    ("dtype", "contiguous int64 vector"),
    ("shape", "contiguous int64 vector"),
    ("layout", "contiguous int64 vector"),
    ("length", "T \\* k entries"),
    ("k33", "T \\* k entries"),
    ("empty", "T \\* k entries"),
    ("device", "CUDA device"),
    ("output_rows", "output_index needs output_rows"),
    ("fp8_stochastic", "rounds to nearest only"),
    ("fp8_grad_stochastic", "rounds to nearest only"),
])
def test_refusals(case, match):
    x, si, kw = _tokens(), torch.randperm(8), {}
    if case == "dtype":
        si = si.int()
    elif case == "shape":
        si = si.reshape(4, 2)
    elif case == "layout":
        si = torch.randperm(16)[::2]
    elif case == "length":
        si = torch.randperm(7)
    elif case == "k33":
        x, si = _tokens(T=1), torch.randperm(33)
    elif case == "empty":
        si = torch.empty(0, dtype=torch.int64)
    elif case == "output_rows":
        kw["output_index"] = torch.arange(8)
    elif case == "fp8_stochastic":
        kw.update(bits="e4m3", stochastic=True)
    elif case == "fp8_grad_stochastic":
        kw.update(bits=4, grad_bits="e5m2", stochastic=True)
    with pytest.raises(ValueError, match=match):
        cgx.differentiable_all_to_all_dispatch(x, si, **kw)


def test_combine_input_index_refused():
    x = torch.zeros(8, 16)
    with pytest.raises(ValueError, match="input_index must be a contiguous int64"):
        cgx.all_to_all_combine(torch.empty(4, 16), x, torch.ones(4, 2), torch.randperm(8),
                               input_index=torch.arange(8).int())


def test_exported():
    from torch_cgx_b200 import parallel

    assert cgx.differentiable_all_to_all_dispatch is parallel.differentiable_all_to_all_dispatch
    assert "differentiable_all_to_all_dispatch" in cgx.__all__
