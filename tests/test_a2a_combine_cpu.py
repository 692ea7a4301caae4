"""The weighted top-k combine without a GPU: the oracle's fma chain (k = 1, the order it pins, NaN,
Inf and -0), the composition reference on a small routed exchange, and every refusal of
``cgx.all_to_all_combine`` that fires before anything needs a device."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O

from _bitwise import assert_same

DTYPES = (torch.float32, torch.float16, torch.bfloat16)


@pytest.mark.parametrize("dtype", DTYPES)
def test_k1_is_one_rounded_product(dtype):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(64, 96, generator=g, dtype=torch.float64) * 3).to(dtype)
    gate = torch.rand(64, 1, generator=g)
    want = (gate * x.float()).to(dtype)  # one fp32 multiply, then one rounding to the dtype
    assert_same(O.combine_rows_reference(x, gate), want)


def test_chain_is_an_fma_per_choice_in_order():
    # c = 0: 1 * 1 = 1; c = 1: fma(2^-24, 1, 1) rounds to 1 (a tie to even); c = 2 the same: the
    # ascending chain stays 1. Reversed, the two small terms meet first, sum exactly to 2^-23 and
    # survive: 1 + 2^-23.
    x = torch.tensor([[1.0], [1.0], [1.0]])
    gate = torch.tensor([[1.0, 2.0 ** -24, 2.0 ** -24]])
    fwd = O.combine_rows_reference(x, gate)
    rev = O.combine_rows_reference(x.flip(0), gate.flip(1))
    assert fwd.item() == 1.0
    assert rev.item() == 1.0 + 2.0 ** -23


def test_fma_rounds_once():
    # g * g = 1 + 2^-11 + 2^-24 exactly; with acc = -1 an fma keeps the 2^-24, a multiply then an add
    # would round it away first
    g = 1.0 + 2.0 ** -12
    x = torch.tensor([[1.0], [g]])
    gate = torch.tensor([[-1.0, g]])
    got = O.combine_rows_reference(x, gate).item()
    assert got == 2.0 ** -11 + 2.0 ** -24
    assert got != float(np.float32(np.float32(g) * np.float32(g)) - np.float32(1.0))


def test_nan_inf_and_signed_zero():
    inf, nan = math.inf, math.nan
    # one token per case, k = 2
    x = torch.tensor([[nan], [1.0],        # NaN in a slot
                      [inf], [-inf],       # +Inf + -Inf
                      [inf], [1.0],        # Inf stays
                      [-0.0], [-0.0],      # -0 * 1 + -0 = -0
                      [0.0], [-0.0],       # +0 + -0 = +0
                      [1.0], [2.0],        # a NaN gate
                      [inf], [1.0]])       # 0 * Inf
    gate = torch.tensor([[1.0, 1.0], [1.0, 1.0], [2.0, 1.0], [1.0, 1.0], [1.0, 1.0], [nan, 1.0], [0.0, 1.0]])
    out = O.combine_rows_reference(x, gate).reshape(-1)
    assert math.isnan(out[0]) and math.isnan(out[1])
    assert out[2].item() == inf
    assert out[3].item() == 0.0 and math.copysign(1.0, out[3].item()) < 0
    assert out[4].item() == 0.0 and math.copysign(1.0, out[4].item()) > 0
    assert math.isnan(out[5]) and math.isnan(out[6])


def test_overflow_to_dtype_rounds_to_inf():
    x = torch.tensor([[60000.0], [60000.0]], dtype=torch.float16)
    out = O.combine_rows_reference(x, torch.ones(1, 2))
    assert out.item() == math.inf


@pytest.mark.parametrize("bits", (4, 32, "e4m3"))
def test_composition_reference(bits):
    # two ranks, T = 3 tokens of k = 2 on each: the combine reads the slots the routed reference wrote
    W, H, k, T = 2, 512, 2, 3
    g = torch.Generator().manual_seed(7)
    rows = [[2, 4], [4, 2]]  # rows[q][r], sum over q of rows[q][r] == T * k
    counts = [[v * H for v in r] for r in rows]
    xs = [torch.randn(sum(rows[q]) * H, generator=g) for q in range(W)]
    oi = [torch.randperm(T * k, generator=g) for _ in range(W)]
    gates = [torch.rand(T, k, generator=g) for _ in range(W)]
    slots, outs = O.routed_all_to_all_combine_reference(xs, counts, oi, gates, H, bits=bits, bucket_size=512)
    plain = O.routed_all_to_all_reference(xs, counts, [None] * W, oi, H, bits=bits, bucket_size=512,
                                          outputs=[torch.zeros(T * k * H)] * W)
    for r in range(W):
        assert_same(slots[r], plain[r])
        s = slots[r].reshape(T, k, H)
        want = torch.from_numpy(O._fma32_np(gates[r][:, 1, None].numpy(), s[:, 1].numpy(),
                                            (gates[r][:, 0, None] * s[:, 0]).numpy()))
        assert_same(outs[r].reshape(T, H), want)


# ---- refusals before anything runs (CPU tensors: the device check comes last) -----------------------
def _args(T=4, k=2, H=512, dtype=torch.bfloat16):
    x = torch.zeros(T * k, H, dtype=dtype)
    return dict(output=torch.empty(T, H, dtype=dtype), input=x, gate=torch.rand(T, k),
                output_index=torch.randperm(T * k))


@pytest.mark.parametrize("case,match", [
    ("gate_dtype", "gate must be a contiguous float32"),
    ("gate_shape", "gate must be a contiguous float32"),
    ("gate_layout", "gate must be a contiguous float32"),
    ("k33", "at most 32"),
    ("index_len", "T \\* k"),
    ("index_dtype", "int64"),
    ("output_shape", "output must be a contiguous tensor of shape"),
    ("codes_output", "codes output has no combine"),
    ("slots_shape", "slots must be"),
    ("output_overlaps", "the output overlaps the input"),
    ("slots_overlap", "slots overlaps the input"),
    ("gate_overlaps", "the gate overlaps the input"),
    ("device", "must be on the input's CUDA device"),
])
def test_refusals(case, match):
    a = _args()
    if case == "gate_dtype":
        a["gate"] = a["gate"].double()
    elif case == "gate_shape":
        a["gate"] = a["gate"].reshape(-1)
    elif case == "gate_layout":
        a["gate"] = torch.rand(2, 4).t()
    elif case == "k33":
        a = _args(T=1, k=33)
    elif case == "index_len":
        a["output_index"] = a["output_index"][:-1]
    elif case == "index_dtype":
        a["output_index"] = a["output_index"].int()
    elif case == "output_shape":
        a["output"] = torch.empty(5, 512, dtype=torch.bfloat16)
    elif case == "codes_output":
        a["output"] = torch.empty(4, 512, dtype=torch.float8_e4m3fn)
    elif case == "slots_shape":
        a["slots"] = torch.empty(4, 512, dtype=torch.bfloat16)
    elif case == "output_overlaps":
        a["output"] = a["input"][:4]
    elif case == "slots_overlap":
        a["slots"] = a["input"]
    elif case == "gate_overlaps":
        buf = torch.zeros(8 * 512 + 8)
        a["input"] = buf[:8 * 512].reshape(8, 512)
        a["output"] = torch.empty(4, 512)
        a["gate"] = buf[8 * 512 - 4:8 * 512 + 4].reshape(4, 2)
    with pytest.raises(ValueError, match=match):
        cgx.all_to_all_combine(**a)


def test_differentiable_refuses_before_sending():
    a = _args(k=33, T=1)
    with pytest.raises(ValueError, match="at most 32"):
        cgx.differentiable_all_to_all_combine(a["input"], a["gate"], a["output_index"])


def test_fp8_stochastic_refused():
    with pytest.raises(ValueError):
        cgx.all_to_all_combine(**_args(), bits="e4m3", stochastic=True)
