"""The combine's backward without a GPU: the gate-gradient oracle's order (lanes, the xor butterfly,
short and ragged rows, k 1 and 32) against a plain loop over its definition, NaN / Inf / -0, its
closeness to a float64 sum, the scaled routed reference against the explicit composition, every
``input_scale`` / ``gate_grad`` refusal that fires before anything is sent, and the autograd wiring
at world 1."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import functional as F
from torch_cgx_b200.parallel import hooks

from _bitwise import assert_same

DTYPES = (torch.float32, torch.float16, torch.bfloat16)
F32 = np.float32


def _gate_grad_loop(go: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """the definition, one element at a time: per lane an fma chain in increasing h, then the butterfly"""
    T, H = go.shape
    k = x.shape[0] // T
    V = 16 // go.element_size()
    g, xs = go.float().numpy(), x.float().reshape(T, k, H).numpy()
    out = np.zeros((T, k), dtype=F32)
    for t in range(T):
        for c in range(k):
            lane = [F32(0.0)] * 32
            for h in range(H):
                l = (h // V) % 32
                lane[l] = F32(O._fma32_np(g[t, h], xs[t, c, h], lane[l]))
            with np.errstate(all="ignore"):
                for m in (16, 8, 4, 2, 1):
                    lane = [F32(lane[i] + lane[i ^ m]) for i in range(32)]
            assert all(v.tobytes() == lane[0].tobytes() or (np.isnan(v) and np.isnan(lane[0])) for v in lane)
            out[t, c] = lane[0]
    return torch.from_numpy(out)


def test_order_pins_lanes_and_butterfly():
    # bf16, V = 8: 2^24 in lane 0, 1 in lane 1, -2^24 in lane 2. In h order the 1 is absorbed by
    # 2^24 (a tie to even) and the sum is 0; the butterfly adds lanes 0 and 2 first (m = 2) and keeps it.
    go = torch.ones(1, 24, dtype=torch.bfloat16)
    x = torch.zeros(1, 24, dtype=torch.bfloat16)
    x[0, 0], x[0, 8], x[0, 16] = 2.0 ** 24, 1.0, -2.0 ** 24
    assert O.combine_gate_grad_reference(go, x).item() == 1.0
    assert float(sum(np.float32(v) for v in x.float().reshape(-1).numpy())) == 0.0


def test_fma_within_a_lane():
    # one lane (H < V): acc = fma(g, g, -1) keeps the 2^-24 a rounded product would lose
    g = 1.0 + 2.0 ** -12
    go = torch.tensor([[-1.0, g]])
    x = torch.tensor([[1.0, g]])
    assert O.combine_gate_grad_reference(go, x).item() == 2.0 ** -11 + 2.0 ** -24


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k,H", [(1, 7), (1, 300), (2, 13), (3, 255), (32, 21), (32, 1), (4, 1030)])
def test_oracle_matches_the_definition(dtype, k, H):
    g = torch.Generator().manual_seed(k * 1000 + H)
    T = 3
    go = torch.randn(T, H, generator=g).to(dtype)
    x = (torch.randn(T * k, H, generator=g) * 4).to(dtype)
    assert_same(O.combine_gate_grad_reference(go, x), _gate_grad_loop(go, x))


def test_cancellation_across_lanes_against_the_definition():
    # large values of both signs spread over many lanes and several rounds per lane
    g = torch.Generator().manual_seed(9)
    T, k, H = 2, 5, 8 * 32 * 3 + 5
    go = torch.randn(T, H, generator=g).to(torch.bfloat16)
    x = (torch.randn(T * k, H, generator=g) * torch.where(torch.rand(T * k, H, generator=g) < 0.1, 1e6, 1.0))
    x = x.to(torch.bfloat16)
    assert_same(O.combine_gate_grad_reference(go, x), _gate_grad_loop(go, x))


def test_nan_inf_and_signed_zero():
    inf, nan = math.inf, math.nan
    T, k, H = 5, 1, 40  # fp32: V = 4, so h = 0 is lane 0 and h = 4 is lane 1
    go = torch.ones(T, H)
    x = torch.zeros(T * k, H)
    x[0, 3] = nan                      # a NaN slot value
    x[1, 0], x[1, 4] = inf, -inf       # +Inf and -Inf meet in the butterfly: NaN
    x[2, 0] = inf                      # Inf stays
    go[3, 7] = 0.0
    x[3, 7] = inf                      # 0 * Inf: NaN
    x[4] = -0.0                        # -0 products from +0: +0
    out = O.combine_gate_grad_reference(go, x).reshape(-1)
    assert math.isnan(out[0]) and math.isnan(out[1]) and math.isnan(out[3])
    assert out[2].item() == inf
    assert out[4].item() == 0.0 and math.copysign(1.0, out[4].item()) > 0
    assert_same(out.reshape(T, k), _gate_grad_loop(go, x))


def test_close_to_float64():
    g = torch.Generator().manual_seed(4)
    T, k, H = 6, 8, 7168
    go = torch.randn(T, H, generator=g).to(torch.bfloat16)
    x = torch.randn(T * k, H, generator=g).to(torch.bfloat16)
    got = O.combine_gate_grad_reference(go, x).double()
    prod = go.double().unsqueeze(1) * x.double().reshape(T, k, H)
    want, scale = prod.sum(-1), prod.abs().sum(-1)
    assert ((got - want).abs() <= 1e-6 * scale).all()


# ---- the scaled routed reference ---------------------------------------------------------------------
@pytest.mark.parametrize("bits", (4, 32, "e4m3"))
@pytest.mark.parametrize("dtype", DTYPES)
def test_scaled_reference_is_the_composition(bits, dtype):
    W, H = 2, 512
    g = torch.Generator().manual_seed(3)
    rows = [[3, 2], [1, 4]]  # rows[q][r]
    counts = [[v * H for v in r] for r in rows]
    xs = [torch.randn(5, H, generator=g).to(dtype) for _ in range(W)]
    ii = [torch.randint(0, 5, (sum(rows[q]),), generator=g) for q in range(W)]  # repeats allowed
    sc = [torch.randn(sum(rows[q]), generator=g) * 3 for q in range(W)]
    sc[0][0], sc[0][1], sc[1][0] = -0.0, float("inf"), 1e30  # -0, Inf, and products beyond fp16's range
    oi = [torch.randperm(sum(rows[q][r] for q in range(W)) + 2, generator=g)[:sum(rows[q][r] for q in range(W))]
          for r in range(W)]
    outs = [torch.zeros((len(oi[r]) + 2) * H, dtype=dtype) for r in range(W)]
    got = O.routed_all_to_all_reference(xs, counts, ii, oi, H, bits=bits, bucket_size=512, outputs=outs,
                                        input_scale=sc)
    sent = [(xs[q].index_select(0, ii[q]).float() * sc[q][:, None]).to(dtype) for q in range(W)]
    want = O.routed_all_to_all_reference(sent, counts, [None] * W, oi, H, bits=bits, bucket_size=512, outputs=outs)
    for r in range(W):
        assert_same(got[r], want[r], f"rank {r}")
    assert O.routed_all_to_all_reference(xs, counts, ii, oi, H, bits=bits, bucket_size=512, outputs=outs,
                                         input_scale=[None, None])[0].equal(
        O.routed_all_to_all_reference(xs, counts, ii, oi, H, bits=bits, bucket_size=512, outputs=outs)[0])


# ---- refusals before anything is sent ----------------------------------------------------------------
@pytest.fixture
def no_send(monkeypatch):
    """a process group lookup that records it was reached (nothing may be sent before a refusal)"""
    reached = []
    monkeypatch.setattr(hooks, "_native_backend", lambda *a, **k: reached.append(1))
    yield reached
    assert not reached


def _scale_args():
    x = torch.zeros(6, 512, dtype=torch.bfloat16)
    return dict(output=torch.zeros(4, 512, dtype=torch.bfloat16), input=x,
                input_index=torch.tensor([0, 2, 2, 5]), input_scale=torch.ones(4))


@pytest.mark.parametrize("case,match", [
    ("no_index", "needs an input_index"),
    ("dtype", "contiguous float32 vector"),
    ("shape", "contiguous float32 vector"),
    ("layout", "contiguous float32 vector"),
    ("length", "contiguous float32 vector"),
    ("codes", "no codes output"),
    ("overlap", "overlaps the output"),
    ("device", "CUDA device"),
])
def test_input_scale_refusals(no_send, case, match):
    a = _scale_args()
    if case == "no_index":
        del a["input_index"]
    elif case == "dtype":
        a["input_scale"] = a["input_scale"].double()
    elif case == "shape":
        a["input_scale"] = a["input_scale"].reshape(2, 2)
    elif case == "layout":
        a["input_scale"] = torch.ones(4, 2)[:, 0]
    elif case == "length":
        a["input_scale"] = torch.ones(5)
    elif case == "codes":
        a["output"] = torch.empty(4, 512, dtype=torch.float8_e4m3fn)
        a.update(bits="e4m3", output_scales=torch.empty(4, 1))
    elif case == "overlap":
        a["output"] = torch.zeros(4, 512)
        a["input"] = torch.zeros(6, 512)
        a["input_scale"] = a["output"].reshape(-1)[:4]
    with pytest.raises(ValueError, match=match):
        cgx.all_to_all_single(**a)


def test_gate_grad_keyword_refused_before_sending(monkeypatch):
    sent = []
    monkeypatch.setattr(F, "all_to_all_combine", lambda *a, **k: sent.append(k))
    x = torch.zeros(4, 8, requires_grad=True)
    with pytest.raises(ValueError, match="gate_grad"):
        cgx.differentiable_all_to_all_combine(x, torch.rand(2, 2), torch.arange(4), gate_grad="cuda")
    assert not sent


# ---- the autograd wiring at world 1 ------------------------------------------------------------------
class _Done:
    def wait(self):
        return None


def _world1_all_to_all(output, input, output_split_sizes=None, input_split_sizes=None, bits=8, bucket_size=512,
                       group=None, async_op=False, stochastic=False, seed=None, input_index=None,
                       output_index=None, output_scales=None, input_scale=None):
    """the composition at world 1, where the exchange is the own chunk's copy"""
    send = input if input_index is None else input.index_select(0, input_index)
    if input_scale is not None:
        send = (send.float() * input_scale.reshape((-1,) + (1,) * (send.dim() - 1))).to(input.dtype)
    if output_index is None:
        output.copy_(send)
    else:
        output.index_copy_(0, output_index, send)
    return _Done() if async_op else None


def _world1_combine(output, input, gate, output_index, output_split_sizes=None, input_split_sizes=None, bits=8,
                    bucket_size=512, group=None, async_op=False, stochastic=False, seed=None, slots=None):
    slots.index_copy_(0, output_index, input)
    output.copy_(O.combine_rows_reference(slots.reshape(slots.shape[0], -1), gate).reshape(output.shape))


@pytest.mark.parametrize("gate_grad", ("torch", "fused"))
@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16))
def test_backward_wiring_world1(monkeypatch, gate_grad, dtype):
    calls = []

    def a2a(*a, **kw):
        calls.append(kw)
        return _world1_all_to_all(*a, **kw)

    monkeypatch.setattr(F, "all_to_all_single", a2a)
    monkeypatch.setattr(F, "all_to_all_combine", _world1_combine)
    monkeypatch.setattr(cgx._C, "combine_gate_grad", lambda go, x, k: O.combine_gate_grad_reference(go, x),
                        raising=False)
    g = torch.Generator().manual_seed(5)
    T, k, H = 7, 3, 40
    x = torch.randn(T * k, H, generator=g).to(dtype).requires_grad_()
    gate = torch.rand(T, k, generator=g).requires_grad_()
    oi = torch.randperm(T * k, generator=g)
    y = cgx.differentiable_all_to_all_combine(x, gate, oi, [T * k], [T * k], bits=4, grad_bits=8,
                                              gate_grad=gate_grad)
    w = torch.randn(T, H, generator=g).to(dtype)
    y.backward(w)
    assert len(calls) == 1 and calls[0]["bits"] == 8 and calls[0]["async_op"]
    assert calls[0]["input_index"].equal(oi // k)
    # the input gradient: today's grad_slots, gathered by output_index
    grad_slots = (w.reshape(T, 1, H) * gate.detach().unsqueeze(-1)).to(dtype).reshape(T * k, H)
    assert_same(x.grad, grad_slots.index_select(0, oi), "input gradient")
    slots = torch.zeros(T * k, H, dtype=dtype).index_copy_(0, oi, x.detach())
    if gate_grad == "torch":
        want = (w.reshape(T, 1, H).float() * slots.reshape(T, k, H).float()).sum(-1)
    else:
        want = O.combine_gate_grad_reference(w, slots)
    assert_same(gate.grad, want, "gate gradient")
