"""The routed all-to-all without a GPU: the row predicate a2a_rows_fit against a brute force over
the items a2a_block_item produces, the reference composition (index_select, all-to-all,
index_copy_) with its autograd, and the autograd wiring of differentiable_all_to_all_single."""
import math

import pytest
import torch

import torch_cgx_b200 as cgx
from torch_cgx_b200.ops import oracle as O
from torch_cgx_b200.parallel import functional as F

from _bitwise import assert_same

C = cgx._C
ROWS = (1, 7, 8, 100, 256, 512, 640, 1024, 1536, 4096, 7168)
FIT_BITS = (1, 2, 3, 4, 5, 6, 7, 8, 32)
FIT_BUCKETS = (1, 8, 64, 100, 512, 1024, 3000, 8192)
MAX_BLOCK = 8192


def _crossing(n, H, bits, bucket, dtype):
    """whether some item of an n-element chunk spans two rows of H elements"""
    items = C.a2a_items(n, bits, bucket, dtype)
    off, cnt = items[:, 0], items[:, 6]
    return bool(((off // H) != ((off + cnt - 1) // H)).any())


@pytest.mark.parametrize("H", ROWS)
def test_rows_fit_matches_brute_force(H):
    # the items repeat with the block and the rows with H: lcm(H, block) plus two blocks of rows
    # shows every item a chunk of whole rows can produce; short chunks add the partial last blocks
    big = -(-(math.lcm(H, MAX_BLOCK) + 2 * MAX_BLOCK) // H)
    for dtype in (0, 1, 2):
        for bits in FIT_BITS:
            for bucket in FIT_BUCKETS:
                fit = C.a2a_rows_fit(H, bits, bucket, dtype)
                what = f"H={H} bits={bits} bucket={bucket} dtype={dtype}"
                if fit:
                    for R in (1, 2, 3, 17, big):
                        assert not _crossing(R * H, H, bits, bucket, dtype), what
                else:
                    assert _crossing(big * H, H, bits, bucket, dtype), what


def test_typical_moe_widths_fit():
    for H in (1024, 2048, 4096, 7168, 8192):
        for bits in FIT_BITS:
            for bucket in (512, 1024):
                assert C.a2a_rows_fit(H, bits, bucket, 2), (H, bits, bucket)
    assert not C.a2a_rows_fit(100, 4, 1024, 2) and not C.a2a_rows_fit(640, 4, 1024, 2)
    assert not C.a2a_rows_fit(0, 4, 512, 2)


# ---- the reference composition and its autograd --------------------------------------------------
class _RefA2A(torch.autograd.Function):
    """all_to_all_reference over W ranks' flat tensors; the backward sends the gradient back exactly."""

    @staticmethod
    def forward(ctx, counts, bits, *xs):
        ctx.counts = counts
        return tuple(O.all_to_all_reference(list(xs), counts, bits=bits, bucket_size=512))

    @staticmethod
    def backward(ctx, *grads):
        W = len(grads)
        back = [[ctx.counts[q][r] for q in range(W)] for r in range(W)]
        gs = O.all_to_all_reference([g.contiguous() for g in grads], back, bits=32, bucket_size=512)
        return (None, None, *gs)


def _routing(W, T, k, H, seed):
    """top-k routing of T tokens on each of W ranks: the send index (token of each sent row, sorted
    by destination rank), the row counts and the combine index (slot token * k + choice)"""
    g = torch.Generator().manual_seed(seed)
    send_ix, comb_ix, rows = [], [], []
    for _ in range(W):
        dest = torch.stack([torch.randperm(W, generator=g)[:k] for _ in range(T)])  # [T, k], distinct ranks
        order = torch.argsort(dest.reshape(-1), stable=True)
        send_ix.append(order // k)
        comb_ix.append(order)
        rows.append([int((dest == q).sum()) for q in range(W)])
    return send_ix, comb_ix, rows


def test_reference_composition_shapes_zero_rows_and_duplicate_gradients():
    W, T, k, H = 3, 10, 2, 8
    send_ix, comb_ix, rows = _routing(W, T, k, H, seed=0)
    counts = [[rows[q][r] * H for r in range(W)] for q in range(W)]
    g = torch.Generator().manual_seed(1)
    xs = [torch.randn(T, H, generator=g, requires_grad=True) for _ in range(W)]
    # dispatch with the routed reference, then its composition under autograd
    recv_rows = [sum(rows[q][r] for q in range(W)) for r in range(W)]
    disp = O.routed_all_to_all_reference(xs, counts, send_ix, [None] * W, H, bits=4, bucket_size=512)
    sent = [x.index_select(0, ix).reshape(-1) for x, ix in zip(xs, send_ix)]
    got = _RefA2A.apply(counts, 4, *sent)
    for r in range(W):
        assert disp[r].shape == (recv_rows[r] * H,)
        assert_same(got[r].detach(), disp[r], f"dispatch rank {r}")
    # combine back into [T * k + 2] slots: the two extra rows nobody names stay zero
    back = [[counts[r][q] for r in range(W)] for q in range(W)]
    outs0 = [torch.zeros(T * k + 2, H) for _ in range(W)]
    ys = [d.reshape(-1, H) * 2 for d in got]
    comb = O.routed_all_to_all_reference([y.detach() for y in ys], back, [None] * W, comb_ix, H, bits=8,
                                         bucket_size=512, outputs=outs0)
    flat = _RefA2A.apply(back, 8, *[y.reshape(-1) for y in ys])
    outs = [torch.zeros(T * k + 2, H).index_copy(0, ix, f.reshape(-1, H)) for ix, f in zip(comb_ix, flat)]
    for r in range(W):
        assert comb[r].shape == ((T * k + 2) * H,)
        assert_same(outs[r].detach().reshape(-1), comb[r], f"combine rank {r}")
        assert (outs[r][T * k:] == 0).all()
    # every token went to k ranks and came back into k slots: its gradient sums k copies
    wts = [torch.randn(T * k + 2, H, generator=g) for _ in range(W)]
    torch.stack([(o * w).sum() for o, w in zip(outs, wts)]).sum().backward()
    for r in range(W):
        want = torch.zeros(T, H)
        for s in range(T * k):
            want[s // k] += 2 * wts[r][s]
        torch.testing.assert_close(xs[r].grad, want, rtol=0, atol=1e-5)


# ---- differentiable_all_to_all_single's routing, at world 1 on the CPU -----------------------------
def _world1_all_to_all(output, input, output_split_sizes=None, input_split_sizes=None, bits=8, bucket_size=512,
                       group=None, async_op=False, stochastic=False, seed=None, input_index=None,
                       output_index=None):
    """the composition at world 1, where the exchange is the own chunk's copy"""
    send = input if input_index is None else input.index_select(0, input_index)
    if output_index is None:
        output.copy_(send)
    else:
        output.index_copy_(0, output_index, send)


@pytest.mark.parametrize("which", ["input", "output", "both"])
def test_differentiable_routing_matches_autograd_world1(monkeypatch, which):
    monkeypatch.setattr(F, "all_to_all_single", _world1_all_to_all)
    g = torch.Generator().manual_seed(3)
    T, H, k = 12, 8, 3
    ii = torch.randint(0, T, (T * k,), generator=g) if which != "output" else None  # repeats on purpose
    n = T * k if ii is not None else T
    oi = torch.randperm(n + 5, generator=g)[:n] if which != "input" else None
    x = torch.randn(T, H, generator=g, requires_grad=True)
    y = F.differentiable_all_to_all_single(x, [n], [n], bits=8, input_index=ii, output_index=oi,
                                           output_rows=None if oi is None else n + 5)
    w = torch.randn(y.shape, generator=g)
    (y * w).sum().backward()
    x2 = x.detach().clone().requires_grad_()
    send = x2 if ii is None else x2.index_select(0, ii)
    y2 = send if oi is None else torch.zeros(n + 5, H).index_copy(0, oi, send)
    (y2 * w).sum().backward()
    with torch.no_grad():
        assert_same(y, y2, "forward")
    assert_same(x.grad, x2.grad, "backward")
    if oi is not None:
        named = torch.zeros(n + 5, dtype=torch.bool)
        named[oi] = True
        assert (y.detach()[~named] == 0).all()


def test_differentiable_output_index_needs_rows():
    with pytest.raises(ValueError, match="output_rows"):
        F.differentiable_all_to_all_single(torch.zeros(2, 2), output_index=torch.arange(2))
