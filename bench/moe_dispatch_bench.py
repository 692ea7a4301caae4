#!/usr/bin/env python
"""MoE token dispatch and combine on W virtual ranks of one GPU (C.LocalSraGroup): the routed
all-to-all (rows gathered and scattered by index inside a2a_kernel) against the composition a
caller writes without it, index_select + plain all-to-all + index_copy_.

Every rank holds T tokens of H elements and routes each to top-k of E = 8 W experts (8 per rank),
seeded. The sent rows are sorted by destination rank: row i is token input_index[i]; the combine
returns them into T k slots (token * k + choice), slot output_index[j] for received row j.

  dispatch (a): send = x.index_select(0, input_index); all_to_all(recv, send)
  dispatch (b): all_to_all(recv, x, input_index)
  combine  (a): all_to_all(back, recv); out.index_copy_(0, output_index, back)
  combine  (b): all_to_all(out, recv, output_index)

With --codes, an FP8 expert GEMM's input instead (e4m3, routed dispatch, bucket 128 and bucket = H):

  dispatch (c): all_to_all(recv, x, input_index, bits="e4m3"), then the per-group FP8 quantize a
                caller writes in torch (amax, scale, cast) to get codes and scales for the GEMM
  dispatch (d): all_to_all(codes, x, input_index, bits="e4m3", output_scales=scales)

With --combine, the weighted top-k combine that follows (fp32 gates [T, k], seeded):

  combine (b)+sum: all_to_all(slots, recv, output_index), then the torch weighted sum of the README's
                   earlier recipe, (slots.view(T, k, H) * gate.unsqueeze(-1)).sum(1) (fp32 result)
  combine (e):     all_to_all(slots, recv, output_index, gate=gate, combine_out=out), the fused combine

Arm (e)'s output is checked bit for bit against the composition it is defined as: its slots equal
arm (b)'s, and rank 0's first 64 tokens equal the oracle's fma chain over those slots. Bytes: both
run arm (b)'s kernel; (e) then reads the T k slot rows back and writes T rows in the dtype; the
torch sum reads the slots, writes and reads an fp32 [T, k, H] product and writes T fp32 rows.

With --combine-backward, the backward of differentiable_all_to_all_combine (grad_out [T, H] in the
dtype, the forward's slots [T k, H] and fp32 gates [T, k], seeded):

  backward torch: grad_slots = (grad_out * gate) in the dtype, all_to_all(gin, grad_slots,
                  input_index=output_index), and the torch gate gradient (grad_out.float() *
                  slots.float()).sum(-1)
  backward fused: all_to_all(gin, grad_out, input_index=output_index // k,
                  input_scale=gate.view(-1)[output_index]) and combine_gate_grad(grad_out, slots, k)

The input gradients of the two arms are checked bit for bit, and rank 0's first 64 fused gate
gradients against the oracle. Bytes: both run the same exchange; the torch arm adds grad_slots
(read grad_out, write and read an fp32 [T, k, H] product, write the dtype) and its gate gradient
(fp32 copies of grad_out and the slots, the fp32 product written and read); the fused arm reads
grad_out and the slots once.

With --dispatch-backward, the backward of the dispatch (the gradient of the received rows [T k, H]
in the dtype, seeded), which returns every slot's gradient to its token's rank and sums each
token's k rows:

  backward index_add_: all_to_all(gin, grad), then zeros(T, H).index_add_(0, order // k, gin), the
                       backward of differentiable_all_to_all_single with input_index
  backward fused:      all_to_all(slots, grad, output_index=order, gate=ones(T, k), combine_out=out),
                       the unit-gate combine of differentiable_all_to_all_dispatch

Both arms exchange the same rows. Each row also reports whether every timed run of an arm gave the
bits of its first run (index_add_ adds with atomics in whatever order they land), the largest
absolute difference of each arm from the float64 sum of the same slots, and checks rank 0's first
64 fused tokens against the oracle. Bytes: the index_add_ arm adds the zero fill of [T, H], the read
of gin and a read-modify-write of a [T, H] row per slot (2 T k H es); the fused arm reads the slots
back, writes [T, H] and reads the T k fp32 unit gates.

Arms alternate in one run, CUDA events around each, medians over --iters after --warmup. The HBM
bytes of an arm are computed from shapes, all ranks together: the kernel reads the sent rows and
writes the received rows (2 N H es), writes and reads its wire image once (2 N H bits / 8, plus
8 bytes per 512-element bucket; raw at 32 bits, and own chunks are copied, not counted as wire);
arm (a) adds the permutation's read and write of N rows (2 N H es). Virtual ranks share one GPU's
HBM and exchange through it, so NVLink is not part of these numbers.
For (c) and (d) the wire is 1 byte per element plus 8 per bucket; (c) writes the received rows in
the dtype and its quantize reads them and writes 1 byte per element plus 4 per bucket, (d) writes
those codes and scales directly.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402

C = cgx._C


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def routing(W, T, k, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    E = 8 * W
    per_rank = []
    for _ in range(W):
        experts = torch.rand(T, E, generator=g, device=device).topk(k, dim=1).indices  # [T, k], distinct
        dest = (experts // 8).reshape(-1)
        order = torch.argsort(dest, stable=True)
        per_rank.append((order // k, order, torch.bincount(dest, minlength=W).tolist()))
    return per_rank


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def run_config(W, T, H, k, bits, iters, warmup, lanes, slot_mb, dtype=torch.bfloat16):
    dev = torch.device("cuda", 0)
    es = torch.tensor([], dtype=dtype).element_size()
    route = routing(W, T, k, seed=T * 31 + H * 7 + k, device=dev)
    send_rows = [route[q][2] for q in range(W)]
    recv_n = [sum(send_rows[q][r] for q in range(W)) for r in range(W)]
    disp_counts = [[send_rows[q][r] * H for r in range(W)] for q in range(W)]
    comb_counts = [[disp_counts[r][q] for r in range(W)] for q in range(W)]
    g = C.LocalSraGroup(W, lanes, slot_mb << 20, 20000, 256)
    xs = [torch.randn(T, H, device=dev, dtype=dtype) for _ in range(W)]
    send = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    recv = [torch.empty(recv_n[r], H, device=dev, dtype=dtype) for r in range(W)]
    back = send  # free once the dispatch has run: the combine's arm (a) reuses it
    out = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    ii = [route[q][0] for q in range(W)]
    oi = [route[q][1] for q in range(W)]
    flat = lambda ts: [t.reshape(-1) for t in ts]  # noqa: E731

    def disp_a():
        for q in range(W):
            torch.index_select(xs[q], 0, ii[q], out=send[q])
        g.all_to_all(flat(send), flat(recv), disp_counts, bits=bits, bucket_size=512)

    def disp_b():
        g.all_to_all(flat(xs), flat(recv), disp_counts, bits=bits, bucket_size=512, input_index=ii, row=H)

    def comb_a():
        g.all_to_all(flat(recv), flat(back), comb_counts, bits=bits, bucket_size=512)
        for q in range(W):
            out[q].index_copy_(0, oi[q], back[q])

    def comb_b():
        g.all_to_all(flat(recv), flat(out), comb_counts, bits=bits, bucket_size=512, output_index=oi, row=H)

    arms = {"dispatch_a": disp_a, "dispatch_b": disp_b, "combine_a": comb_a, "combine_b": comb_b}
    ts = {name: [] for name in arms}
    for it in range(warmup + iters):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ts[name].append(e0.elapsed_time(e1) * 1000.0)
    g.check()
    # the arms compute the same bytes
    ref_out = [o.clone() for o in out]
    comb_a()
    torch.cuda.synchronize()
    for q in range(W):
        assert torch.equal(ref_out[q], out[q]), "combine arms differ"

    N = T * k * W  # rows sent by all ranks
    own = sum(send_rows[q][q] for q in range(W))
    elems_wire = (N - own) * H
    wbits = 8 if isinstance(bits, str) else bits  # the FP8 formats move the bytes of bits 8
    wire = elems_wire * es if wbits >= 32 else elems_wire * wbits // 8 + (elems_wire // 512) * 8
    kernel_bytes = 2 * N * H * es + 2 * wire
    perm_bytes = 2 * N * H * es
    res = {"W": W, "T": T, "H": H, "topk": k, "bits": bits, "dtype": str(dtype).replace("torch.", "")}
    for name in arms:
        res[name + "_us"] = round(median(ts[name]), 1)
    res["bytes_b_GB"] = round(kernel_bytes / 1e9, 3)
    res["bytes_a_GB"] = round((kernel_bytes + perm_bytes) / 1e9, 3)
    del g, xs, send, recv, back, out
    torch.cuda.empty_cache()
    return res


def run_combine(W, T, H, k, bits, iters, warmup, lanes, slot_mb, dtype=torch.bfloat16):
    from torch_cgx_b200.ops import oracle as O

    dev = torch.device("cuda", 0)
    es = torch.tensor([], dtype=dtype).element_size()
    route = routing(W, T, k, seed=T * 31 + H * 7 + k, device=dev)
    send_rows = [route[q][2] for q in range(W)]
    recv_n = [sum(send_rows[q][r] for q in range(W)) for r in range(W)]
    comb_counts = [[send_rows[r][q] * H for r in range(W)] for q in range(W)]
    g = C.LocalSraGroup(W, lanes, slot_mb << 20, 20000, 256)
    gen = torch.Generator(device=dev).manual_seed(T + H + k)
    recv = [torch.randn(recv_n[r], H, device=dev, generator=gen).to(dtype) for r in range(W)]
    gate = [torch.rand(T, k, device=dev, generator=gen) for _ in range(W)]
    slots_b = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    slots_e = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    out_e = [torch.empty(T, H, device=dev, dtype=dtype) for _ in range(W)]
    out_b = [None] * W
    oi = [route[q][1] for q in range(W)]
    flat = lambda ts: [t.reshape(-1) for t in ts]  # noqa: E731

    def comb_b_sum():
        g.all_to_all(flat(recv), flat(slots_b), comb_counts, bits=bits, bucket_size=512, output_index=oi, row=H)
        for q in range(W):
            out_b[q] = (slots_b[q].view(T, k, H) * gate[q].unsqueeze(-1)).sum(1)

    def comb_e():
        g.all_to_all(flat(recv), flat(slots_e), comb_counts, bits=bits, bucket_size=512, output_index=oi, row=H,
                     gate=gate, combine_out=flat(out_e))

    arms = {"combine_b_sum": comb_b_sum, "combine_fused": comb_e}
    ts = {name: [] for name in arms}
    for it in range(warmup + iters):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ts[name].append(e0.elapsed_time(e1) * 1000.0)
    g.check()
    for q in range(W):
        assert torch.equal(slots_b[q], slots_e[q]), "the fused combine's slots differ from the routed call's"
    n = min(T, 64)
    want = O.combine_rows_reference(slots_b[0][:n * k].cpu(), gate[0][:n].cpu())
    assert torch.equal(want.view(torch.int16), out_e[0][:n].cpu().view(torch.int16)), "fused combine != composition"

    N = T * k * W
    own = sum(send_rows[q][q] for q in range(W))
    elems_wire = (N - own) * H
    wbits = 8 if isinstance(bits, str) else bits
    wire = elems_wire * es if wbits >= 32 else elems_wire * wbits // 8 + (elems_wire // 512) * 8
    kernel_bytes = 2 * N * H * es + 2 * wire
    fused_bytes = kernel_bytes + N * H * es + W * T * H * es
    torch_bytes = kernel_bytes + N * H * es + 2 * N * H * 4 + W * T * H * 4
    res = {"W": W, "T": T, "H": H, "topk": k, "bits": bits, "dtype": str(dtype).replace("torch.", "")}
    for name in arms:
        res[name + "_us"] = round(median(ts[name]), 1)
        res[name + "_spread_us"] = [round(min(ts[name]), 1), round(max(ts[name]), 1)]
    res["bytes_fused_GB"] = round(fused_bytes / 1e9, 3)
    res["bytes_b_sum_GB"] = round(torch_bytes / 1e9, 3)
    del g, recv, slots_b, slots_e, out_e, out_b
    torch.cuda.empty_cache()
    return res


def run_combine_backward(W, T, H, k, bits, iters, warmup, lanes, slot_mb, dtype=torch.bfloat16):
    from torch_cgx_b200.ops import oracle as O

    dev = torch.device("cuda", 0)
    es = torch.tensor([], dtype=dtype).element_size()
    route = routing(W, T, k, seed=T * 31 + H * 7 + k, device=dev)
    send_rows = [route[q][2] for q in range(W)]
    recv_n = [sum(send_rows[q][r] for q in range(W)) for r in range(W)]
    back_counts = [[send_rows[q][r] * H for r in range(W)] for q in range(W)]  # the combine's, swapped
    g = C.LocalSraGroup(W, lanes, slot_mb << 20, 20000, 256)
    gen = torch.Generator(device=dev).manual_seed(T + H + k)
    grad = [torch.randn(T, H, device=dev, generator=gen).to(dtype) for _ in range(W)]
    slots = [torch.randn(T * k, H, device=dev, generator=gen).to(dtype) for _ in range(W)]
    gate = [torch.rand(T, k, device=dev, generator=gen) for _ in range(W)]
    oi = [route[q][1] for q in range(W)]
    gin_t = [torch.empty(recv_n[r], H, device=dev, dtype=dtype) for r in range(W)]
    gin_f = [torch.empty(recv_n[r], H, device=dev, dtype=dtype) for r in range(W)]
    gg_t, gg_f = [None] * W, [None] * W
    flat = lambda ts: [t.reshape(-1) for t in ts]  # noqa: E731

    def bwd_torch():
        gs = [(grad[q].reshape(T, 1, H) * gate[q].unsqueeze(-1)).to(dtype).reshape(T * k, H) for q in range(W)]
        g.all_to_all(flat(gs), flat(gin_t), back_counts, bits=bits, bucket_size=512, input_index=oi, row=H)
        for q in range(W):
            gg_t[q] = (grad[q].reshape(T, 1, H).float() * slots[q].reshape(T, k, H).float()).sum(-1)

    def bwd_fused():
        ii = [torch.div(ix, k, rounding_mode="floor") for ix in oi]
        sc = [gate[q].reshape(-1)[oi[q]] for q in range(W)]
        g.all_to_all(flat(grad), flat(gin_f), back_counts, bits=bits, bucket_size=512, input_index=ii, row=H,
                     input_scale=sc)
        for q in range(W):
            gg_f[q] = C.combine_gate_grad(grad[q], slots[q], k)

    arms = {"backward_torch": bwd_torch, "backward_fused": bwd_fused}
    ts = {name: [] for name in arms}
    for it in range(warmup + iters):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ts[name].append(e0.elapsed_time(e1) * 1000.0)
    g.check()
    for r in range(W):
        assert torch.equal(gin_t[r].view(torch.int16), gin_f[r].view(torch.int16)), "input gradients differ"
    n = min(T, 64)
    want = O.combine_gate_grad_reference(grad[0][:n].cpu(), slots[0][:n * k].cpu())
    assert torch.equal(want, gg_f[0][:n].cpu()), "fused gate gradient != oracle"

    N = T * k * W
    own = sum(send_rows[q][q] for q in range(W))
    elems_wire = (N - own) * H
    wbits = 8 if isinstance(bits, str) else bits
    wire = elems_wire * es if wbits >= 32 else elems_wire * wbits // 8 + (elems_wire // 512) * 8
    kernel_bytes = 2 * N * H * es + 2 * wire
    TH, TkH = W * T * H, N * H
    torch_bytes = kernel_bytes + (TH * es + 8 * TkH + TkH * es) + (TH * (es + 8) + TkH * (es + 16))
    fused_bytes = kernel_bytes + TH * es + TkH * es
    res = {"W": W, "T": T, "H": H, "topk": k, "bits": bits, "dtype": str(dtype).replace("torch.", "")}
    for name in arms:
        res[name + "_us"] = round(median(ts[name]), 1)
        res[name + "_spread_us"] = [round(min(ts[name]), 1), round(max(ts[name]), 1)]
    res["bytes_fused_GB"] = round(fused_bytes / 1e9, 3)
    res["bytes_torch_GB"] = round(torch_bytes / 1e9, 3)
    del g, grad, slots, gin_t, gin_f
    torch.cuda.empty_cache()
    return res


def run_dispatch_backward(W, T, H, k, bits, iters, warmup, lanes, slot_mb, dtype=torch.bfloat16):
    from torch_cgx_b200.ops import oracle as O

    dev = torch.device("cuda", 0)
    es = torch.tensor([], dtype=dtype).element_size()
    route = routing(W, T, k, seed=T * 31 + H * 7 + k, device=dev)
    send_rows = [route[q][2] for q in range(W)]
    recv_n = [sum(send_rows[q][r] for q in range(W)) for r in range(W)]
    back_counts = [[send_rows[r][q] * H for r in range(W)] for q in range(W)]  # the dispatch's, swapped
    g = C.LocalSraGroup(W, lanes, slot_mb << 20, 20000, 256)
    gen = torch.Generator(device=dev).manual_seed(T + H + k)
    grad = [torch.randn(recv_n[r], H, device=dev, generator=gen).to(dtype) for r in range(W)]
    ii = [route[q][0] for q in range(W)]
    oi = [route[q][1] for q in range(W)]
    unit = [torch.ones(T, k, device=dev) for _ in range(W)]
    gin = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    slots = [torch.empty(T * k, H, device=dev, dtype=dtype) for _ in range(W)]
    out_a = [torch.empty(T, H, device=dev, dtype=dtype) for _ in range(W)]
    out_f = [torch.empty(T, H, device=dev, dtype=dtype) for _ in range(W)]
    flat = lambda ts: [t.reshape(-1) for t in ts]  # noqa: E731

    def bwd_index_add():
        g.all_to_all(flat(grad), flat(gin), back_counts, bits=bits, bucket_size=512)
        for q in range(W):
            out_a[q].zero_().index_add_(0, ii[q], gin[q])

    def bwd_fused():
        g.all_to_all(flat(grad), flat(slots), back_counts, bits=bits, bucket_size=512, output_index=oi, row=H,
                     gate=unit, combine_out=flat(out_f))

    arms = {"backward_index_add": (bwd_index_add, out_a), "backward_fused": (bwd_fused, out_f)}
    ts = {name: [] for name in arms}
    first = {}
    stable = {name: True for name in arms}
    for it in range(warmup + iters):
        for name, (fn, outs) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ts[name].append(e0.elapsed_time(e1) * 1000.0)
            if name not in first:
                first[name] = [o.clone() for o in outs]
            else:
                stable[name] &= all(torch.equal(a.view(torch.uint8), b.view(torch.uint8))
                                    for a, b in zip(first[name], outs))
    g.check()
    n = min(T, 64)
    want = O.dispatch_sum_reference(slots[0][:n * k].cpu(), k)
    assert torch.equal(want.view(torch.int16), out_f[0][:n].cpu().view(torch.int16)), "fused backward != oracle"
    err = {name: 0.0 for name in arms}
    for q in range(W):
        exact = slots[q].view(T, k, H).double().sum(1)
        for name, (_, outs) in arms.items():
            err[name] = max(err[name], float((outs[q].double() - exact).abs().max()))
        del exact

    N = T * k * W
    own = sum(send_rows[q][q] for q in range(W))
    elems_wire = (N - own) * H
    wbits = 8 if isinstance(bits, str) else bits
    wire = elems_wire * es if wbits >= 32 else elems_wire * wbits // 8 + (elems_wire // 512) * 8
    kernel_bytes = 2 * N * H * es + 2 * wire
    TH, TkH = W * T * H, N * H
    index_add_bytes = kernel_bytes + TH * es + TkH * es + 2 * TkH * es
    fused_bytes = kernel_bytes + TkH * es + TH * es + N * 4
    res = {"W": W, "T": T, "H": H, "topk": k, "bits": bits, "dtype": str(dtype).replace("torch.", "")}
    for name in arms:
        res[name + "_us"] = round(median(ts[name]), 1)
        res[name + "_spread_us"] = [round(min(ts[name]), 1), round(max(ts[name]), 1)]
        res[name + "_bitwise_stable"] = stable[name]
        res[name + "_max_abs_err_vs_f64"] = err[name]
    res["bytes_index_add_GB"] = round(index_add_bytes / 1e9, 3)
    res["bytes_fused_GB"] = round(fused_bytes / 1e9, 3)
    del g, grad, gin, slots, out_a, out_f, first
    torch.cuda.empty_cache()
    return res


def run_codes(W, T, H, k, bucket, iters, warmup, lanes, slot_mb, dtype=torch.bfloat16):
    """routed e4m3 dispatch: decode + torch quantize (c) against the codes output (d)"""
    dev = torch.device("cuda", 0)
    es = torch.tensor([], dtype=dtype).element_size()
    route = routing(W, T, k, seed=T * 31 + H * 7 + k, device=dev)
    send_rows = [route[q][2] for q in range(W)]
    recv_n = [sum(send_rows[q][r] for q in range(W)) for r in range(W)]
    counts = [[send_rows[q][r] * H for r in range(W)] for q in range(W)]
    g = C.LocalSraGroup(W, lanes, slot_mb << 20, 20000, 256)
    xs = [torch.randn(T, H, device=dev, dtype=dtype) for _ in range(W)]
    ii = [route[q][0] for q in range(W)]
    recv = [torch.empty(recv_n[r], H, device=dev, dtype=dtype) for r in range(W)]
    codes = [torch.empty(recv_n[r], H, device=dev, dtype=torch.float8_e4m3fn) for r in range(W)]
    scales = [torch.empty(recv_n[r], H // bucket, device=dev, dtype=torch.float32) for r in range(W)]
    tq = [None] * W
    flat = lambda ts: [t.reshape(-1) for t in ts]  # noqa: E731

    def disp_c():
        g.all_to_all(flat(xs), flat(recv), counts, bits="e4m3", bucket_size=bucket, input_index=ii, row=H)
        for r in range(W):
            v = recv[r].reshape(-1, bucket).float()
            unit = v.abs().amax(dim=1, keepdim=True) * (1.0 / 448.0)
            inv = torch.where(unit > 0, 1.0 / unit, torch.zeros_like(unit))
            tq[r] = ((v * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn), unit)

    def disp_d():
        g.all_to_all(flat(xs), flat(codes), counts, bits="e4m3", bucket_size=bucket, input_index=ii, row=H,
                     output_scales=flat(scales))

    arms = {"dispatch_c": disp_c, "dispatch_d": disp_d}
    ts = {name: [] for name in arms}
    for it in range(warmup + iters):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ts[name].append(e0.elapsed_time(e1) * 1000.0)
    g.check()
    # (d) decodes to what (c) received, before its rounding to the dtype
    for r in range(W):
        dec = (codes[r].float().reshape(-1, bucket) * scales[r].reshape(-1, 1)).reshape(recv[r].shape).to(dtype)
        own = sum(send_rows[q][r] for q in range(r))  # the own chunk: encoded by (d), copied by (c)
        mine = slice(own, own + send_rows[r][r])
        keep = torch.ones(recv_n[r], dtype=torch.bool, device=dev)
        keep[mine] = False
        assert torch.equal(dec[keep], recv[r][keep]), "codes arm differs from the decoded arm"

    N = T * k * W
    own = sum(send_rows[q][q] for q in range(W))
    elems_wire = (N - own) * H
    wire = elems_wire + (elems_wire // bucket) * 8
    codes_out = N * H + N * H // bucket * 4
    d_bytes = N * H * es + 2 * wire + codes_out
    c_bytes = N * H * es + 2 * wire + N * H * es + N * H * es + codes_out
    res = {"W": W, "T": T, "H": H, "topk": k, "bits": "e4m3", "bucket": bucket, "dtype": str(dtype).replace("torch.", "")}
    for name in arms:
        res[name + "_us"] = round(median(ts[name]), 1)
    res["bytes_c_GB"] = round(c_bytes / 1e9, 3)
    res["bytes_d_GB"] = round(d_bytes / 1e9, 3)
    del g, xs, recv, codes, scales, tq
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--hidden", type=int, nargs="+", default=[4096, 7168])
    ap.add_argument("--tokens", type=int, nargs="+", default=[4096, 16384])
    ap.add_argument("--topk", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--bits", type=lambda b: b if b in ("e4m3", "e5m2") else int(b), nargs="+", default=[4, 8, 32],
                    help="widths 1..8 or 32, or the FP8 wire formats e4m3 / e5m2")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    # 16 lanes x 8 ranks = 128 CTAs: the virtual ranks together occupy the GPU, as one real rank would its own
    ap.add_argument("--lanes", type=int, default=16)
    ap.add_argument("--slot-mb", type=int, default=4)
    ap.add_argument("--max-gb", type=float, default=60.0, help="skip configurations whose buffers exceed this")
    ap.add_argument("--out", type=str, default=None, help="also write the JSON lines here")
    ap.add_argument("--codes", action="store_true",
                    help="time the FP8 codes output, arms (c) and (d) at bucket 128 and bucket = H, instead")
    ap.add_argument("--combine", action="store_true",
                    help="time the weighted top-k combine, arm (e) against arm (b) and the torch sum, instead")
    ap.add_argument("--combine-backward", action="store_true",
                    help="time the combine's backward, the scaled send and the gate-gradient kernel against "
                         "grad_slots, the routed call and the torch gate gradient, instead")
    ap.add_argument("--dispatch-backward", action="store_true",
                    help="time the dispatch's backward, the unit-gate combine against the routed call and "
                         "index_add_, instead")
    args = ap.parse_args()
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    rows = []
    if args.dispatch_backward:
        for H in args.hidden:
            for T in args.tokens:
                for k in args.topk:
                    need = (args.world * (T * k * 3 * 2 + T * 4 * 2) + T * k * 8) * H / 1e9
                    if need > args.max_gb:
                        print(json.dumps({"H": H, "T": T, "topk": k, "skipped": f"needs {need:.1f} GB"}), flush=True)
                        continue
                    for bits in args.bits:
                        r = run_dispatch_backward(args.world, T, H, k, bits, args.iters, args.warmup, args.lanes,
                                                  args.slot_mb)
                        r.update(gpu=name, power_limit=power)
                        rows.append(r)
                        print(json.dumps(r), flush=True)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))
        return
    if args.combine_backward:
        for H in args.hidden:
            for T in args.tokens:
                for k in args.topk:
                    need = args.world * (T * k * (2 + 2 + 8) + T * 6) * H / 1e9
                    if need > args.max_gb:
                        print(json.dumps({"H": H, "T": T, "topk": k, "skipped": f"needs {need:.1f} GB"}), flush=True)
                        continue
                    for bits in args.bits:
                        r = run_combine_backward(args.world, T, H, k, bits, args.iters, args.warmup, args.lanes,
                                                 args.slot_mb)
                        r.update(gpu=name, power_limit=power)
                        rows.append(r)
                        print(json.dumps(r), flush=True)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))
        return
    if args.combine:
        for H in args.hidden:
            for T in args.tokens:
                for k in args.topk:
                    need = args.world * (2 * T * k * 2 + T * (2 + 4 * k)) * H / 1e9
                    if need > args.max_gb:
                        print(json.dumps({"H": H, "T": T, "topk": k, "skipped": f"needs {need:.1f} GB"}), flush=True)
                        continue
                    for bits in args.bits:
                        r = run_combine(args.world, T, H, k, bits, args.iters, args.warmup, args.lanes, args.slot_mb)
                        r.update(gpu=name, power_limit=power)
                        rows.append(r)
                        print(json.dumps(r), flush=True)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))
        return
    if args.codes:
        for H in args.hidden:
            for T in args.tokens:
                for k in args.topk:
                    need = args.world * (2 * T * k + T) * H * 2 / 1e9
                    if need > args.max_gb:
                        print(json.dumps({"H": H, "T": T, "topk": k, "skipped": f"needs {need:.1f} GB"}), flush=True)
                        continue
                    for bucket in (128, H):
                        r = run_codes(args.world, T, H, k, bucket, args.iters, args.warmup, args.lanes, args.slot_mb)
                        r.update(gpu=name, power_limit=power)
                        rows.append(r)
                        print(json.dumps(r), flush=True)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))
        return
    for H in args.hidden:
        for T in args.tokens:
            for k in args.topk:
                need = args.world * (3 * T * k + T) * H * 2 / 1e9
                if need > args.max_gb:
                    print(json.dumps({"H": H, "T": T, "topk": k, "skipped": f"needs {need:.1f} GB"}), flush=True)
                    continue
                for bits in args.bits:
                    r = run_config(args.world, T, H, k, bits, args.iters, args.warmup, args.lanes, args.slot_mb)
                    r.update(gpu=name, power_limit=power)
                    rows.append(r)
                    print(json.dumps(r), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
