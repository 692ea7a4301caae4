#!/usr/bin/env python
"""Device time of the channels_last BatchNorm (+ ReLU), native kernels against the eager ATen ops they
replace, at every distinct BatchNorm shape of ResNet-50 (bf16, channels_last, batch 128 / 224 px).

    python bench/batchnorm_bench.py [--batch 128] [--iters 20]
    python bench/batchnorm_bench.py --profile-step [--batch 128] [--steps 3]

Per shape and ReLU on/off (ReLU shapes only where ResNet-50 fuses one):
  forward   native: C.batchnorm_cl_forward                          3 passes (stats read; transform r+w)
            eager:  aten.native_batch_norm (+ relu_)                3 (+ 2) passes
  backward  native: C.batchnorm_cl_backward                         5 passes (reduce 2 reads; elemt 2 reads + write)
            eager:  (threshold_backward +) native_batch_norm_backward  5 (+ 3) passes
CUDA events around `iters` back-to-back calls over rotating operand sets (more than 2x L2 in total),
median of 3. A torch.profiler pass over the same calls splits each op into its kernels; every kernel's
TB/s is its passes' bytes over its time, with the fraction of the 3.35 TB/s data-sheet bandwidth
(H100 SXM at 700 W; the card's power limit is reported alongside).

--profile-step runs one torch.profiler trace of ResNet-50 SGD steps (bf16 autocast, channels_last,
no DDP) and sums kernel time per step by group: BN statistics, transform, backward reduction,
backward element-wise, ReLU, residual join, other. Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

HBM_TBS = 3.35
# (shape without batch, followed by a fused ReLU in ResNet-50)
SHAPES = [((64, 112, 112), True), ((64, 56, 56), True), ((256, 56, 56), False), ((128, 56, 56), True),
          ((128, 28, 28), True), ((512, 28, 28), False), ((256, 28, 28), True), ((256, 14, 14), True),
          ((1024, 14, 14), False), ((512, 14, 14), True), ((512, 7, 7), True), ((2048, 7, 7), False)]
# kernel-name fragment -> (group, passes over the activation)
GROUPS = [("bn_stats_kernel", "bn_stats", 1), ("collect_statistics", "bn_stats", 1),
          ("bn_transform_kernel", "bn_transform", 2), ("transform_input", "bn_transform", 2),
          ("bn_bwd_reduce_kernel", "bn_bwd_reduce", 2), ("backward_reduce", "bn_bwd_reduce", 2),
          ("bn_bwd_elemt_kernel", "bn_bwd_elemt", 3), ("backward_elemt", "bn_bwd_elemt", 3),
          ("update_stats_and_invert", "bn_stats", 0),
          ("clamp_min", "relu", 2), ("threshold", "relu", 3), ("residual_relu", "join", 0)]


def group_of(name: str):
    for frag, g, passes in GROUPS:
        if frag in name:
            return g, passes
    return "other", 0


def kernel_times(prof):
    """(name, µs) of every device kernel in a torch.profiler run"""
    import torch

    out = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out.append((e.name, e.time_range.elapsed_us()))
    return out


def card():
    import subprocess

    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def bench_kernels(args):
    import torch
    from torch.profiler import ProfilerActivity, profile

    import torch_cgx_b200 as cgx

    C = cgx._C
    dev = torch.device("cuda", 0)
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size

    def timeit(fn, sets):
        for s in sets[:2]:
            fn(*s)
        reps = []
        for _ in range(3):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.iters):
                fn(*sets[i % len(sets)])
            e1.record()
            torch.cuda.synchronize()
            reps.append(e0.elapsed_time(e1) * 1e3 / args.iters)
        return sorted(reps)[1]

    def per_kernel(fn, sets, nbytes):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.iters):
                fn(*sets[i % len(sets)])
            torch.cuda.synchronize()
        acc = {}
        for name, us in kernel_times(prof):
            g, passes = group_of(name)
            t, p = acc.get(g, (0.0, 0))
            acc[g] = (t + us / args.iters, max(p, passes))  # ATen's stats group has a 0-pass update kernel
        return {g: {"us": round(t, 1), **({"tbs": round(p * nbytes / t / 1e6, 2),
                                          "of_peak": round(p * nbytes / t / 1e6 / HBM_TBS, 2)} if p and t else {})}
                for g, (t, p) in acc.items()}

    rows = []
    for (c, h, w), relu_in_model in SHAPES:
        shape = (args.batch, c, h, w)

        def act():
            return torch.randn(shape, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

        nbytes = act().numel() * 2
        nsets = max(2, -(-4 * l2 // (2 * nbytes)))
        sets = []
        for _ in range(nsets):
            x, g = act(), act()
            prm = [torch.randn(c, device=dev) for _ in range(2)] + [torch.zeros(c, device=dev),
                                                                    torch.ones(c, device=dev)]
            y, mean, invstd = C.batchnorm_cl_forward(x, *prm, 0.1, 1e-5, relu_in_model)
            sets.append((x, g, y, mean, invstd, *prm))
        for relu in sorted({False, relu_in_model}):
            def fwd_native(x, g, y, mean, invstd, w, b, rm, rv):
                return C.batchnorm_cl_forward(x, w, b, rm, rv, 0.1, 1e-5, relu)

            def fwd_eager(x, g, y, mean, invstd, w, b, rm, rv):
                out = torch.ops.aten.native_batch_norm(x, w, b, rm, rv, True, 0.1, 1e-5)[0]
                return torch.relu_(out) if relu else out

            def bwd_native(x, g, y, mean, invstd, w, b, rm, rv):
                return C.batchnorm_cl_backward(g, x, w, b, mean, invstd, relu)

            def bwd_eager(x, g, y, mean, invstd, w, b, rm, rv):
                gg = torch.ops.aten.threshold_backward(g, y, 0) if relu else g
                return torch.ops.aten.native_batch_norm_backward(gg, x, w, rm, rv, mean, invstd, True, 1e-5,
                                                                 [True, True, True])

            row = {"shape": list(shape), "relu": relu, "mb": round(nbytes / 2**20, 1)}
            for name, fn in (("fwd_native", fwd_native), ("fwd_eager", fwd_eager), ("bwd_native", bwd_native),
                             ("bwd_eager", bwd_eager)):
                row[f"{name}_us"] = round(timeit(fn, sets), 1)
                row[f"{name}_kernels"] = per_kernel(fn, sets, nbytes)
            rows.append(row)
        del sets
    return {"rows": rows}


def profile_step(args):
    import torch
    import torch.nn.functional as F
    from torch.profiler import ProfilerActivity, profile

    from torch_cgx_b200.models import resnet50

    torch.manual_seed(0)
    model = resnet50().cuda().to(memory_format=torch.channels_last)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    x = torch.randn(args.batch, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    target = torch.randint(0, 1000, (args.batch,), device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x), target)
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    groups = {}
    for name, us in kernel_times(prof):
        g, _ = group_of(name)
        groups[g] = groups.get(g, 0.0) + us / args.steps / 1e3
    return {"profile_step_ms": {g: round(v, 3) for g, v in sorted(groups.items())},
            "total_kernel_ms": round(sum(groups.values()), 3), "batch": args.batch, "model": "resnet50",
            "note": "kernel time per step, torch.profiler, no DDP, bf16 autocast, channels_last"}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=128)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--profile-step", action="store_true")
    args = p.parse_args()

    import torch

    assert torch.cuda.is_available(), "batchnorm_bench.py measures on a GPU"
    out = profile_step(args) if args.profile_step else bench_kernels(args)
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
