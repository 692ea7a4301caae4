"""Adaptive per-layer widths on one H100: the estimator kernel, the DDP step, mixed-width allreduce.

    python bench/adaptive_bits_bench.py [--steps 20] [--warmup 5]

(a) ``ops.quantization_error`` over the ResNet-50 and GPT-2-medium gradient layer tables (fp32,
    bucket 512, the layers the hook compresses), with 1 and 7 candidates: time, GB/s over the
    bytes read once, and the share of the 3.35 TB/s HBM3 data-sheet bandwidth. If seven candidates
    take clearly longer than one, arithmetic bounds the kernel, otherwise memory does.
(b) ResNet-50 DDP steps at world 1 (batch 128, bf16 autocast, channels_last, SGD), device-timed with
    CUDA events: native hook 4 bits, Python hook 4 bits, and AdaptiveCGXState on the Python and on
    the native hook at period 1, 100 and "never" (one decision right after registration, inside
    the warm-up). The arms run in two rounds, the second in reverse order.
(c) The fused allreduce (world 1: quantize + decode in one kernel) of every ResNet-50 bucket with
    the adaptive assignment against uniform 4 bits.
(d) The host time of one decision on the ResNet-50 layer table, replayed call by call: group sum of
    the float64 table plus the copy to the host, the allocator (C++ against the NumPy reference),
    the broadcast of the widths and their application to the registry.
Prints the card and its power limit first; one JSON line per result.
"""
import argparse
import json
import socket
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import torch_cgx_b200 as cgx  # noqa: E402
from torch_cgx_b200 import models  # noqa: E402

HBM_BPS = 3.35e12
BUCKET = 512
MIN_SIZE = 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def emit(d):
    print(json.dumps(d), flush=True)


def time_events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def layer_table(net):
    layers, off = [], 0
    for p in net.parameters():
        if p.dim() > 1 and p.numel() >= MIN_SIZE:
            layers.append((off, p.numel(), 4, BUCKET))
        off += p.numel()
    return layers, off


def bench_estimator():
    for name, ctor in (("resnet50", models.resnet50), ("gpt2-medium", models.gpt2_medium)):
        layers, n = layer_table(ctor())
        g = torch.randn(n, device="cuda") * 1e-3
        nbytes = 4 * sum(l[1] for l in layers)
        for cands in ((4,), (2, 3, 4, 5, 6, 7, 8)):
            for stoch in (False, True):
                fn = lambda: cgx.ops.quantization_error(g, layers, cands, stochastic=stoch)  # noqa: E731
                for _ in range(5):
                    fn()
                t = time_events(fn, 50)
                emit({"part": "a", "model": name, "layers": len(layers), "elements": nbytes // 4,
                      "candidates": len(cands), "stochastic": stoch, "time_us": round(t * 1e6, 1),
                      "GBps": round(nbytes / t / 1e9, 1), "hbm_share": round(nbytes / t / HBM_BPS, 3)})


NEVER = 1 << 40  # a period no run reaches: only the decision right after registration


def make_step(kind, period=None):
    torch.manual_seed(0)
    net = models.resnet50().cuda().to(memory_format=torch.channels_last)
    ddp = torch.nn.parallel.DistributedDataParallel(net, device_ids=[0], gradient_as_bucket_view=True)
    params = {"bits": 4, "bucket_size": BUCKET}
    if kind in ("adaptive", "adaptive_native"):
        state = cgx.AdaptiveCGXState(None, MIN_SIZE, params, period=period)
        cgx.register_cgx_hook(ddp, state, native=kind == "adaptive_native")
    else:
        state = cgx.CGXState(None, MIN_SIZE, params)
        if kind == "native":
            cgx.register_cgx_hook(ddp, state)
        else:
            ddp.register_comm_hook(state, cgx.cgx_hook)
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    gen = torch.Generator("cuda").manual_seed(1)
    x = torch.randn(128, 3, 224, 224, device="cuda", generator=gen).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (128,), device="cuda", generator=gen)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(ddp(x), y)
        loss.backward()
        opt.step()
    return step, state, ddp


def bench_steps(steps, warmup):
    arms = [("native", None), ("python", None)]
    arms += [(kind, period) for period in (1, 100, NEVER) for kind in ("adaptive", "adaptive_native")]
    adaptive_state = None
    for rnd, order in enumerate((arms, arms[::-1])):
        for kind, period in order:
            cgx.reset_layers()
            step, state, ddp = make_step(kind, period)
            for _ in range(max(warmup, 4)):
                step()
            torch.cuda.synchronize()
            t = time_events(step, steps)
            emit({"part": "b", "round": rnd, "hook": kind, "period": "never" if period == NEVER else period,
                  "steps": steps, "step_ms": round(t * 1e3, 2), "images_per_s": round(128 / t, 1)})
            if kind == "adaptive" and period == 100:
                adaptive_state = state
            del step, ddp
    return adaptive_state


def bench_decision(state, reps=20):
    """One decision's host work, replayed with the calls both hooks make."""
    import time

    from torch_cgx_b200 import _C
    from torch_cgx_b200.ops.bit_allocation import layer_wire_bytes
    from torch_cgx_b200.ops.oracle import allocate_bits_reference

    rows = list(state.adapted_layers)
    table = state.last_errors.cuda()
    K = len(state.candidate_bits)
    numels = [n for (_, _, _, n) in rows]
    budget = sum(layer_wire_bytes(n, 4, BUCKET) for n in numels)
    current = [state.assignment.get((b, l), 4) for (b, l, _, _) in rows]
    err = state.last_errors.numpy()
    args = (numels, [BUCKET] * len(rows), list(state.candidate_bits), budget, current)

    def timed(fn):
        best = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            best.append(time.perf_counter() - t0)
        return round(sorted(best)[len(best) // 2] * 1e6, 1)  # median

    def group_sum_copy():
        t = table.clone()
        dist.all_reduce(t)
        t.view(-1, K).cpu()

    picked = _C.allocate_bits(err, *args, 4096, 4)
    assert picked == allocate_bits_reference(err, *args, 4096, target_bits=4)
    choice = torch.tensor(picked, dtype=torch.int32)

    def broadcast():
        c = choice.cuda()
        dist.broadcast(c, src=0)
        c.cpu()

    def apply():
        for (b, l, _, _), bits in zip(rows, picked):
            _C.set_quantization_bits(b, l, bits)

    emit({"part": "d", "layers": len(rows), "candidates": K,
          "group_sum_copy_us": timed(group_sum_copy),
          "allocator_cpp_us": timed(lambda: _C.allocate_bits(err, *args, 4096, 4)),
          "allocator_numpy_us": timed(lambda: allocate_bits_reference(err, *args, 4096, target_bits=4)),
          "broadcast_us": timed(broadcast), "apply_from_python_us": timed(apply)})


def bench_mixed_allreduce(state):
    be = cgx.get_backend()
    assign = dict(state.assignment)
    buckets = sorted({b for (b, _) in assign})
    sizes = {b: sum(n for (n, _, _) in cgx._C.registered_bucket(b)) for b in buckets}
    bufs = {b: torch.randn(sizes[b], device="cuda") * 1e-3 for b in buckets}

    def run():
        for b in buckets:
            be.allreduce_bucket(bufs[b], b, True).wait()

    res = {}
    for label in ("adaptive", "uniform4"):
        for (b, l), bits in assign.items():
            cgx.set_quantization_bits(b, l, bits if label == "adaptive" else 4)
        for _ in range(5):
            run()
        res[label] = time_events(run, 50)
    hist = {}
    for v in assign.values():
        hist[v] = hist.get(v, 0) + 1
    emit({"part": "c", "buckets": len(buckets), "elements": sum(sizes.values()),
          "adaptive_us": round(res["adaptive"] * 1e6, 1), "uniform4_us": round(res["uniform4"] * 1e6, 1),
          "width_histogram": dict(sorted(hist.items()))})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adaptive_bits_bench needs a GPU")
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    emit({"card": card(), "torch": torch.__version__})
    bench_estimator()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("cgx", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        state = bench_steps(args.steps, args.warmup)
        bench_decision(state)
        bench_mixed_allreduce(state)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
