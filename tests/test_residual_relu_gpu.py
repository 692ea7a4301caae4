"""The native residual join (``C.residual_relu_forward`` / ``C.residual_relu_backward``) against the
eager composition it replaces, bitwise: ``relu_(a + b)`` forward, the autograd engine's gradient
accumulation followed by ``threshold_backward(grad, y, 0)`` backward. NaN positions must match and
every other element bit for bit, the sign of zero included (NaN payloads are not compared).

Also one training step of ResNet-18 (CIFAR stem) and ResNet-50 under bf16 autocast and
channels_last with the native join against the same step with the eager join.
"""
import copy

import pytest
import torch

import torch_cgx_b200 as cgx

from _bitwise import mismatch
from _edge_inputs import edge_inputs

pytestmark = pytest.mark.gpu

C = cgx._C
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_INT = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
# numel 1, odd numels (vector tail, several blocks), and a layer1 block output at batch 128
SHAPES = {"one": (1, 1, 1, 1), "odd": (3, 5, 7, 9), "odd_big": (5, 17, 13, 37), "layer1": (128, 256, 56, 56)}


def assert_same(a, b, what=""):
    """NaN-aware bitwise equality, evaluated on the device (the layer1 case has 103 M elements)."""
    assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride(), what
    iv = _INT[a.dtype]
    na, nb = torch.isnan(a), torch.isnan(b)
    ok = torch.equal(na, nb) and not ((a.view(iv) != b.view(iv)) & ~na).any().item()
    if not ok:
        pytest.fail(f"{what}: {mismatch(a.contiguous().reshape(-1), b.contiguous().reshape(-1))}")


def specials(dtype):
    """Values whose sums exercise every rule: signed zeros, infinities, NaN, subnormals, the largest
    finite value (sums overflow to inf) and neighbours of 1 (sums round to nearest even)."""
    fi = torch.finfo(dtype)
    one_up = 1.0 + fi.eps
    return torch.tensor([0.0, -0.0, 1.0, -1.0, float("inf"), float("-inf"), float("nan"), fi.tiny / 4, -fi.tiny / 4,
                         fi.tiny, fi.max, -fi.max, fi.eps / 2, -fi.eps / 2, one_up, -one_up, fi.eps / 4, 3.0],
                        dtype=torch.float64).to(dtype)


def operands(dtype, shape, seed, k):
    """k tensors of `shape`: random normals with the hostile buckets of edge_inputs planted, and
    every pair of special values at the start."""
    n = 1
    for s in shape:
        n *= s
    g = torch.Generator(device="cpu").manual_seed(seed)
    if n <= 1 << 20:
        outs, _ = edge_inputs(dtype, n, 64, seed, world=k)
        outs = [o.cuda() for o in outs]
    else:  # the layer1 case: random data made on the device, specials planted below
        gg = torch.Generator(device="cuda").manual_seed(seed)
        outs = [torch.randn(n, generator=gg, device="cuda", dtype=torch.float32).to(dtype) for _ in range(k)]
    sp = specials(dtype).cuda()
    m = sp.numel()
    if n >= m * m and k >= 2:  # all (x, y) pairs of specials on operands 0 and 1
        outs[0][: m * m] = sp.repeat_interleave(m)
        outs[1][: m * m] = sp.repeat(m)
    elif k >= 2:
        perm = torch.randint(0, m, (2, n), generator=g)
        outs[0][:] = sp[perm[0].cuda()]
        outs[1][:] = sp[perm[1].cuda()]
    return [o.view(shape) for o in outs]


def layout(t, fmt):
    return t.contiguous(memory_format=torch.channels_last) if fmt == "channels_last" else t.contiguous()


def eager_forward(a, b):
    return torch.relu_(a + b)


def eager_backward(y, ga, gb):
    return torch.ops.aten.threshold_backward(ga if gb is None else ga + gb, y, 0)


@pytest.mark.parametrize("shape", list(SHAPES), ids=list(SHAPES))
@pytest.mark.parametrize("fmt", ["contiguous", "channels_last"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_join_matches_eager_bitwise(dtype, fmt, shape):
    a, b, ga, gb = (layout(t, fmt) for t in operands(dtype, SHAPES[shape], 1, 4))
    y = C.residual_relu_forward(a, b)
    y_ref = eager_forward(a, b)
    assert_same(y, y_ref, "forward")
    # gradients: an independent pair, and the specials again against the forward's NaNs and zeros
    for gx, gy in ((ga, gb), (a, b)):
        assert_same(C.residual_relu_backward(y, gx, gy), eager_backward(y_ref, gx, gy), "backward with gb")
        assert_same(C.residual_relu_backward(y, gx, None), eager_backward(y_ref, gx, None), "backward without gb")
        assert_same(C.residual_relu_backward(y, gx), eager_backward(y_ref, gx, None), "backward, gb omitted")


@pytest.mark.parametrize("n", [1, 7, 8, 4103, 70001])
@pytest.mark.parametrize("off", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f16", "bf16"])
def test_unaligned_views_take_the_scalar_path(dtype, off, n):
    """Views at element offsets 1 and 3 (not 16-byte aligned) of larger buffers, for the operands and
    for y in backward: results match and the buffers are left as they were."""
    bufs = operands(dtype, (n + off + 16,), 7 + off, 4)
    guard = [t.clone() for t in bufs]
    a, b, ga, gb = (t[off: off + n] for t in bufs)
    y = C.residual_relu_forward(a, b)
    y_ref = eager_forward(a, b)
    assert_same(y, y_ref, "forward")
    yv = torch.empty(n + off, dtype=dtype, device="cuda")[off:]  # an unaligned y in backward as well
    yv.copy_(y)
    for y_in in (y, yv):
        assert_same(C.residual_relu_backward(y_in, ga, gb), eager_backward(y_ref, ga, gb), "backward with gb")
        assert_same(C.residual_relu_backward(y_in, ga, None), eager_backward(y_ref, ga, None), "backward without gb")
    for t, g in zip(bufs, guard):
        assert_same(t, g, "inputs untouched")


def test_rejects_operands_it_cannot_walk_linearly():
    a = torch.randn(2, 8, 4, 4, device="cuda")
    ok = torch.randn_like(a)
    with pytest.raises(RuntimeError, match="sizes"):
        C.residual_relu_forward(a, torch.randn(2, 8, 4, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="Half|dtype|Float"):
        C.residual_relu_forward(a, ok.half())
    with pytest.raises(RuntimeError, match="strides"):
        C.residual_relu_forward(a, ok.contiguous(memory_format=torch.channels_last))
    with pytest.raises(RuntimeError, match="CUDA"):
        C.residual_relu_forward(a, ok.cpu())
    with pytest.raises(RuntimeError, match="dense"):
        wide = torch.randn(2, 8, 4, 8, device="cuda")
        C.residual_relu_forward(wide[..., ::2], wide[..., 1::2])
    with pytest.raises(RuntimeError, match="unsupported dtype"):
        C.residual_relu_forward(a.double(), ok.double())
    y = C.residual_relu_forward(a, ok)
    with pytest.raises(RuntimeError, match="gb.*sizes"):
        C.residual_relu_backward(y, ok, torch.randn(2, 8, 4, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="ga.*strides"):
        C.residual_relu_backward(y, ok.contiguous(memory_format=torch.channels_last), None)


# ---- one training step of the models, native join vs eager join -------------------------------

class _Counting:
    """Stands in for the extension inside residual.py and counts the join's calls."""

    def __init__(self, C):
        self.C, self.calls = C, {"residual_relu_forward": 0, "residual_relu_backward": 0}

    def __getattr__(self, name):
        fn = getattr(self.C, name)
        if name in self.calls:
            def counted(*a, **k):
                self.calls[name] += 1
                return fn(*a, **k)
            return counted
        return fn


def _train_step(net, x, y):
    opt = torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = torch.nn.functional.cross_entropy(net(x), y)
    loss.backward()
    grads = [p.grad.clone() for p in net.parameters()]
    opt.step()
    return loss.detach(), grads


@pytest.mark.parametrize("arch", ["resnet18_cifar", "resnet50"])
def test_training_step_bitwise_equal_to_eager_join(arch, monkeypatch):
    from torch_cgx_b200.models import residual, resnet18, resnet50

    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    torch.manual_seed(0)
    if arch == "resnet50":
        net0, size, nblocks = resnet50(num_classes=100), 64, 16
    else:
        net0, size, nblocks = resnet18(num_classes=10, cifar_stem=True), 32, 8
    # the last BN of every branch starts at zero weight; random weights make every join non-trivial
    with torch.no_grad():
        for m in net0.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
    net0 = net0.cuda().to(memory_format=torch.channels_last)
    x = torch.randn(4, 3, size, size, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (4,), device="cuda")

    native, eager = copy.deepcopy(net0), copy.deepcopy(net0)
    counting = _Counting(residual._C)
    monkeypatch.setattr(residual, "_C", counting)
    loss_n, grads_n = _train_step(native, x, y)
    torch.cuda.synchronize()
    # every join runs natively; in backward all but the last block's: the pooling's backward hands it a
    # gradient in another memory format than y, so that one takes the eager threshold_backward
    assert counting.calls == {"residual_relu_forward": nblocks, "residual_relu_backward": nblocks - 1}, counting.calls

    monkeypatch.setattr(residual, "fusable", lambda *ts: False)
    loss_e, grads_e = _train_step(eager, x, y)
    assert counting.calls["residual_relu_forward"] == nblocks  # the eager run did not touch the kernels

    assert_same(loss_n, loss_e, "loss")
    names = [n for n, _ in native.named_parameters()]
    for name, gn, ge in zip(names, grads_n, grads_e):
        assert_same(gn, ge, f"grad of {name}")
    for (name, pn), pe in zip(native.named_parameters(), eager.parameters()):
        assert_same(pn.detach(), pe.detach(), f"updated {name}")
    for (name, bn), be in zip(native.named_buffers(), eager.buffers()):
        if bn.is_floating_point():
            assert_same(bn, be, f"buffer {name}")
        else:
            assert torch.equal(bn, be), name
