"""The ResNets' pair-threaded residual join on CPU.

Every block returns ``(y, alias of y)`` and the next block feeds conv1 and its identity or
downsample path from the two. On CPU the join is the eager ``relu_(a + b)``; with the autograd
Function (``ResidualReLU``) the engine's accumulation of the two gradients moves into the join's
backward. Both must give exactly the gradients of the plain eager model.
"""
import copy
from types import SimpleNamespace

import pytest
import torch

from torch_cgx_b200.models import residual, resnet18, resnet50
from torch_cgx_b200.models.resnet import BasicBlock, Bottleneck


def eager_forward(net, x):
    """The model as it was written before the join was fused: one tensor between blocks."""
    x = net.stem(x)
    for layer in (net.layer1, net.layer2, net.layer3, net.layer4):
        for blk in layer:
            idt = x if blk.downsample is None else blk.downsample(x)
            out = blk.relu(blk.bn1(blk.conv1(x)))
            if isinstance(blk, Bottleneck):
                out = blk.relu(blk.bn2(blk.conv2(out)))
                out = blk.bn3(blk.conv3(out))
            else:
                out = blk.bn2(blk.conv2(out))
            x = blk.relu(out + idt)
    return net.fc(torch.flatten(net.pool(x), 1))


def make(arch):
    torch.manual_seed(0)
    net = resnet50(num_classes=10) if arch == "resnet50" else resnet18(num_classes=10, cifar_stem=True)
    with torch.no_grad():  # zero-initialised last BNs would make every join's first operand 0
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
    x = torch.randn(2, 3, 32, 32)
    y = torch.randint(0, 10, (2,))
    return net, x, y


def grads_of(net, forward, x, y):
    loss = torch.nn.functional.cross_entropy(forward(net, x), y)
    loss.backward()
    return loss.detach(), [p.grad for p in net.parameters()]


def assert_equal_runs(a, b):
    (la, ga), (lb, gb) = a, b
    assert torch.equal(la, lb)
    assert len(ga) == len(gb)
    for i, (u, v) in enumerate(zip(ga, gb)):
        assert u is not None and torch.equal(u, v), i


@pytest.mark.parametrize("arch", ["resnet18_cifar", "resnet50"])
def test_pair_threaded_model_matches_eager(arch):
    net, x, y = make(arch)
    twin = copy.deepcopy(net)
    assert_equal_runs(grads_of(net, lambda n, v: n(v), x, y), grads_of(twin, eager_forward, x, y))
    for bn, be in zip(net.buffers(), twin.buffers()):
        assert torch.equal(bn, be)


def _reference_kernels(calls):
    """CPU stand-ins with the kernels' definitions (bit-exact on CPU), counting the backward calls
    that get no gb."""
    def fwd(a, b):
        return torch.relu(a + b)

    def bwd(y, ga, gb=None):
        calls.append(gb is None)
        return torch.ops.aten.threshold_backward(ga if gb is None else ga + gb, y, 0)

    return SimpleNamespace(residual_relu_forward=fwd, residual_relu_backward=bwd)


@pytest.mark.parametrize("arch", ["resnet18_cifar", "resnet50"])
def test_join_function_matches_eager(arch, monkeypatch):
    """The autograd Function itself, with the kernels replaced by their definitions: the two outputs
    get their gradients separately, the last block's alias gets none, and the result is the eager
    model's."""
    calls = []
    monkeypatch.setattr(residual, "_C", _reference_kernels(calls))
    monkeypatch.setattr(residual, "fusable", lambda *ts: True)
    net, x, y = make(arch)
    twin = copy.deepcopy(net)
    assert_equal_runs(grads_of(net, lambda n, v: n(v), x, y), grads_of(twin, eager_forward, x, y))
    nblocks = 16 if arch == "resnet50" else 8
    assert calls == [True] + [False] * (nblocks - 1)  # backward runs from layer4's last block


def test_join_returns_an_alias_and_the_same_values():
    calls = []
    a, b = torch.randn(2, 4, 3, 3), torch.randn(2, 4, 3, 3)
    ya, yb = residual.residual_relu(a, b)  # CPU: the eager join, one tensor twice
    assert ya is yb and torch.equal(ya, torch.relu(a + b))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(residual, "_C", _reference_kernels(calls))
        mp.setattr(residual, "fusable", lambda *ts: True)
        ar, br = a.clone().requires_grad_(), b.clone().requires_grad_()
        ya, yb = residual.residual_relu(ar, br)
        assert ya.data_ptr() == yb.data_ptr() and torch.equal(ya, yb)
        (ya.sum() + 2 * yb.sum()).backward()
    expect = torch.where(torch.relu(a + b) <= 0, 0.0, 3.0)
    assert torch.equal(ar.grad, expect) and torch.equal(br.grad, expect)
    assert calls == [False]


@pytest.mark.parametrize("block", ["basic", "bottleneck"])
def test_block_accepts_a_plain_tensor(block):
    torch.manual_seed(0)
    if block == "basic":
        blk = BasicBlock(8, 8)
    else:
        blk = Bottleneck(16, 4)
    blk.eval()
    x = torch.randn(2, blk.conv1.in_channels, 5, 5)
    ya, yb = blk(x)
    za, zb = blk((x, x))
    assert torch.equal(ya, za) and torch.equal(yb, zb)
