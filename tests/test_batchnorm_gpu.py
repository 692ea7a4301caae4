"""The native channels_last BatchNorm (``C.batchnorm_cl_forward`` / ``C.batchnorm_cl_backward``,
``models.batchnorm``) against the eager ops it replaces, bitwise: ``aten.native_batch_norm`` in
training mode (output, saved mean and invstd, running stats) followed by ``relu_``; in backward
``threshold_backward`` then ``aten.native_batch_norm_backward`` (grad_input, grad_weight, grad_bias);
and autograd through ``F.batch_norm`` + ``relu_``. NaN positions must match and every other element
bit for bit.

Also one training step of ResNet-18 (CIFAR stem) and ResNet-50 under bf16 autocast and
channels_last, native BatchNorm against eager BatchNorm.
"""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import torch_cgx_b200 as cgx
from torch_cgx_b200.models import batchnorm as bnmod
from torch_cgx_b200.models.resnet import resnet18, resnet50

from _bitwise import mismatch

pytestmark = pytest.mark.gpu

C = cgx._C
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_INT = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}

# every distinct BatchNorm input of ResNet-50 at batch 128 / 224 px (grid.y = 128, 98 and 25 in
# ATen's launch configuration), then one shape per other branch of it
FLAGSHIP = [(128, 64, 112, 112), (128, 64, 56, 56), (128, 256, 56, 56), (128, 128, 56, 56),
            (128, 128, 28, 28), (128, 512, 28, 28), (128, 256, 28, 28), (128, 256, 14, 14),
            (128, 1024, 14, 14), (128, 512, 14, 14), (128, 512, 7, 7), (128, 2048, 7, 7)]
SMALL = [(4, 64, 5, 5),       # grid.y < 8: no grid merge
         (8, 3, 17, 19), (2, 16, 33, 31), (4, 96, 9, 7), (3, 100, 11, 13), (16, 1000, 3, 3),  # C < 32, odd C
         (64, 256, 1, 1), (5, 40, 1, 1),  # H = W = 1
         (1, 8, 2, 3), (2, 5, 1, 1),      # M smaller than a block
         (8, 100, 16, 16)]                # grid merge on the one-element path, partial last slab


def assert_same(a, b, what=""):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    a, b = a.contiguous(), b.contiguous()
    iv = _INT[a.dtype]
    na, nb = torch.isnan(a), torch.isnan(b)
    ok = torch.equal(na, nb) and not ((a.view(iv) != b.view(iv)) & ~na).any().item()
    if not ok:
        pytest.fail(f"{what}: {mismatch(a.reshape(-1), b.reshape(-1))}")


def make_input(shape, dtype, seed, hostile):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(shape, generator=g, device="cuda") * 3 + 1).to(dtype)
    x = x.contiguous(memory_format=torch.channels_last)
    if hostile:
        n, c = shape[0], shape[1]
        fi = torch.finfo(dtype)
        v = x.permute(0, 2, 3, 1).reshape(-1, c)  # a view of x: [M][C]
        m = v.shape[0]
        specials = [float("nan"), float("inf"), -float("inf"), fi.max, fi.tiny / 4, -fi.tiny]
        for k, s in enumerate(specials):
            if c > k + 1:
                v[(k * 7919) % m, k + 1] = s
        if c > 8:
            v[:, 8] = 2.5             # a constant channel: var = 0
        if c > 9:
            v[:, 9] = fi.max          # mean overflows to inf
        if c > 10:
            v[:, 10] = fi.max / 2     # huge values: m2 overflows
            v[1::2, 10] = -fi.max / 2
        if c > 11:
            v[:, 11] = fi.tiny / 8    # denormal channel
    return x


def params(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    w = torch.randn(c, generator=g, device="cuda")
    b = torch.randn(c, generator=g, device="cuda")
    rm = torch.randn(c, generator=g, device="cuda")
    rv = torch.rand(c, generator=g, device="cuda") + 0.5
    return w, b, rm, rv


def check_forward(shape, dtype, relu, seed=0, hostile=False):
    x = make_input(shape, dtype, seed, hostile)
    w, b, rm, rv = params(shape[1], seed)
    rm2, rv2 = rm.clone(), rv.clone()
    y_ref, mean_ref, invstd_ref = torch.ops.aten.native_batch_norm(x, w, b, rm2, rv2, True, 0.1, 1e-5)
    if relu:
        torch.relu_(y_ref)
    y, mean, invstd = C.batchnorm_cl_forward(x, w, b, rm, rv, 0.1, 1e-5, relu)
    assert y.stride() == y_ref.stride()
    assert_same(y, y_ref, "y")
    assert_same(mean, mean_ref, "save_mean")
    assert_same(invstd, invstd_ref, "save_invstd")
    assert_same(rm, rm2, "running_mean")
    assert_same(rv, rv2, "running_var")

    g = make_input(shape, dtype, seed + 7, hostile)
    g_ref = torch.ops.aten.threshold_backward(g, y_ref, 0) if relu else g
    gx_ref, gw_ref, gb_ref = torch.ops.aten.native_batch_norm_backward(
        g_ref, x, w, rm2, rv2, mean_ref, invstd_ref, True, 1e-5, [True, True, True])
    gx, gw, gb = C.batchnorm_cl_backward(g, x, w, b, mean, invstd, relu)
    assert gx.stride() == gx_ref.stride()
    assert_same(gx, gx_ref, "grad_input")
    assert_same(gw, gw_ref, "grad_weight")
    assert_same(gb, gb_ref, "grad_bias")


@pytest.mark.parametrize("shape", FLAGSHIP, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("relu", [False, True])
def test_forward_flagship_shapes(shape, relu):
    check_forward(shape, torch.bfloat16, relu, seed=1, hostile=relu)


@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("hostile", [False, True])
def test_forward_small_shapes(shape, dtype, relu, hostile):
    check_forward(shape, dtype, relu, seed=2, hostile=hostile)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("relu", [False, True])
def test_forward_layer_shapes_all_dtypes(dtype, relu):
    for shape in [(128, 64, 56, 56), (128, 2048, 7, 7), (32, 256, 28, 28)]:
        check_forward(shape, dtype, relu, seed=3, hostile=True)


def test_forward_unaligned_view():
    """a storage offset that breaks 16-byte alignment takes the one-element path"""
    base = make_input((9, 64, 6, 6), torch.bfloat16, 4, False)
    x = base[1:]  # still channels_last-dense, offset by one image
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    xu = flat[1:].as_strided(x.shape, x.stride())
    xu.copy_(x)
    w, b, rm, rv = params(64, 4)
    rm2, rv2 = rm.clone(), rv.clone()
    y_ref, m_ref, i_ref = torch.ops.aten.native_batch_norm(xu, w, b, rm2, rv2, True, 0.1, 1e-5)
    y, m, i = C.batchnorm_cl_forward(xu, w, b, rm, rv, 0.1, 1e-5, False)
    for a, r in ((y, y_ref), (m, m_ref), (i, i_ref), (rm, rm2), (rv, rv2)):
        assert_same(a, r)
    gu = torch.empty_like(flat)[1:].as_strided(x.shape, x.stride())
    gu.copy_(make_input(x.shape, torch.bfloat16, 5, False))
    ref = torch.ops.aten.native_batch_norm_backward(gu, xu, w, rm2, rv2, m_ref, i_ref, True, 1e-5, [True] * 3)
    for a, r in zip(C.batchnorm_cl_backward(gu, xu, w, b, m, i, False), ref):
        assert_same(a, r)


def test_binding_rejects_bad_operands():
    x = make_input((2, 8, 3, 3), torch.bfloat16, 0, False)
    w, b, rm, rv = params(8, 0)
    with pytest.raises(RuntimeError, match="channels_last"):
        C.batchnorm_cl_forward(x.contiguous(), w, b, rm, rv, 0.1, 1e-5, False)
    with pytest.raises(RuntimeError, match="float32"):
        C.batchnorm_cl_forward(x, w.double(), b, rm, rv, 0.1, 1e-5, False)
    with pytest.raises(RuntimeError, match="channels"):
        C.batchnorm_cl_forward(x, w[:4], b, rm, rv, 0.1, 1e-5, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        C.batchnorm_cl_forward(x.cpu(), w, b, rm, rv, 0.1, 1e-5, False)
    with pytest.raises(RuntimeError, match="strides"):
        C.batchnorm_cl_backward(x.contiguous(), x, w, b, rm, rv, False)
    with pytest.raises(RuntimeError, match="float32"):
        C.batchnorm_cl_backward(x, x, w, b, rm.half(), rv, False)


def _autograd_pair(shape, dtype, relu, seed):
    x0 = make_input(shape, dtype, seed, False)
    bn_n = nn.BatchNorm2d(shape[1]).cuda()
    with torch.no_grad():
        bn_n.weight.normal_()
        bn_n.bias.normal_()
    bn_e = copy.deepcopy(bn_n)
    xn = x0.clone().requires_grad_()
    xe = x0.clone().requires_grad_()
    yn = bnmod.batch_norm_act(bn_n, xn, relu)
    ye = bn_e(xe)
    if relu:
        ye = torch.relu_(ye)
    g = torch.randn_like(yn).contiguous(memory_format=torch.channels_last)
    yn.backward(g)
    ye.backward(g)
    assert_same(yn.detach(), ye.detach(), "y")
    assert_same(xn.grad, xe.grad, "grad_input")
    for (name, pn), pe in zip(bn_n.named_parameters(), bn_e.parameters()):
        assert_same(pn.grad, pe.grad, name)
    for (name, bn_), be in zip(bn_n.named_buffers(), bn_e.buffers()):
        if bn_.is_floating_point():
            assert_same(bn_, be, name)
        else:
            assert torch.equal(bn_, be), name


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("relu", [False, True])
def test_autograd_matches_eager(dtype, relu, monkeypatch):
    # eager fp32 / fp16 BatchNorm runs cuDNN unless it is disabled; bf16 never does
    with torch.backends.cudnn.flags(enabled=dtype == torch.bfloat16):
        n = _count_native(monkeypatch)
        _autograd_pair((16, 64, 14, 14), dtype, relu, seed=5)
        assert n["calls"] == 1


def test_fallbacks():
    bn = nn.BatchNorm2d(8).cuda()
    x = make_input((2, 8, 3, 3), torch.bfloat16, 0, False)
    assert bnmod.native_ok(bn, x)
    assert not bnmod.native_ok(bn, x.contiguous())          # NCHW
    assert not bnmod.native_ok(bn.eval(), x)                # eval mode
    bn.train()
    with torch.backends.cudnn.flags(enabled=True):
        if torch.backends.cudnn.is_available():               # eager runs cuDNN for fp32
            assert not bnmod.native_ok(bn, x.float())
    assert not bnmod.native_ok(bn, x[:1, :, :1, :1])         # one value per channel: eager raises
    bn1 = nn.BatchNorm2d(1).cuda()                            # C = 1, NCHW strides: ATen's contiguous kernels
    x1 = make_input((2, 1, 3, 3), torch.bfloat16, 0, False).contiguous()
    assert x1.is_contiguous(memory_format=torch.channels_last) and not bnmod.native_ok(bn1, x1)
    bn.momentum = None                                       # cumulative average
    assert not bnmod.native_ok(bn, x)


@pytest.mark.parametrize("relu", [False, True])
def test_backward_gradient_with_other_strides_runs_eager(relu, monkeypatch):
    """a gradient whose strides differ from x's takes the eager backward and still matches"""
    calls = {"n": 0}
    real = C.batchnorm_cl_backward

    def counting(*a):
        calls["n"] += 1
        return real(*a)

    monkeypatch.setattr(C, "batchnorm_cl_backward", counting)
    x0 = make_input((4, 32, 6, 6), torch.bfloat16, 6, False)
    bn_n = nn.BatchNorm2d(32).cuda()
    bn_e = copy.deepcopy(bn_n)
    xn, xe = x0.clone().requires_grad_(), x0.clone().requires_grad_()
    yn = bnmod.batch_norm_act(bn_n, xn, relu)
    ye = bn_e(xe)
    ye = torch.relu_(ye) if relu else ye
    g = torch.randn(yn.shape, device="cuda").to(yn.dtype)  # NCHW-contiguous
    yn.backward(g)
    ye.backward(g)
    assert calls["n"] == 0
    assert_same(xn.grad, xe.grad, "grad_input")
    assert_same(bn_n.weight.grad, bn_e.weight.grad, "grad_weight")
    assert_same(bn_n.bias.grad, bn_e.bias.grad, "grad_bias")


def _count_native(monkeypatch):
    n = {"calls": 0}
    real = bnmod.BatchNormAct.apply

    def counting(*a):
        n["calls"] += 1
        return real(*a)

    monkeypatch.setattr(bnmod.BatchNormAct, "apply", counting)
    return n


def _step(model, x, target, native, monkeypatch):
    if not native:
        monkeypatch.setattr(bnmod, "native_ok", lambda bn, x: False)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.cross_entropy(model(x), target)
    loss.backward()
    opt.step()
    monkeypatch.undo()
    return loss.detach()


@pytest.mark.parametrize("arch,batch,px", [("resnet18", 32, 32), ("resnet50", 16, 64), ("resnet50", 128, 224)])
def test_training_step_matches_eager(arch, batch, px, monkeypatch):
    torch.manual_seed(0)
    ctor = resnet18 if arch == "resnet18" else resnet50
    base = ctor(num_classes=10 if arch == "resnet18" else 1000, cifar_stem=arch == "resnet18")
    base = base.cuda().to(memory_format=torch.channels_last)
    m_native, m_eager = copy.deepcopy(base), copy.deepcopy(base)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(batch, 3, px, px, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
    target = torch.randint(0, 10, (batch,), generator=g, device="cuda")

    n = _count_native(monkeypatch)
    nb = {"n": 0}
    real_bwd = C.batchnorm_cl_backward

    def counting_bwd(*a):
        nb["n"] += 1
        return real_bwd(*a)

    monkeypatch.setattr(C, "batchnorm_cl_backward", counting_bwd)
    loss_n = _step(m_native, x, target, True, monkeypatch)
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in base.modules())
    assert n["calls"] == n_bn, "every BatchNorm layer runs natively"
    assert nb["n"] == n_bn, "every BatchNorm backward runs natively"
    loss_e = _step(m_eager, x, target, False, monkeypatch)

    assert_same(loss_n, loss_e, "loss")
    for (name, pn), pe in zip(m_native.named_parameters(), m_eager.parameters()):
        assert_same(pn.grad, pe.grad, f"{name}.grad")
        assert_same(pn.detach(), pe.detach(), name)
    for (name, bn_), be in zip(m_native.named_buffers(), m_eager.buffers()):
        if bn_.is_floating_point():
            assert_same(bn_, be, name)
        else:
            assert torch.equal(bn_, be), name
