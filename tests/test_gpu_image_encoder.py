"""DAMSM image encoder on the GPU: every convolution kind, the pooling kernels and the whole CNN_ENCODER (forward and
input gradient) on both engines (exact-fp32 SIMT and the f16x3 tensor cores) against the float64 oracle
(oracle/image_encoder_oracle.py), and bitwise-equal repeat backward runs."""
import pytest
import torch
import torch.nn.functional as F

from objgan_b200 import lib, model, ops
from objgan_b200.ops import _p
from oracle import image_encoder_oracle as E

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]


@pytest.fixture
def engine(request, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", request.param)
    return request.param


_enc = {}


def encoder():
    if not _enc:
        net = model.CNN_ENCODER(256)
        net.load_state_dict(E.test_state_dict(net.state_dict(), seed=0))
        _enc["net"] = net.to(DEV)
        _enc["sd64"] = {k: (v.double() if v.is_floating_point() else v).to(DEV) for k, v in net.state_dict().items()}
    return _enc["net"], _enc["sd64"]


def _rel_max(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def _rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _nhwc(x):
    return ops.to_nhwc(x.float().contiguous())


def _nchw(y, c):
    return y[..., :c].permute(0, 3, 1, 2)


# (name, cin, cout, kernel, stride, padding, input size); the 1x1 case runs three siblings fused along N
KINDS = [("1x1_fused", 192, (64, 48, 64), (1, 1), 1, (0, 0), 35), ("1x7", 128, 128, (1, 7), 1, (0, 3), 17),
         ("7x1", 128, 192, (7, 1), 1, (3, 0), 17), ("1x3", 384, 384, (1, 3), 1, (0, 1), 8),
         ("3x1", 384, 384, (3, 1), 1, (1, 0), 8), ("3x3_p0", 32, 32, (3, 3), 1, (0, 0), 149),
         ("3x3_p1", 64, 96, (3, 3), 1, (1, 1), 35), ("5x5", 48, 64, (5, 5), 1, (2, 2), 35),
         ("s2_299", 3, 32, (3, 3), 2, (0, 0), 299), ("s2_35", 288, 384, (3, 3), 2, (0, 0), 35),
         ("s2_17", 192, 320, (3, 3), 2, (0, 0), 17)]


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("kind", KINDS, ids=[k[0] for k in KINDS])
def test_conv_kind(engine, kind):
    name, cin, couts, (kh, kw), stride, pad, size = kind
    couts = couts if isinstance(couts, tuple) else (couts,)
    g = torch.Generator().manual_seed(7)
    n = 16 if size <= 17 else 2           # 8x8 maps at 16 images reach the tensor cores (TC_MIN_PIXELS)
    convs = []
    for co in couts:
        c = model.BasicConv2d(cin, co, (kh, kw), stride, pad)
        c.conv.weight.data = torch.randn(co, cin, kh, kw, generator=g) * (2.0 / (cin * kh * kw)) ** 0.5
        c.bn.weight.data = 1 + 0.1 * torch.randn(co, generator=g)
        c.bn.bias.data = 0.1 * torch.randn(co, generator=g)
        c.bn.running_mean.data = 0.1 * torch.randn(co, generator=g)
        c.bn.running_var.data = 1 + 0.2 * torch.rand(co, generator=g)
        convs.append(c.to(DEV).requires_grad_(False))
    layer = model._enc_layer(convs)
    x = torch.randn(n, cin, size, size, generator=g).to(DEV)
    xin = _nhwc(x)
    oh, ow = layer.out_hw(size, size)
    y = torch.empty((n, oh, ow, layer.cout), device=DEV)
    ops.enc_conv_fwd(layer, xin, y)
    gy = torch.randn(n, layer.cout, oh, ow, generator=g).to(DEV)
    # oracle: each BasicConv2d in float64, the siblings concatenated; the input gradient goes through OUR ReLU mask
    # (a pre-activation within rounding of 0 may take either side)
    xr = x.double().requires_grad_(True)
    pre = []
    for c in convs:
        pre.append(F.batch_norm(F.conv2d(xr, c.conv.weight.double(), None, stride, pad), c.bn.running_mean.double(),
                                c.bn.running_var.double(), c.bn.weight.double(), c.bn.bias.double(), False, 0.0, E.BN_EPS))
    pre = torch.cat(pre, 1)
    assert _rel_max(_nchw(y, layer.cout), F.relu(pre)) <= 1e-3
    gp = (_nhwc(gy) * (y > 0)).contiguous()
    (pre * _nchw(gp, layer.cout).double()).sum().backward()
    gx = ops.enc_conv_dgrad(layer, gp, size, size)
    assert _rel_max(_nchw(gx, cin), xr.grad) <= 1e-3


@pytest.mark.parametrize("size", [147, 71, 35, 17])
def test_maxpool(size):
    g = torch.Generator().manual_seed(size)
    x = torch.randn(3, 64, size, size, generator=g).to(DEV)
    x[:, :, 0:4, 0:4] = 0.0                              # ties: the first maximum in scan order takes the gradient
    xn = _nhwc(x)
    oh = (size - 3) // 2 + 1
    y = torch.empty((3, oh, oh, 64), device=DEV)
    lib.get()
    ops._call("og_maxpool3s2_fwd", _p(xn), 3, size, size, 64, _p(y), 64, 0)
    ref = F.max_pool2d(x, 3, 2)
    assert torch.equal(_nchw(y, 64), ref)
    gy = torch.randn(ref.shape, generator=g).to(DEV)
    xr = x.double().requires_grad_(True)
    (F.max_pool2d(xr, 3, 2) * gy.double()).sum().backward()
    gx = torch.empty_like(xn)
    ops._call("og_maxpool3s2_bwd", _p(xn), _p(_nhwc(gy)), 64, 0, 3, size, size, 64, _p(gx))
    assert _rel_max(_nchw(gx, 64), xr.grad) <= 1e-6


@pytest.mark.parametrize("size", [35, 17, 8])
def test_avgpool(size):
    g = torch.Generator().manual_seed(size)
    x = torch.randn(3, 64, size, size, generator=g).to(DEV)
    xn = _nhwc(x)
    y = torch.empty_like(xn)
    ops._call("og_avgpool3s1_fwd", _p(xn), 3, size, size, 64, _p(y))
    xr = x.double().requires_grad_(True)
    ref = F.avg_pool2d(xr, 3, 1, 1)
    assert _rel_max(_nchw(y, 64), ref) <= 1e-6
    gy = torch.randn(ref.shape, generator=g).to(DEV)
    (ref * gy.double()).sum().backward()
    gx = torch.empty_like(xn)
    ops._call("og_avgpool3s1_bwd", _p(_nhwc(gy)), 3, size, size, 64, _p(gx))
    assert _rel_max(_nchw(gx, 64), xr.grad) <= 1e-6


def _encoder_case(b, size, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(b, 3, size, size, generator=g) * 2 - 1).to(DEV)
    a = torch.randn(b, 256, 17, 17, generator=g).to(DEV)
    c = torch.randn(b, 256, generator=g).to(DEV)
    return x, a, c


def _oracle(sd64, x, a, c):
    xr = x.double().requires_grad_(True)
    f, code = E.cnn_encoder_forward(sd64, xr)
    ((f * a.double()).sum() + (code * c.double()).sum()).backward()
    return f.detach(), code.detach(), xr.grad


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("b", [1, 3, 16])
def test_encoder_forward(engine, b):
    net, sd64 = encoder()
    x, _, _ = _encoder_case(b, 256, b)
    with torch.no_grad():
        f, code = net(x)
        rf, rc = E.cnn_encoder_forward(sd64, x.double())
    assert f.shape == (b, 256, 17, 17) and code.shape == (b, 256)
    assert _rel_max(f, rf) <= 1e-3, engine
    assert _rel_max(code, rc) <= 1e-3, engine


def test_encoder_input_gradient(monkeypatch):
    """Both engines within 1e-2 relative L2 of the float64 oracle, f16x3 no further than 3x simt + 1e-3."""
    net, sd64 = encoder()
    x, a, c = _encoder_case(4, 256, 11)
    rf, rc, rg = _oracle(sd64, x, a, c)
    err = {}
    for engine in ENGINES:
        monkeypatch.setattr(ops, "CONV_ENGINE", engine)
        xg = x.clone().requires_grad_(True)
        f, code = net(xg)
        ((f * a).sum() + (code * c).sum()).backward()
        err[engine] = _rel_l2(xg.grad, rg)
        print(f"{engine}: input-gradient relative L2 {err[engine]:.3e}, max {_rel_max(xg.grad, rg):.3e}")
    assert max(err.values()) <= 1e-2, err
    assert err["f16x3"] <= 3 * err["simt"] + 1e-3, err


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_backward_deterministic(engine):
    net, _ = encoder()
    x, a, c = _encoder_case(16, 256, 5)
    grads = []
    for _ in range(2):
        xg = x.clone().requires_grad_(True)
        f, code = net(xg)
        ((f * a).sum() + (code * c).sum()).backward()
        grads.append(xg.grad)
    assert torch.equal(grads[0], grads[1])


def test_no_grad_keeps_nothing():
    net, _ = encoder()
    x, _, _ = _encoder_case(2, 256, 3)
    torch.cuda.synchronize()
    with torch.no_grad():
        f, code = net(x)
    del f, code
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    f, code = net(x)          # x does not require grad: the forward keeps no buffers either
    assert torch.cuda.memory_allocated() - base < 8 * 1024 * 1024


def test_bn_refold_after_load():
    net, _ = encoder()
    x, _, _ = _encoder_case(1, 256, 9)
    with torch.no_grad():
        f0, _ = net(x)
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        sd2 = dict(sd)
        sd2["Conv2d_1a_3x3.bn.running_var"] = sd["Conv2d_1a_3x3.bn.running_var"] * 2
        net.load_state_dict(sd2)
        f1, _ = net(x)
        net.load_state_dict(sd)
        f2, _ = net(x)
    assert not torch.equal(f0, f1)
    assert torch.equal(f0, f2)
