"""GPU tests of the tensor-core convolution's schedule (conv_tc.cu): the N tile width is fitted to each layer, the
last channel chunk issues only the k-steps it needs, and a reduction may be split over several CTAs.  None of that
may change a result: an output element's k-sum has the same stages, partial sums and order whatever the tile width,
so outputs are compared bitwise where only the tiling differs, and against the torch-CPU fp32 convolution at the
1e-4 bar of test_gpu_tc.py otherwise."""
import pytest
import torch
import torch.nn.functional as F

from objgan_b200 import model, ops
from objgan_b200.lib import PAD_REFLECT, PAD_ZERO, UPSAMPLE2X

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert torch.isfinite(a).all()
    return (a - b).abs().max().item() / b.abs().max().item()


def _conv(w, x, mode=PAD_REFLECT, **kw):
    """NCHW output of a Conv2dP holding weight w (cout, cin, 3, 3) on the NCHW input x, on the GPU."""
    m = model.Conv2dP(w.shape[1], w.shape[0], 3, 1, 1, mode=mode, **kw).to(DEV)
    with torch.no_grad():
        m.weight.copy_(w)
        y = m(ops.to_nhwc(x.to(DEV)))
    return ops.to_nchw(y, w.shape[0])


def test_n_tile_width_does_not_change_results(monkeypatch):
    """A 400-channel layer runs as 4 tiles of 104 columns; the same output channels computed as layers of 200 (2 x
    104), 96, 64 and 48 columns, cut across the wide layer's tile boundaries, are bitwise equal to its columns.  (At
    <= 32 channels the stacked-weight form takes over, which drops the a_lo * w_lo term: not compared here.)"""
    monkeypatch.setattr(ops, "CONV_ENGINE", "f16x3")
    torch.manual_seed(11)
    # 128 pixel tiles: even the one-N-tile layers have enough CTAs not to split the reduction (which would add the
    # slices' partial outputs in another order)
    cin, n, h = 200, 4, 64
    w = torch.randn(400, cin, 3, 3) * 0.05
    x = torch.randn(n, cin, h, h)
    # the operand scale comes from max|w|: give every narrow layer the wide layer's maximum (output channel 100)
    w[100, 0, 0, 0] = 4 * w.abs().max()
    wide = _conv(w, x)
    ref = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w)
    assert _rel(wide, ref) <= 1e-4
    for lo, cnt in ((4, 200), (100, 96), (92, 64), (60, 48)):
        narrow = _conv(w[lo:lo + cnt], x)
        assert torch.equal(narrow, wide[:, lo:lo + cnt]), (lo, cnt)


EDGES = [
    # cin, cout, mode, split, N, H, W: what each CTA's reduction looks like
    (48, 96, UPSAMPLE2X, 48, 2, 32, 32),    # upsample phases, C <= 64: nk = 4 taps x 1 chunk, last chunk 3 k-steps
    (64, 48, PAD_REFLECT, 0, 2, 48, 48),    # nk = 9 (odd) x 1 full chunk
    (24, 96, PAD_ZERO, 0, 3, 40, 40),       # nk = 9, the only chunk 2 k-steps deep
    (8, 104, PAD_ZERO, 0, 2, 64, 64),       # one k-step per stage; 104 columns in one tile
    (200, 200, PAD_REFLECT, 0, 4, 16, 16),  # 8 pixel tiles: the reduction is split over CTAs; last chunk 1 k-step
    (130, 136, PAD_ZERO, 0, 2, 16, 16),     # split reduction, 3 chunks (last 1 k-step), N tiles of 72 -> 96 columns
]


@pytest.mark.parametrize("engine,tol", [("f16x3", 1e-4)])
@pytest.mark.parametrize("case", EDGES)
def test_pipeline_edges(case, engine, tol, monkeypatch):
    cin, cout, mode, split, n, h, w_ = case
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(cin + cout + h)
    m = model.Conv2dP(cin, cout, 3, 1, 1, mode=mode, split=split).to(DEV)
    assert ops._tc_kind(n, h, w_, ops.cpad(cin), 3, 3, 1, 1, mode)
    x = torch.randn(n, cin, h, w_)
    w = m.weight.detach().cpu().clone()
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    if mode == PAD_REFLECT:
        yr = F.conv2d(F.pad(xr, (1, 1, 1, 1), mode="reflect"), wr)
    elif mode == UPSAMPLE2X:
        yr = F.conv2d(F.interpolate(xr, scale_factor=2, mode="nearest"), wr, None, 1, 1)
    else:
        yr = F.conv2d(xr, wr, None, 1, 1)
    gy = torch.randn_like(yr)
    gxr, gwr = torch.autograd.grad(yr, (xr, wr), gy)
    xg = x.to(DEV).requires_grad_(True)
    y_nhwc = m(ops.to_nhwc(xg))
    if split:
        sp = ops.cpad(split)
        y = torch.cat((y_nhwc[..., :split], y_nhwc[..., sp:sp + split]), -1).permute(0, 3, 1, 2)
        gfull = torch.zeros_like(y_nhwc)
        g_nhwc = gy.permute(0, 2, 3, 1).to(DEV)
        gfull[..., :split] = g_nhwc[..., :split]
        gfull[..., sp:sp + split] = g_nhwc[..., split:]
        assert _rel(y, yr) <= tol, ("fwd", _rel(y, yr))
        y_nhwc.backward(gfull)
    else:
        y = ops.to_nchw(y_nhwc, cout)
        assert _rel(y, yr) <= tol, ("fwd", _rel(y, yr))
        y.backward(gy.to(DEV))
    assert _rel(xg.grad, gxr) <= tol, ("dgrad", _rel(xg.grad, gxr))
    assert _rel(m.weight.grad, gwr) <= tol, ("wgrad", _rel(m.weight.grad, gwr))


def test_two_runs_bitwise_equal(monkeypatch):
    """Forward, input and weight gradient of the res-block conv1 shape (K = 400) and of a split-reduction layer,
    twice: bitwise equal."""
    monkeypatch.setattr(ops, "CONV_ENGINE", "f16x3")
    for cin, cout, split, n, h in ((194, 388, 194, 2, 64), (200, 200, 0, 4, 16)):
        torch.manual_seed(cin + h)
        m = model.Conv2dP(cin, cout, 3, 1, 1, mode=PAD_REFLECT, split=split).to(DEV)
        x = ops.to_nhwc(torch.randn(n, cin, h, h, device=DEV))
        runs = []
        for _ in range(2):
            xg = x.clone().requires_grad_(True)
            m.weight.grad = None
            y = m(xg)
            g = torch.randn(y.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
            y.backward(g)
            runs.append((y.detach().clone(), xg.grad.clone(), m.weight.grad.clone()))
        for a, b in zip(*runs):
            assert torch.equal(a, b)
