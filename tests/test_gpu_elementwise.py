"""The bandwidth-bound helpers of csrc/elementwise.cu against float64 restatements, at the shapes the step uses and at
the edges where their index math branches.

Pure data movement (reflection pad forward, row gather, channel copy, channel permute, channel broadcast) must be
bitwise exact.  Everything else is held to a bound derived from its fp32 arithmetic, stated per test: a sum of k fp32
terms is within (k - 1) 2^-24 sum|terms| of the exact sum, a product or quotient adds 2^-24 relative per rounding, and
expf / logf add a few ulps.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from objgan_b200 import ops
from objgan_b200.lib import ACT_LRELU, ACT_SIGMOID, ACT_TANH

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24          # fp32 unit roundoff
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"elementwise worst error {k}: {WORST[k]:.3e} of its bound")


def _call(name, *args):
    ops._call(name, *[ops._p(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _within(name, got, ref, bound):
    """elementwise |got - ref| <= bound (float64 tensors or scalars)"""
    got = got.double()
    assert torch.isfinite(got).all(), name
    r = ((got - ref).abs() / bound).max().item()
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


def _randn(*shape, seed=0):
    return torch.randn(*shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))


# ---------------------------------------------------------------------------------------------------
# reflection pad, nearest-upsample adjoint
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W,C", [(2, 2, 2, 8), (3, 3, 2, 4), (2, 2, 5, 12), (1, 3, 3, 4), (16, 32, 32, 200),
                                     (4, 64, 64, 24), (2, 128, 128, 200)])
def test_reflect_pad(N, H, W, C):
    """Forward bitwise equal to F.pad(reflect); the adjoint sums up to four halo copies of an input element (H or W in
    {2, 3}: one input row feeds several halo rows): <= 3 U sum|terms|."""
    x = _randn(N, H, W, C, seed=H * W + C)
    xp = torch.empty(N, H + 2, W + 2, C, device=DEV)
    _call("og_reflect_pad_fwd", x, N, H, W, C, xp)
    want = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1)
    assert torch.equal(xp, want)
    gp = _randn(N, H + 2, W + 2, C, seed=7)
    gx = torch.empty_like(x)
    _call("og_reflect_pad_bwd", gp, N, H, W, C, gx)
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    F.pad(x64, (1, 1, 1, 1), mode="reflect").backward(gp.double().permute(0, 3, 1, 2))
    xa = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    F.pad(xa, (1, 1, 1, 1), mode="reflect").backward(gp.double().abs().permute(0, 3, 1, 2))
    _within("og_reflect_pad_bwd", gx, x64.grad.permute(0, 2, 3, 1), 3 * U * xa.grad.permute(0, 2, 3, 1) + 1e-45)


@pytest.mark.parametrize("N,H,W,C", [(16, 64, 64, 96), (3, 5, 7, 4), (1, 1, 1, 8)])
def test_upsample2x_bwd(N, H, W, C):
    """Sum of the four children of each pixel (fp32, 3 roundings).  16 x 64^2 x 96 has 1.57 M channel quads: beyond one
    grid-stride trip on an H100."""
    gu = _randn(N, 2 * H, 2 * W, C, seed=C)
    gx = torch.empty(N, H, W, C, device=DEV)
    _call("og_upsample2x_bwd", gu, N, H, W, C, gx)
    g4 = gu.double().reshape(N, H, 2, W, 2, C)
    _within("og_upsample2x_bwd", gx, g4.sum((2, 4)), 3 * U * g4.abs().sum((2, 4)) + 1e-45)


# ---------------------------------------------------------------------------------------------------
# bilinear resize (align_corners=True)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,IH,IW,C,OH,OW", [(4, 64, 64, 16, 512, 512), (2, 128, 128, 16, 512, 512),
                                              (1, 256, 256, 12, 512, 512), (3, 7, 5, 8, 13, 11), (2, 9, 6, 4, 1, 5),
                                              (2, 6, 9, 4, 4, 1), (1, 1, 3, 4, 3, 7)])
def test_bilinear(N, IH, IW, C, OH, OW):
    """Forward and adjoint against F.interpolate(align_corners=True) in float64.  The kernels compute the source
    coordinate dst * (in - 1) / (out - 1) and the weights in fp32 (like ATen): the coordinate is off by <= 2 U in, which
    moves a weight by as much, so the forward is within (4 U (IH + IW) + 8 U) max|x|; the adjoint adds each output's
    four weighted contributions with fp32 atomics, within (k + 8) U of the sum of |contributions| plus the weight error
    4 U (IH + IW) on each of them, k the number of contributions an input receives."""
    x = _randn(N, C, IH, IW, seed=IH + OH)
    xn = x.permute(0, 2, 3, 1).contiguous()
    y = torch.empty(N, OH, OW, C, device=DEV)
    _call("og_bilinear_fwd", xn, N, IH, IW, C, OH, OW, y)
    x64 = x.double().requires_grad_(True)
    ref = F.interpolate(x64, size=(OH, OW), mode="bilinear", align_corners=True)
    idx = 4 * U * (IH + IW) + 8 * U
    _within("og_bilinear_fwd", y, ref.permute(0, 2, 3, 1), idx * x.abs().max().item())
    g = _randn(N, OH, OW, C, seed=3)
    gx = torch.empty(N, IH, IW, C, device=DEV)
    _call("og_bilinear_bwd", g, N, IH, IW, C, OH, OW, gx)
    ref.backward(g.double().permute(0, 3, 1, 2))
    xa = x.double().requires_grad_(True)
    F.interpolate(xa, size=(OH, OW), mode="bilinear", align_corners=True).backward(g.double().abs().permute(0, 3, 1, 2))
    k = 4 * (math.ceil(OH / max(IH - 1, 1)) + 1) * (math.ceil(OW / max(IW - 1, 1)) + 1)
    bound = (k + 8) * U * xa.grad.permute(0, 2, 3, 1) + 4 * U * (IH + IW) * k * g.abs().max().item()
    _within("og_bilinear_bwd", gx, x64.grad.permute(0, 2, 3, 1), bound)


# ---------------------------------------------------------------------------------------------------
# conv bias gradient, activation adjoint
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,C,n_out,acc", [(1, 8, 8, 0), (63, 24, 20, 0), (63, 132, 132, 1), (1 << 20, 16, 12, 0),
                                           (1 << 20, 96, 96, 1)])
def test_channel_sum(P, C, n_out, acc):
    """fp64 sums of fp32 values, rounded once to fp32 (and once more when accumulating): <= 2 U |ref| + 2^-30 sum|x|;
    a second call gives the same bits."""
    x = _randn(P, C, seed=P % 1000 + C) + 0.5
    scratch = torch.empty(C, device=DEV, dtype=torch.float64)
    out0 = _randn(n_out, seed=9)
    out = out0.clone()
    _call("og_channel_sum", x, P, C, scratch, out, n_out, acc)
    ref = x.double().sum(0)[:n_out] + (out0.double() if acc else 0)
    _within("og_channel_sum", out, ref, 2 * U * ref.abs() + 2.0 ** -30 * x.double().abs().sum(0)[:n_out] + 1e-45)
    out2 = out0.clone()
    _call("og_channel_sum", x, P, C, scratch, out2, n_out, acc)
    assert torch.equal(out, out2)                     # the per-CTA sums are added in a fixed order


@pytest.mark.parametrize("act", [ACT_LRELU, ACT_TANH, ACT_SIGMOID])
def test_act_backward(act):
    """Gradient through LeakyReLU / tanh / sigmoid from the saved output, saturated outputs included (tanh = +-1,
    sigmoid = 0 / 1, LeakyReLU at exactly 0).  1 - o^2 is one rounding of o * o away (<= U absolute), o (1 - o) is
    exact in its subtraction for o >= 1/2: <= 3 U |ref| + U |g|."""
    n = 4 * 70001
    g = _randn(n, seed=act)
    pre = _randn(n, seed=10 + act) * 6
    o = {ACT_LRELU: torch.where(pre > 0, pre, 0.2 * pre), ACT_TANH: torch.tanh(pre), ACT_SIGMOID: torch.sigmoid(pre)}[act]
    edge = {ACT_LRELU: [0.0, -0.0, 1e-38, -1e-38], ACT_TANH: [1.0, -1.0, 1 - U, 0.0],
            ACT_SIGMOID: [0.0, 1.0, 1 - U, 2.0 ** -126]}[act]
    o[:4] = torch.tensor(edge, device=DEV)
    o = o.float().contiguous()
    gin = torch.empty_like(g)
    _call("og_act_backward", o, g, n, act, 0.2, gin)
    o64, g64 = o.double(), g.double()
    ref = {ACT_LRELU: torch.where(o64 > 0, g64, 0.2 * g64), ACT_TANH: g64 * (1 - o64 * o64),
           ACT_SIGMOID: g64 * o64 * (1 - o64)}[act]
    _within("og_act_backward", gin, ref, 3 * U * ref.abs() + U * g64.abs() + 1e-45)


# ---------------------------------------------------------------------------------------------------
# GLU (CA_NET), reparametrisation, losses
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,Ch", [(16, 100), (3, 7), (1000, 33)])
def test_glu(P, Ch):
    """a sigmoid(b) with expf (<= 2 ulp) and an IEEE divide: <= 6 U |ref|; the gradient terms add two more roundings
    and the 1 - s cancellation (<= U absolute in s), gates at +-30 and +-100 included (exp(100) overflows: s = 0,
    where the true s is below the fp32 normal range, 2^-126)."""
    x = _randn(P, 2 * Ch, seed=Ch) * 3
    x[0, Ch:Ch + 4] = torch.tensor([30.0, -30.0, 100.0, -100.0], device=DEV)[:min(4, Ch)]
    out = torch.empty(P, Ch, device=DEV)
    _call("og_glu_fwd", x, P, Ch, out)
    a, b = x.double()[:, :Ch], x.double()[:, Ch:]
    s = torch.sigmoid(b)
    _within("og_glu_fwd", out, a * s, 6 * U * (a * s).abs() + 2.0 ** -126 * a.abs() + 1e-45)
    g = _randn(P, Ch, seed=1)
    gx = torch.empty_like(x)
    _call("og_glu_bwd", x, g, P, Ch, gx)
    g64 = g.double()
    ref = torch.cat((g64 * s, g64 * a * s * (1 - s)), 1)
    bound = torch.cat((6 * U * (g64 * s).abs(), 10 * U * (g64 * a * s).abs()), 1) + 2.0 ** -126 * (1 + a.abs().repeat(1, 2)) * g64.abs().repeat(1, 2) + 1e-45
    _within("og_glu_bwd", gx, ref, bound)


def test_reparam():
    """c = eps exp(logvar / 2) + mu with logvar up to +-80 (exp(40) ~ 2e17): expf <= 2 ulp, so <= 4 U (|eps e| + |c|);
    the backward accumulates into gx (pre-loaded) with the same exp."""
    B, D, xs, cs = 16, 100, 232, 120
    x = _randn(B, xs, seed=4)
    x[:, D:2 * D] *= 4
    x[0, D:D + 4] = torch.tensor([80.0, -80.0, 40.0, -40.0], device=DEV)
    eps = _randn(B, D, seed=5)
    c = torch.full((B, cs), 7.0, device=DEV)
    _call("og_reparam_fwd", x, xs, eps, B, D, c, cs)
    mu, lv, e64 = x.double()[:, :D], x.double()[:, D:2 * D], eps.double()
    t = e64 * torch.exp(0.5 * lv)
    _within("og_reparam_fwd", c[:, :D], t + mu, 4 * U * (t.abs() + (t + mu).abs()) + 1e-45)
    assert (c[:, D:] == 7.0).all()
    gc = _randn(B, cs, seed=6)
    gx0 = _randn(B, xs, seed=8)
    gx = gx0.clone()
    _call("og_reparam_bwd", x, xs, eps, gc, cs, B, D, gx)
    g64 = gc.double()[:, :D]
    ref = gx0.double().clone()
    ref[:, :D] += g64
    ref[:, D:2 * D] += g64 * e64 * 0.5 * torch.exp(0.5 * lv)
    bound = gx0.double().abs() * U + 1e-45
    bound[:, :D] += U * (gx0.double()[:, :D] + g64).abs()
    bound[:, D:2 * D] += 6 * U * ((g64 * e64 * 0.5 * torch.exp(0.5 * lv)).abs() + ref[:, D:2 * D].abs())
    _within("og_reparam_bwd", gx, ref, bound)


@pytest.mark.parametrize("n,target,weight", [(4001, 1.0, 1.0), (4001, 0.0, 0.5), (300, 1.0, 2.0), (7, 0.0, 1.0)])
def test_bce(n, target, weight):
    """nn.BCELoss: log terms clamped at -100, gradient (p - t) / max(p (1 - p), 1e-12), p in {0, 1, 1e-30, 1 - 2^-24}
    included.  The loss is added to the accumulator (one block: each thread sums its n / 256 terms, then two tree
    levels): <= (n / 256 + 40) U sum|terms| plus logf's ulps; the gradient is three roundings and a divide."""
    p = torch.sigmoid(_randn(n, seed=n) * 4)
    p[:4] = torch.tensor([0.0, 1.0, 1e-30, 1 - 2.0 ** -24], device=DEV)
    p = p.float().contiguous()
    loss = torch.full((1,), 1.5, device=DEV)
    gp = torch.empty_like(p)
    _call("og_bce", p, n, target, weight, loss, gp)
    p64 = p.double()
    l1 = torch.log(p64).clamp(min=-100)
    l0 = torch.log1p(-p64).clamp(min=-100)
    terms = -(target * l1 + (1 - target) * l0)
    want = 1.5 + weight * terms.mean()
    sabs = weight * terms.abs().sum().item() / n
    _within("og_bce loss", loss, want, (n / 256 + 40) * U * sabs + 4 * U * (1.5 + abs(want.item())))
    ref = weight / n * (p64 - target) / torch.clamp(p64 * (1 - p64), min=1e-12)
    _within("og_bce grad", gp, ref, 8 * U * ref.abs() + 1e-45)


def test_kl():
    """KL_loss with rows [mu | logvar] at a row stride above 2 D: the stride padding is neither read nor written."""
    B, D, xs = 16, 100, 240
    x = _randn(B, xs, seed=12)
    x[:, 2 * D:] = float("nan")                 # never read
    loss = torch.full((1,), -0.25, device=DEV)
    gx = torch.full((B, xs), 3.0, device=DEV)
    _call("og_kl", x, xs, B, D, 0.7, loss, gx)
    mu, lv = x.double()[:, :D], x.double()[:, D:2 * D]
    terms = 1 + lv - mu * mu - torch.exp(lv)
    n = B * D
    want = -0.25 - 0.5 * 0.7 * terms.mean()
    sabs = 0.5 * 0.7 * (1 + lv.abs() + mu * mu + torch.exp(lv)).sum().item() / n
    _within("og_kl loss", loss, want, (n / 256 + 40) * U * sabs + 4 * U * (0.25 + abs(want.item())))
    ref_mu = 0.7 / n * mu
    ref_lv = 0.7 / n * (-0.5) * (1 - torch.exp(lv))
    _within("og_kl grad", gx[:, :D], ref_mu, 4 * U * ref_mu.abs() + 1e-45)
    _within("og_kl grad", gx[:, D:2 * D], ref_lv, 8 * U * (ref_lv.abs() + 0.35 / n * torch.exp(lv)) + 1e-45)
    assert (gx[:, 2 * D:] == 3.0).all()


# ---------------------------------------------------------------------------------------------------
# gathers, scatters, broadcasts, copies
# ---------------------------------------------------------------------------------------------------
def test_scatter_rows_add_and_gather():
    """gx[idx[i]] += g[i] with repeated indices (fp32 atomics: <= (k - 1) U sum|terms| for k repeats); the gather is
    bitwise."""
    n_in, rowlen = 37, 48
    idx = torch.tensor([0, 5, 5, 5, 36, 0, 17, 5, 36, 2] * 13, device=DEV, dtype=torch.long)
    g = _randn(idx.numel(), rowlen, seed=13)
    gx = torch.full((n_in, rowlen), 9.0, device=DEV)
    _call("og_scatter_rows_add", g, idx, idx.numel(), n_in, rowlen, gx)
    ref = torch.zeros(n_in, rowlen, device=DEV, dtype=torch.float64).index_add_(0, idx, g.double())
    sabs = torch.zeros_like(ref).index_add_(0, idx, g.double().abs())
    k = torch.bincount(idx, minlength=n_in).double()[:, None]
    _within("og_scatter_rows_add", gx, ref, (k * U) * sabs + 1e-45)
    x = _randn(n_in, rowlen, seed=14)
    out = torch.empty(idx.numel(), rowlen, device=DEV)
    _call("og_gather_rows", x, idx, idx.numel(), rowlen, out)
    assert torch.equal(out, x[idx])


def test_broadcast_channels_and_adjoint():
    """The code vector broadcast into a channel slice of every pixel of its image (bitwise), and the adjoint: a
    sequential fp32 sum over the image's pixels, <= (pixels - 1) U sum|terms|, over several images."""
    B, Cc, cstride, off, hh = 5, 100, 232, 120, 16 * 16
    c = _randn(B, Cc, seed=15)
    dst = torch.full((B * hh, cstride), 2.0, device=DEV)
    _call("og_broadcast_channels", c, B, Cc, dst, cstride, off, hh)
    want = torch.full_like(dst, 2.0)
    want[:, off:off + Cc] = c.repeat_interleave(hh, 0)
    assert torch.equal(dst, want)
    g = _randn(B * hh, cstride, seed=16)
    gc = torch.empty(B, Cc, device=DEV)
    _call("og_broadcast_channels_bwd", g, B, Cc, cstride, off, hh, gc)
    gs = g.double()[:, off:off + Cc].reshape(B, hh, Cc)
    _within("og_broadcast_channels_bwd", gc, gs.sum(1), (hh - 1) * U * gs.abs().sum(1) + 1e-45)


def test_copy_and_permute_channels_bitwise():
    P, sstride, dstride = 1000, 52, 40
    src = _randn(P, sstride, seed=17)
    dst0 = _randn(P, dstride, seed=18)
    dst = dst0.clone()
    _call("og_copy_channels", src, sstride, 3, dst, dstride, 5, 30, P, 0)
    want = dst0.clone()
    want[:, 5:35] = src[:, 3:33]
    assert torch.equal(dst, want)
    _call("og_copy_channels", src, sstride, 3, dst, dstride, 5, 30, P, 1)
    want[:, 5:35] = want[:, 5:35] + src[:, 3:33]
    assert torch.equal(dst, want)
    for Pp in (4096, 4099):                       # float4 path and the scalar path
        B, C = 3, 80
        x = _randn(B, C, Pp, seed=Pp)
        perm = torch.stack([torch.randperm(C, device=DEV) for _ in range(B)])
        out = torch.empty_like(x)
        _call("og_permute_channels", x, perm, B, C, Pp, out)
        assert torch.equal(out, torch.gather(x, 1, perm[:, :, None].expand(B, C, Pp)))
