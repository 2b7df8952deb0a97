"""GPU tests of the tensor-core convolution path's operand handling (operands.cu, norm.cu): the exact hi/lo operand
split, the producer-side operand copies of the normalisation pass, and the refusal of a missing lo copy.  Every writer
is compared bit for bit with a numpy restatement in tests/test_gpu_operands.py; the convolutions themselves are
compared with float64 at every layer shape in tests/test_gpu_conv.py."""
import pytest
import torch
import torch.nn.functional as F

from objgan_b200 import model, ops
from objgan_b200.lib import ACT_NONE, NA_GLU, NA_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert torch.isfinite(a).all()
    return (a - b).abs().max().item() / b.abs().max().item()


def test_prep_split_exact():
    """(hi + lo) / 2^k reconstructs x to 2^-21 (relative, or 2^-38 of max|x| for tiny elements), the scale puts
    max|x| in [2^13, 2^14), the reflection halo matches F.pad, the space-to-depth blocks are the four phases."""
    x = torch.randn(2, 8, 6, 8, device=DEV) * 3
    x[0, 0, 0, 0] = 1e-7          # far below the maximum: only absolute accuracy is promised
    xn = ops.to_nhwc(x)
    hi, lo, am = ops._split(xn, 1)
    shi, slo, sam = ops._split(xn, s2d=True)
    amax = x.abs().max().item()
    assert am.view(torch.float32).item() == amax and sam.view(torch.float32).item() == amax
    import math
    k = 13 - math.floor(math.log2(amax))
    assert 2.0 ** 13 <= hi.float().abs().max().item() < 2.0 ** 14
    want = F.pad(x, (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1)

    def close(got, ref):
        tol = torch.maximum(ref.abs() * 2.0 ** -21, torch.full_like(ref, amax * 2.0 ** -38))
        return ((got - ref).abs() <= tol).all()

    rec = (hi.double() + lo.double()) * 2.0 ** -k
    assert close(rec, want.double())
    srec = (shi.double() + slo.double()) * 2.0 ** -k
    for a in range(2):
        for b in range(2):
            blk = srec[(a * 2 + b) * 2:(a * 2 + b + 1) * 2]
            assert close(blk, x[:, :, a::2, b::2].permute(0, 2, 3, 1).double())


@pytest.mark.parametrize("engine", ["f16x3"])
def test_norm_apply_emits_operand_copies(engine, monkeypatch):
    """A chain of residual blocks + upBlock with the producer-side operand split (og_norm_apply_split: the normalisation
    pass writes the next convolution's fp16 hi / lo copies, reflection halo included, scaled by an a-priori bound) against
    the same chain with separate og_norm_apply + og_prep_split passes: outputs and all gradients agree to fp32
    rounding level (the two differ only in the power of two the operands are scaled by)."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(3)
    c = 194
    blocks = torch.nn.Sequential(*[model.HmapResBlock(c) for _ in range(3)]).to(DEV)
    up = model.upBlock(c, 48).to(DEV)
    model._chain_res_blocks(blocks, 0)
    x0 = torch.randn(2, 32, 32, ops.cpad(c), device=DEV)
    x0[..., c:] = 0

    def unfused(x):          # the blocks' own forward without split_pad: og_norm_apply, then the conv's og_prep_split
        for blk in blocks:
            y = ops.instance_norm_act(blk.block[1](x), NA_GLU)
            x = ops.instance_norm_act(blk.block[5](y), NA_NONE, res=x)
        return up(x)

    res = {}
    for fused in (False, True, False):     # the first pass also packs the weights: only the last two are compared / counted
        calls0 = ops._lib.get().launches
        x = x0.clone().requires_grad_(True)
        for p_ in list(blocks.parameters()) + list(up.parameters()):
            p_.grad = None
        out = up(blocks(x)) if fused else unfused(x)
        gout = torch.ones_like(out) * torch.linspace(-1, 1, out.shape[-1], device=DEV)
        out.backward(gout)
        res[fused] = (out.detach().clone(), x.grad.clone(), [p_.grad.clone() for p_ in blocks.parameters()],
                      ops._lib.get().launches - calls0)
    tol = 1e-5
    assert _rel(res[True][0], res[False][0]) <= tol
    assert _rel(res[True][1], res[False][1]) <= 10 * tol
    for a, b in zip(res[True][2], res[False][2]):
        assert _rel(a, b) <= 10 * tol


def test_null_lo_copy_is_refused():
    """Every entry point that writes or reads an fp16 hi / lo operand pair returns an error for a null pointer in the
    pair (checked before any work is issued): the same call with both copies succeeds."""
    import ctypes
    torch.manual_seed(5)
    n, h, w, c = 1, 16, 16, 8
    x = torch.randn(n, h, w, c, device=DEV)
    word = lambda: torch.empty(1, device=DEV, dtype=torch.int32)
    half = lambda shape: ops._empty_slack(shape, DEV)
    wt = torch.randn(c, c, 3, 3, device=DEV)
    aw = word()
    ops._call("og_amax", ops._p(wt), wt.numel(), ops._p(aw))
    mean, rstd = torch.zeros(n * c, device=DEV), torch.ones(n * c, device=DEV)
    bound = word()
    ops._call("og_norm_bound", 0, 0, 0, h * w, 0, ops._p(bound))
    xs, gs = ops._split(x, 0), ops._split(torch.randn(n, h, w, c, device=DEV), 0)
    wh, wl = half((9, c, c)), half((9, c, c))
    ops._call("og_pack_weights_f16", ops._p(wt), c, c, 3, 3, c, c, 0, 0, 1, ops._p(aw), ops._p(wh), ops._p(wl))
    y = torch.empty(n, h, w, c, device=DEV)
    taps = ops._int_array([(i - 1, j - 1, 0, i * 3 + j) for i in range(3) for j in range(3)])
    ents = ops._int_array([(0, i - 1, j - 1, 0, i * 3 + j) for i in range(3) for j in range(3)])
    dw = torch.empty(9 * c * c, device=DEV)

    calls = {   # name -> call with the lo pointer(s) given
        "og_prep_split": lambda lo: ops._call("og_prep_split", ops._p(x), n, h, w, c, 1, 0, ops._p(word()), 0,
                                              ops._p(half((n, h + 2, w + 2, c))), lo(half((n, h + 2, w + 2, c)))),
        "og_prep_split_s2d": lambda lo: ops._call("og_prep_split_s2d", ops._p(x), n, h, w, c, ops._p(word()), 0,
                                                  ops._p(half((4 * n, h // 2, w // 2, c))),
                                                  lo(half((4 * n, h // 2, w // 2, c)))),
        "og_norm_apply_split": lambda lo: ops._call(
            "og_norm_apply_split", ops._p(x), n, h, w, c, 1, ops._p(mean), ops._p(rstd), 0, 0, 0, NA_NONE, 0.2, 0,
            ops._p(bound), 1, ops._p(half((n, h + 2, w + 2, c))), lo(half((n, h + 2, w + 2, c)))),
        "og_pack_weights_f16": lambda lo: ops._call("og_pack_weights_f16", ops._p(wt), c, c, 3, 3, c, c, 0, 0, 1,
                                                    ops._p(aw), ops._p(half((9, c, c))), lo(half((9, c, c)))),
        "og_pack_upsample_weights": lambda lo: ops._call(
            "og_pack_upsample_weights", ops._p(wt), c, c, c, c, 0, 0, 1, ops._p(aw), ops._p(word()),
            ops._p(half((16, c, c))), lo(half((16, c, c)))),
    }
    for name, lo_x, lo_w in (("og_conv2d_tc x", True, False), ("og_conv2d_tc w", False, True)):
        calls[name] = lambda lo, lo_x=lo_x, lo_w=lo_w: ops._call(
            "og_conv2d_tc", ops._p(xs[0]), lo(xs[1]) if lo_x else ops._p(xs[1]), ops._p(xs[2]), n, n, h, w, c,
            ops._p(wh), lo(wl) if lo_w else ops._p(wl), ops._p(aw), 9, c, ops._p(y), h, w, c, h * w * c, w * c, c,
            h, w, 1, 1, 0, 0, ctypes.addressof(taps), 9, 0, ACT_NONE, 0.2)
    for name, lo_g, lo_x in (("og_conv2d_wgrad_tc g", True, False), ("og_conv2d_wgrad_tc x", False, True)):
        calls[name] = lambda lo, lo_g=lo_g, lo_x=lo_x: ops._call(
            "og_conv2d_wgrad_tc", ops._p(gs[0]), lo(gs[1]) if lo_g else ops._p(gs[1]), ops._p(gs[2]), n, n, h, w, c,
            ops._p(xs[0]), lo(xs[1]) if lo_x else ops._p(xs[1]), ops._p(xs[2]), n, h, w, c, ops._p(dw), 9,
            ctypes.addressof(ents), 9)
    for name, call in calls.items():
        call(ops._p)
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError):
            call(lambda t: 0)
    torch.cuda.synchronize()
