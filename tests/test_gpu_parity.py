"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerance (north_star): 1e-3 relative fp32, measured as max|delta| / max|reference| per tensor; ROI index
math bit-exact.  End-to-end *gradients* through the whole G+D stack are compared at 1e-2 because the reference
itself only reproduces them to ~4e-3 when its summation order changes (8 vs 1 CPU threads, see DESIGN.md
"Parity budget"); every individual operator is held to 1e-3 (and typically lands at 1e-5..1e-6).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import reference_fixtures as fixtures
from objgan_b200 import lib, model, ops, synth, trainer
from objgan_b200.config import cfg
from objgan_b200.lib import (ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, NA_GLU, NA_LRELU, NA_NONE, PAD_REFLECT,
                             PAD_ZERO, UPSAMPLE2X)
from oracle import objgan_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-3
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


def close(a, b, tol=TOL, what=""):
    r = rel(a, b)
    assert r <= tol, (what, r)


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def close_grad(a, b, what="", l2=5e-3, mx=3e-2):
    """Network-level gradients: LeakyReLU / max sign flips on near-zero pre-activations and tiny-batch BatchNorm make
    a handful of entries jump when the summation order changes (the reference does this to itself, DESIGN.md
    "Parity budget"), so these are judged in the L2 norm (5e-3) with a loose max-norm guard (3e-2)."""
    assert rel_l2(a, b) <= l2, (what, "l2", rel_l2(a, b))
    assert rel(a, b) <= mx, (what, "max", rel(a, b))


def nhwc(x):  # NCHW cpu -> NHWC(+pad) cuda
    return ops.to_nhwc(x.to(DEV))


# ---------------------------------------------------------------------------------------------------
# convolution: every addressing mode / stride / kernel the networks use, forward + both gradients
# ---------------------------------------------------------------------------------------------------
CONV_CASES = [
    # cin, cout, k, stride, pad, mode, bias, act, split, H
    (194, 388, 3, 1, 1, PAD_REFLECT, False, ACT_NONE, 194, 12),   # HmapResBlock conv1
    (194, 194, 3, 1, 1, PAD_REFLECT, False, ACT_NONE, 0, 9),      # HmapResBlock conv2
    (194, 96, 3, 1, 1, UPSAMPLE2X, False, ACT_NONE, 48, 7),       # upBlock
    (80, 24, 3, 1, 1, PAD_REFLECT, True, ACT_NONE, 0, 10),        # G_HMAP conv3x3 (+bias)
    (24, 48, 3, 2, 1, PAD_ZERO, False, ACT_LRELU, 0, 10),         # G_HMAP downsample
    (48, 3, 3, 1, 1, PAD_ZERO, False, ACT_TANH, 0, 11),           # GET_IMAGE_G
    (3, 96, 4, 2, 1, PAD_ZERO, False, ACT_LRELU, 0, 16),          # D first layer
    (96, 192, 4, 2, 1, PAD_ZERO, False, ACT_NONE, 0, 8),          # D inner layer
    (64, 1, 4, 2, 0, PAD_ZERO, True, ACT_SIGMOID, 0, 8),          # outlogits (k4 s2 p0 + bias + sigmoid)
    (40, 16, 3, 1, 1, PAD_ZERO, False, ACT_NONE, 0, 5),           # jointConv-like 3x3 zero pad
]


def _ref_conv(x, w, b, k, stride, pad, mode, act):
    if mode == PAD_REFLECT:
        x = F.pad(x, (1, 1, 1, 1), mode="reflect")
        y = F.conv2d(x, w, b, stride, 0)
    elif mode == UPSAMPLE2X:
        y = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, 1, pad)
    else:
        y = F.conv2d(x, w, b, stride, pad)
    if act == ACT_LRELU:
        y = F.leaky_relu(y, 0.2)
    elif act == ACT_TANH:
        y = torch.tanh(y)
    elif act == ACT_SIGMOID:
        y = torch.sigmoid(y)
    return y


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd_bwd(case):
    cin, cout, k, stride, pad, mode, bias, act, split, H = case
    torch.manual_seed(hash(case) % 1000)
    m = model.Conv2dP(cin, cout, k, stride, pad, bias=bias, mode=mode, act=act, split=split).to(DEV)
    x = torch.randn(3, cin, H, H + 1)
    w = m.weight.detach().cpu().clone().requires_grad_(True)
    b = m.bias.detach().cpu().clone().requires_grad_(True) if bias else None
    xr = x.clone().requires_grad_(True)
    yr = _ref_conv(xr, w, b, k, stride, pad, mode, act)
    gy = torch.randn_like(yr)
    yr.backward(gy)
    xg = x.to(DEV).requires_grad_(True)
    y_nhwc = m(ops.to_nhwc(xg))
    if split:  # GLU halves are each padded: compare half by half
        sp = ops.cpad(split)
        y = torch.cat((y_nhwc[..., :split], y_nhwc[..., sp:sp + split]), -1).permute(0, 3, 1, 2)
        assert (y_nhwc[..., split:sp] == 0).all() and (y_nhwc[..., sp + split:] == 0).all()
        gfull = torch.zeros_like(y_nhwc)
        g_nhwc = gy.permute(0, 2, 3, 1).to(DEV)
        gfull[..., :split] = g_nhwc[..., :split]
        gfull[..., sp:sp + split] = g_nhwc[..., split:]
        close(y, yr, what="fwd")
        y_nhwc.backward(gfull)
    else:
        y = ops.to_nchw(y_nhwc, cout)
        close(y, yr, what="fwd")
        y.backward(gy.to(DEV))
    close(xg.grad, xr.grad, what="dgrad")
    close(m.weight.grad, w.grad, what="wgrad")
    if bias:
        close(m.bias.grad, b.grad, what="bgrad")


def test_linear_and_batchnorm1d_glu():
    torch.manual_seed(1)
    st = model.INIT_STAGE_G(48 * 4, 100).to(DEV)
    sd = {k: v.detach().cpu().clone() for k, v in st.state_dict().items()}
    z, c = torch.randn(4, 100), torch.randn(4, 100)
    keys = O.trainable_keys(sd)
    live, leaves = O._with_grad(sd, keys)
    # oracle uses prefix-based keys; wrap with a leading dummy prefix
    pre = {"p." + k: v for k, v in live.items()}
    yr = O.init_stage_g(z, c, pre, "p", True)
    gy = torch.randn_like(yr)
    grads = torch.autograd.grad(yr, [leaves[k] for k in keys], gy)
    y = st(z.to(DEV), c.to(DEV))
    close(y, yr, what="fwd")
    y.backward(gy.to(DEV))
    params = dict(st.named_parameters())
    for k, g in zip(keys, grads):
        close_grad(params[k].grad, g, what=k)
    sd2 = st.state_dict()
    for k in sd2:
        if "running" in k or "num_batches" in k:
            close(sd2[k].float(), pre["p." + k].float(), 1e-4, what=k)


@pytest.mark.parametrize("act", [NA_GLU, NA_LRELU, NA_NONE])
@pytest.mark.parametrize("instance", [True, False])
def test_norm_act(act, instance):
    torch.manual_seed(5)
    n, c, h, w = 3, 16, 9, 7
    x = (torch.randn(n, c, h, w) * 2 + 0.7).requires_grad_(True)
    res = torch.randn(n, c, h, w) if act == NA_NONE else None
    if instance:
        yn = F.instance_norm(x, eps=1e-5)
        gamma = beta = None
    else:
        gamma = torch.randn(c).requires_grad_(True)
        beta = torch.randn(c).requires_grad_(True)
        rm, rv = torch.zeros(c), torch.ones(c)
        yn = F.batch_norm(x, rm, rv, gamma, beta, True, 0.1, 1e-5)
    if act == NA_GLU:
        yr = O.glu(yn)
    elif act == NA_LRELU:
        yr = F.leaky_relu(yn, 0.2)
    else:
        yr = yn + res
    gy = torch.randn_like(yr)
    yr.backward(gy)
    xg = x.detach().to(DEV).requires_grad_(True)
    xn = ops.to_nhwc(xg)
    if instance:
        out = ops.instance_norm_act(xn, act, res=None if res is None else nhwc(res))
    else:
        gg = gamma.detach().to(DEV).requires_grad_(True)
        bb = beta.detach().to(DEV).requires_grad_(True)
        bufs = (torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros((), dtype=torch.long, device=DEV))
        out = ops._NormAct.apply(xn, gg, bb, None if res is None else nhwc(res), bufs, False, act)
    y = ops.to_nchw(out, yr.shape[1])
    close(y, yr, what="fwd")
    y.backward(gy.to(DEV))
    close(xg.grad, x.grad, what="dx")
    if not instance:
        close(gg.grad, gamma.grad, what="dgamma")
        close(bb.grad, beta.grad, what="dbeta")
        close(bufs[0], rm, 1e-5)
        close(bufs[1], rv, 1e-5)
        assert int(bufs[2]) == 1


# ---------------------------------------------------------------------------------------------------
# attention / paint
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,ih,L", [(3, 8, 18), (2, 16, 12), (5, 10, 18)])
def test_att_general(B, ih, L):
    torch.manual_seed(7)
    att = model.ATT_NET(48, 256).to(DEV)
    h = torch.randn(B, 48, ih, ih, requires_grad=True)
    words = torch.randn(B, 256, L, requires_grad=True)
    lens = torch.randint(3, L + 1, (B,))
    lens[0] = L
    mask = torch.arange(L).view(1, L) >= lens.view(B, 1)
    w = att.conv_context.weight.detach().cpu().clone().requires_grad_(True)
    wc_r, a_r = O.global_attention_general(h, words, w, mask)
    g = torch.randn_like(wc_r)
    wc_r.backward(g)
    att.applyMask(mask.to(DEV))
    hg = h.detach().to(DEV).requires_grad_(True)
    wg = words.detach().to(DEV).requires_grad_(True)
    wc, a = att(hg, wg)
    close(wc, wc_r, what="wc")
    close(a, a_r, what="attn")
    wc.backward(g.to(DEV))
    close(hg.grad, h.grad, what="g_h")
    close(att.conv_context.weight.grad, w.grad, what="g_W")
    close(wg.grad, words.grad, what="g_words")


def test_bu_att_and_paint():
    torch.manual_seed(8)
    B, R, L = 4, 7, 18
    bu = model.BT_ATT_NET(48, 256).to(DEV)
    lab, glove, words = torch.randn(B, 50, R, 1), torch.randn(B, 50, L), torch.randn(B, 256, L)
    lab[1, :, 4:] = 0  # padded roi slots
    lens = torch.tensor([18, 11, 9, 5])
    mask = torch.arange(L).view(1, L) >= lens.view(B, 1)
    w = bu.conv_context.weight.detach().cpu().clone().requires_grad_(True)
    wc_r, a_r = O.global_bu_attention(lab, glove, words, w, mask)
    m = torch.rand(B, R, 12, 12)
    m[m < 0.6] = 0
    painted_r = O.pprocess_bt_attns(wc_r, m)
    g = torch.randn_like(painted_r)
    painted_r.backward(g)
    bu.applyMask(mask.to(DEV))
    wc, a = bu(lab.to(DEV), glove.to(DEV), words.to(DEV))
    close(wc, wc_r, what="wc")
    close(a, a_r, what="attn")
    painted = model.pprocess_bt_attns(wc, 12, 12, m.to(DEV))
    close(painted, painted_r, what="paint")
    painted.backward(g.to(DEV))
    close(bu.conv_context.weight.grad, w.grad, what="g_W")
    # the reference's expanded 5-D mask form gives the same result
    p2 = model.pprocess_bt_attns(wc.detach(), 12, 12, m.to(DEV).unsqueeze(2).repeat(1, 1, 48, 1, 1))
    close(p2, painted_r)


def test_func_attention():
    torch.manual_seed(9)
    q, ctx = torch.randn(6, 256, 15, requires_grad=True), torch.randn(6, 256, 17, 17, requires_grad=True)
    w_r, a_r = O.func_attention(q, ctx, 4.0)
    gw, ga = torch.randn_like(w_r), torch.randn_like(a_r)
    (w_r * gw).sum().add((a_r * ga).sum()).backward()
    qg, cg = q.detach().to(DEV).requires_grad_(True), ctx.detach().to(DEV).requires_grad_(True)
    w, a = ops.func_attention(qg, cg, 4.0)
    close(w, w_r)
    close(a, a_r)
    (w * gw.to(DEV)).sum().add((a * ga.to(DEV)).sum()).backward()
    close(qg.grad, q.grad, what="g_query")
    close(cg.grad, ctx.grad, what="g_context")


# ---------------------------------------------------------------------------------------------------
# ROIAlign
# ---------------------------------------------------------------------------------------------------
def _rois(B, n_per, size, seed):
    rng = np.random.RandomState(seed)
    xy = rng.uniform(-4, size * 16 * 0.9, (B * n_per, 2))
    wh = rng.uniform(1, size * 8, (B * n_per, 2))
    idx = np.repeat(np.arange(B), n_per).reshape(-1, 1)
    return np.hstack((idx, xy, xy + wh)).astype(np.float32)


def test_roi_align_bit_exact_vs_oracle():
    feat = torch.randn(2, 6, 16, 16)
    rois = _rois(2, 5, 16, 3)
    rois[0, 1:] = [0, 0, 0, 0]                      # degenerate (the reference pools all 10 slots, valid or not)
    rois[1, 1:] = [300, 300, 400, 400]              # fully outside -> zeros
    want = O.roi_align_forward_np(feat.numpy(), rois, 6, 6, 1.0 / 16)
    got = ops.roi_align(feat.to(DEV), torch.from_numpy(rois).to(DEV), 6, 6, 1.0 / 16).cpu().numpy()
    # Bit-exactness is defined against the reference .cu built for sm_90a (next test).  Against the CPU
    # restatement, nvcc's FMA contraction of "ph * bin + start" (which the reference .cu gets too) moves a sample
    # coordinate by <= 1 ulp, i.e. the interpolated value by ~1e-6: compare with that tolerance here ...
    assert np.array_equal(got == 0, want == 0)
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-5)
    # ... and exactly on rois whose arithmetic is exactly representable (dyadic grid):
    # dyadic rois: every intermediate is exactly representable -> bit-exact equality
    rois_d = np.array([[0, 0, 0, 79, 79], [1, 16, 32, 95, 111], [1, 64, 64, 143, 143]], dtype=np.float32)
    want = O.roi_align_forward_np(feat.numpy(), rois_d, 6, 6, 1.0 / 16)
    got = ops.roi_align(feat.to(DEV), torch.from_numpy(rois_d).to(DEV), 6, 6, 1.0 / 16).cpu().numpy()
    assert np.array_equal(got, want)


def _ref_cu():
    """The reference's roi_align_kernel.cu compiled verbatim by oracle/Makefile (present where the fixtures are
    recorded)."""
    import ctypes
    import os
    ref = ctypes.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                                   "libroi_align_ref_cuda.so"))
    vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    ref.ROIAlignForwardLaucher.argtypes = [vp, cf, ci, ci, ci, ci, ci, ci, vp, vp, vp]
    ref.ROIAlignBackwardLaucher.argtypes = [vp, cf, ci, ci, ci, ci, ci, ci, ci, vp, vp, vp]
    return ref


ROI_CAP = 4096


def test_roi_align_bit_exact_vs_reference_cu():
    """Bit-for-bit against the reference's roi_align_kernel.cu compiled verbatim for sm_90a (its outputs on these
    seeded inputs are stored in tests/golden/reference, a fixed sample of ROI_CAP elements per tensor)."""
    g = torch.Generator().manual_seed(2)
    for (B, C, H, n_per, AH) in [(4, 24, 64, 10, 6), (3, 16, 32, 10, 6), (2, 8, 16, 7, 7)]:
        feat = torch.randn(B, C, H, H, generator=g).to(DEV)
        rois = torch.from_numpy(_rois(B, n_per, H, B + C)).to(DEV)
        R = rois.shape[0]
        gout = torch.randn(R, C, AH, AH, generator=g).to(DEV)

        def produce():
            ref = _ref_cu()
            want = torch.zeros(R, C, AH, AH, device=DEV)
            stream = torch.cuda.current_stream().cuda_stream
            assert ref.ROIAlignForwardLaucher(feat.data_ptr(), 1.0 / 16, R, H, H, C, AH, AH, rois.data_ptr(),
                                              want.data_ptr(), stream) == 1
            wg = torch.zeros_like(feat)
            assert ref.ROIAlignBackwardLaucher(gout.data_ptr(), 1.0 / 16, B, R, H, H, C, AH, AH, rois.data_ptr(),
                                               wg.data_ptr(), stream) == 1
            torch.cuda.synchronize()
            return {"fwd": want, "bwd": wg}
        want = fixtures.recorded(f"roi_align_cu_{B}_{C}_{H}_{AH}", produce, ROI_CAP)
        got = ops.roi_align(feat, rois, AH, AH, 1.0 / 16)
        torch.cuda.synchronize()
        got_s = torch.from_numpy(fixtures.sample(got, ROI_CAP))
        assert torch.equal(got_s, want["fwd"]), (got_s - want["fwd"]).abs().max().item()
        # backward: same per-element products; atomicAdd order is free in both, so compare with a tolerance
        fg = feat.clone().requires_grad_(True)
        ops.roi_align(fg, rois, AH, AH, 1.0 / 16).backward(gout)
        torch.cuda.synchronize()
        close(torch.from_numpy(fixtures.sample(fg.grad, ROI_CAP)), want["bwd"], 1e-5, what="roi bwd vs reference .cu")


def test_roi_align_avg_and_backward():
    torch.manual_seed(3)
    feat = torch.randn(3, 8, 32, 32)
    rois = _rois(3, 10, 32, 5)
    want = O.roi_align_avg_np(feat.numpy(), rois, 5, 5, 1.0 / 16)
    fg = feat.to(DEV).requires_grad_(True)
    got = model.RoIAlignAvg(5, 5, 1.0 / 16)(fg, torch.from_numpy(rois).to(DEV))
    close(got, torch.from_numpy(want), 1e-6, what="avg fwd")
    g = torch.randn(got.shape)
    got.backward(g.to(DEV))
    # adjoint: avg-pool backward then roi-align backward (oracle accumulates in float64)
    g6 = torch.zeros(rois.shape[0], 8, 6, 6)
    for dh in (0, 1):
        for dw in (0, 1):
            g6[:, :, dh:dh + 5, dw:dw + 5] += g / 4
    want_g = O.roi_align_backward_np(g6.numpy(), rois, feat.shape, 6, 6, 1.0 / 16)
    close(fg.grad, torch.from_numpy(want_g), 1e-5, what="avg bwd")
    # plain op backward through the reference-named launcher
    fg2 = feat.to(DEV).requires_grad_(True)
    out = ops.roi_align(fg2, torch.from_numpy(rois).to(DEV), 6, 6, 1.0 / 16)
    out.backward(g6.to(DEV))
    close(fg2.grad, torch.from_numpy(want_g), 1e-5, what="bwd")


def test_torch_extension_roi_align_matches_c_abi():
    """torch.ops.objgan_b200.roi_align_forward_cuda / backward_cuda (TORCH_LIBRARY layer) and the RoIAlignFunction that
    replaces the reference's functions/roi_align.py give the bits of the ctypes path (same launchers underneath)."""
    from objgan_b200.torch_ext import RoIAlignFunction, roi_align
    torch.manual_seed(4)
    feat = torch.randn(3, 16, 32, 32, device=DEV)
    rois = torch.from_numpy(_rois(3, 10, 32, 11)).to(DEV)
    want = ops.roi_align(feat, rois, 6, 6, 1.0 / 16)
    out = feat.new_zeros(rois.size(0), 16, 6, 6)
    assert roi_align.roi_align_forward_cuda(6, 6, 1.0 / 16, feat, rois, out) == 1
    assert torch.equal(out, want)
    fg = feat.clone().requires_grad_(True)
    y = RoIAlignFunction(6, 6, 1.0 / 16)(fg, rois)
    assert torch.equal(y, want)
    g = torch.randn_like(y)
    y.backward(g)
    fg2 = feat.clone().requires_grad_(True)
    ops.roi_align(fg2, rois, 6, 6, 1.0 / 16).backward(g)
    close(fg.grad, fg2.grad, 1e-5, what="grad through the extension")     # atomics: order differs run to run
    with pytest.raises(RuntimeError):
        roi_align.roi_align_forward_cuda(6, 6, 1.0 / 16, feat, rois[:, :4].contiguous(), out)


@pytest.mark.parametrize("B,C,H", [(3, 8, 32), (32, 384, 64), (4, 768, 32)])
def test_roi_align_avg_channels_last_is_bit_identical(B, C, H):
    """The channels-last fused RoIAlignAvg (what the object discriminators run) returns exactly the bits of the NCHW
    reference-ABI path (itself bit-identical to the reference .cu, tests above); its adjoint matches the float64 oracle."""
    torch.manual_seed(31 + C)
    feat = torch.randn(B, C, H, H)
    rois = _rois(B, 10, H, 5 + C)
    rd = torch.from_numpy(rois).to(DEV)
    want = model.RoIAlignAvg(5, 5, 1.0 / 16)(feat.to(DEV), rd)
    fg = feat.to(DEV).permute(0, 2, 3, 1).contiguous().requires_grad_(True)
    got = ops.roi_align_avg_nhwc(fg, rd, 5, 5, 1.0 / 16)
    assert torch.equal(got.permute(0, 3, 1, 2), want)
    g = torch.randn(want.shape)
    got.backward(g.to(DEV).permute(0, 2, 3, 1).contiguous())
    g6 = torch.zeros(rois.shape[0], C, 6, 6)
    for dh in (0, 1):
        for dw in (0, 1):
            g6[:, :, dh:dh + 5, dw:dw + 5] += g / 4
    want_g = O.roi_align_backward_np(g6.numpy(), rois, feat.shape, 6, 6, 1.0 / 16)
    close(fg.grad.permute(0, 3, 1, 2), torch.from_numpy(want_g), 2e-5, what="nhwc avg bwd")


# ---------------------------------------------------------------------------------------------------
# whole networks and the training step
# ---------------------------------------------------------------------------------------------------
def _cpu_sd(m):
    return {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}


def test_g_net_forward_parity():
    torch.manual_seed(11)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    g.to(DEV)
    sd = _cpu_sd(g)
    inp = synth.make_inputs(3, seed=5, parity=True)
    with torch.no_grad():
        ref = O.g_net_forward(sd, inp)
    d = {k: (v.to(DEV) if torch.is_tensor(v) else [t.to(DEV) for t in v] if isinstance(v, list) else v)
         for k, v in inp.items()}
    g.ca_net.eps_override = d["eps"]
    with torch.no_grad():
        out = g(d["z"], d["sent_emb"], d["words_embs"], d["glove_words_embs"], d["slabels_feat"], d["mask"],
                d["hmaps"], d["rois"], d["fm_rois"], d["num_rois"], d["bt_masks"], d["fm_bt_masks"],
                d["glb_max_num_roi"])
    for i in range(3):
        close(out[0][i], ref[0][i], what=f"fake{i}")
    for i in range(2):
        close(out[1][i], ref[1][i], what=f"bt_c{i}")
        close(out[2][i], ref[2][i], what=f"att{i}")
        close(out[3][i], ref[3][i], what=f"bt_att{i}")
    close(out[4], ref[4], what="mu")
    close(out[5], ref[5], what="logvar")
    sd2 = _cpu_sd(g)
    for k in sd:
        if "running" in k:
            close(sd2[k], sd[k], 1e-4, what=k)   # oracle updated sd in place
        if "num_batches" in k:
            assert int(sd2[k]) == int(sd[k]) == 1


def test_g_net_forward_without_boxes():
    """A batch in which no image has a box (max(num_rois) == 0; likely with small per-GPU batches): the bottom-up
    branch contributes zeros (ref: model.py:689-694) -- no kernel may read the empty roi axis."""
    torch.manual_seed(17)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    g.to(DEV)
    sd = _cpu_sd(g)
    inp = synth.make_inputs(2, seed=9, parity=True)
    inp["num_rois"] = torch.zeros_like(inp["num_rois"])
    inp["glb_max_num_roi"] = 0
    inp["slabels_feat"] = inp["slabels_feat"][:, :, :0]
    inp["bt_masks"] = [torch.zeros_like(m) for m in inp["bt_masks"]]
    inp["fm_bt_masks"] = torch.zeros_like(inp["fm_bt_masks"])
    with torch.no_grad():
        ref = O.g_net_forward(sd, inp)
    d = {k: (v.to(DEV) if torch.is_tensor(v) else [t.to(DEV) for t in v] if isinstance(v, list) else v)
         for k, v in inp.items()}
    g.ca_net.eps_override = d["eps"]
    out = g(d["z"], d["sent_emb"], d["words_embs"], d["glove_words_embs"], d["slabels_feat"], d["mask"],
            d["hmaps"], d["rois"], d["fm_rois"], d["num_rois"], d["bt_masks"], d["fm_bt_masks"], 0)
    for i in range(3):
        close(out[0][i], ref[0][i], what=f"fake{i}")
    for i in range(2):
        assert out[1][i].shape == ref[1][i].shape and out[1][i].numel() == 0
        close(out[2][i], ref[2][i], what=f"att{i}")
        assert float(out[3][i].abs().max()) == 0.0 and out[3][i].shape == ref[3][i].shape
    sum(o.sum() for o in out[0]).backward()          # the backward pass must not touch the empty roi axis either
    assert all(torch.isfinite(p.grad).all() for p in g.parameters() if p.grad is not None)


@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
def test_pat_d_loss_parity(engine, l2, mx, monkeypatch):
    """simt = exact fp32 contractions (strict); f16x3 = tensor cores, whose ~1e-5 per-conv rounding is amplified by
    the LeakyReLU / BatchNorm(B=4) chain like any other perturbation (DESIGN.md "Parity budget")."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(12)
    d = model.PAT_D_NET128()
    d.apply(model.weights_init)
    d.to(DEV)
    sd = _cpu_sd(d)
    real, fake, cond = torch.rand(4, 3, 128, 128) * 2 - 1, torch.rand(4, 3, 128, 128) * 2 - 1, torch.rand(4, 256)
    keys = O.trainable_keys(sd)
    live, leaves = O._with_grad(sd, keys)
    err_r = O.pat_d_loss(live, real, fake, cond)
    grads = torch.autograd.grad(err_r, [leaves[k] for k in keys])
    from objgan_b200 import losses
    err = losses.patD_loss(d, real.to(DEV), fake.to(DEV), cond.to(DEV))
    close(err, err_r.detach(), 1e-4, what="errD")
    err.backward()
    params = dict(d.named_parameters())
    for k, g in zip(keys, grads):
        close_grad(params[k].grad, g, what=k, l2=l2, mx=mx)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_cond_head_small_batches(n):
    """D_GET_LOGITS (jointConv + BatchNorm + LeakyReLU + logits conv) on n = 1, 2, 3 samples: patD_loss runs the COND
    head on B - 1 "wrong pair" samples, which is a single sample at per-GPU batch 2."""
    torch.manual_seed(40 + n)
    d = model.PAT_D_NET128()
    d.apply(model.weights_init)
    d.to(DEV)
    sd = _cpu_sd(d)
    h = torch.randn(n, 768, 8, 8) * 0.5
    c = torch.rand(n, 256)
    keys = [k for k in O.trainable_keys(sd) if k.startswith("COND_DNET")]
    live, leaves = O._with_grad(sd, keys)
    hr = h.clone().requires_grad_(True)
    loss_r = O.bce(O.d_get_logits(hr, live, "COND_DNET", c), 0)
    grads = torch.autograd.grad(loss_r, [hr] + [leaves[k] for k in keys])
    hg = h.to(DEV).requires_grad_(True)
    loss = ops.bce(d.COND_DNET(hg, c.to(DEV)), 0.0, 1.0)
    close(loss, loss_r.detach(), 1e-5, what="loss")
    loss.backward()
    close_grad(hg.grad, grads[0], what="g_h")
    params = dict(d.named_parameters())
    for k, g in zip(keys, grads[1:]):
        close_grad(params[k].grad, g, what=k)


def test_adam_ema_kernel():
    torch.manual_seed(13)
    n = 10007
    p, m, v, avg = torch.randn(n), torch.zeros(n), torch.zeros(n), None
    pg, mg, vg = p.to(DEV), m.to(DEV), v.to(DEV)
    avg = p.clone()
    ag = avg.to(DEV)
    for t in range(1, 5):
        g = torch.randn(n)
        O.adam_step(p, g, m, v, t)
        O.ema_update(avg, p)
        ops.adam_ema_(pg, g.to(DEV), mg, vg, ag, t)
        assert ((pg.cpu() - p).abs() / p.abs().clamp(min=1.0)).max().item() < 1e-6
        assert ((ag.cpu() - avg).abs() / avg.abs().clamp(min=1.0)).max().item() < 1e-6


@pytest.mark.parametrize("engine,cos_min,l2_max", [("simt", 0.9999, 5e-2), ("f16x3", 0.999, 0.2)])
def test_step_a_parity(engine, cos_min, l2_max, monkeypatch):
    """One full Step-A step (B=4, ragged captions / roi counts) against oracle.step_a.

    engine "simt": every contraction in exact fp32 FMA arithmetic -- the strict end-to-end check.
    engine "f16x3": the tensor-core path (3xFP16, ~5x fp32 rounding per product).  Forward images, losses and
    the optimiser update are held to the same bounds; the end-to-end gradient direction is held to cos > 0.999
    because the G -> D -> BCE chain amplifies rounding by ~1e4 through LeakyReLU / max / BatchNorm sign flips
    (the reference moves its own gradients by ~1e-2 when only its thread count changes; DESIGN.md "Parity budget")."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    B = 4
    t = trainer.StepATrainer(device=DEV, seed=21)
    state = O.StepAState(_cpu_sd(t.netG), [_cpu_sd(d) for d in t.netsPatD])
    inp = synth.make_inputs(B, seed=33, parity=True)
    keep = {}
    losses_ref = O.step_a(state, inp, keep=keep)
    p0 = {k: v.detach().cpu().clone() for k, v in t.netG.named_parameters()}
    out = t.step(t.to_device(inp))
    for i in range(3):
        close(out["fake_imgs"][i], keep["fake"][i], what=f"fake{i}")
        assert abs(float(out[f"errPatD{i}"]) - losses_ref[f"errPatD{i}"]) < 1e-4 * max(1, abs(losses_ref[f"errPatD{i}"]))
    assert abs(float(out["errG"]) - losses_ref["errG"]) < 1e-3 * abs(losses_ref["errG"])
    assert abs(float(out["kl"]) - losses_ref["kl"]) < 1e-4 * max(1e-3, abs(losses_ref["kl"]))
    # G gradients (the bucket still holds them): direction + per-tensor L2 (see close_grad / module docstring)
    gparams = dict(t.netG.named_parameters())
    keys = [k for k in state.g_keys if not k.endswith("conv3x3.1.bias")]  # bias ahead of InstanceNorm: true grad is 0
    dot = sum((gparams[k].grad.cpu().double() * keep["g_grads"][k].double()).sum() for k in keys)
    na = sum((gparams[k].grad.cpu().double() ** 2).sum() for k in keys).sqrt()
    nb = sum((keep["g_grads"][k].double() ** 2).sum() for k in keys).sqrt()
    assert float(dot / (na * nb)) > cos_min, float(dot / (na * nb))
    worst = max(rel_l2(gparams[k].grad, keep["g_grads"][k]) for k in keys)
    assert worst < l2_max, worst
    # D parameters after their Adam step, G parameters + EMA after theirs (where the gradient is above noise)
    for i, d in enumerate(t.netsPatD):
        dp = dict(d.named_parameters())
        for k in state.d_keys[i]:
            gr = keep["d_grads"][i][k]
            sel = gr.abs() > 0.2 * gr.abs().max()  # first Adam step is sign descent: only clear-signed entries
            assert ((dp[k].detach().cpu() - state.ds[i][k])[sel]).abs().max().item() < 5e-5, (i, k)
        sd = d.state_dict()
        for k in sd:
            if "running" in k:  # batch means are cancellation-heavy: relative-to-max error of a near-zero mean
                close(sd[k], state.ds[i][k], 1e-3 if engine == "simt" else 2e-2, what=k)
    ema = t.bG.ema_state_dict()
    for k in state.g_keys:
        gr = keep["g_grads"][k]
        sel = gr.abs() > 0.2 * gr.abs().max()
        if k.endswith("conv3x3.1.bias") or not sel.any():
            continue
        assert ((gparams[k].detach().cpu() - state.g[k])[sel]).abs().max().item() < 5e-5, k
        assert ((ema[k].cpu() - state.g_avg[k])[sel]).abs().max().item() < 1e-6, k
        moved = (gparams[k].detach().cpu() - p0[k]).abs().max().item()
        assert moved > 1e-5, k   # the optimiser really stepped


def test_device_side_prepare_data_is_exact():
    """f4: the compact batch (no class heat maps, no label-embedding tensor: 14 % of the bytes) + the device-side
    rebuild (trainer.prepare_data: og_form_hmaps / og_form_clabels_feat) gives bit-identical step inputs to the
    host-built batch (ref: miscc/load.py:160-176 heat-map accumulation in roi order; miscc/utils.py:502-522)."""
    inp = synth.make_inputs(5, seed=9, parity=True)
    small = synth.compact(inp)
    assert synth.input_bytes(small) < 0.16 * synth.input_bytes(inp)
    t = trainer.StepATrainer(device=DEV, seed=5)
    dev = t.to_device(small)
    for a, b in zip(dev["hmaps"], inp["hmaps"]):
        assert torch.equal(a.cpu(), b)
    assert torch.equal(dev["slabels_feat"].cpu(), inp["slabels_feat"])
    # reference semantics (no clamp): overlapping same-class boxes add up
    dev2 = dict(t.to_device(small), hmap_clamp=0.0)
    hm = t.prepare_data(dev2)["hmaps"][0].cpu()
    want = torch.zeros_like(inp["hmaps"][0])
    want.scatter_add_(1, small["roi_cls"].view(5, -1, 1, 1).expand_as(inp["bt_masks"][0]), inp["bt_masks"][0])
    assert torch.equal(hm, want)


def test_cuda_graph_replay_matches_eager():
    """A replay of the captured whole-step CUDA graph computes the same step as eager launches from the same state."""
    inp = synth.make_inputs(4, seed=8, parity=True)
    a = trainer.StepATrainer(device=DEV, seed=5)
    b = trainer.StepATrainer(device=DEV, seed=5)
    da, db = a.to_device(inp), b.to_device(inp)
    p_before = b.bG.flat.clone()
    b.capture(db, warmup=2)                      # two eager warm-up steps (undone afterwards), then the capture
    assert torch.equal(b.bG.flat, p_before) and b.bG.step == 0 and int(b.bG.step_dev) == 0   # training state untouched
    # bring the eager trainer to exactly b's state (weights, Adam moments, EMA, BatchNorm buffers, step counters)
    for x, y in zip([a.bG, *a.bD], [b.bG, *b.bD]):
        for name in ("flat", "m", "v"):
            getattr(x, name).copy_(getattr(y, name))
        x.step, _ = y.step, x.step_dev.copy_(y.step_dev)
    a.bG.avg.copy_(b.bG.avg)
    for ma, mb in zip([a.netG, *a.netsPatD], [b.netG, *b.netsPatD]):
        for ba, bb in zip(ma.buffers(), mb.buffers()):
            ba.copy_(bb)
    ops.bump_param_epoch()
    oa = a.step(da)                              # eager
    ob = b.step(db)                              # graph replay
    torch.cuda.synchronize()
    assert b.launches_per_step > 500
    # every reduction of the step adds in a fixed order (DESIGN.md, run-to-run determinism): the replay gives the bits
    for k in ("errPatD0", "errPatD1", "errPatD2", "errG", "kl"):
        assert torch.equal(ob[k], oa[k]), (k, float(ob[k]), float(oa[k]))
    for i in range(3):
        assert torch.equal(ob["fake_imgs"][i], oa["fake_imgs"][i]), f"fake{i}"
    assert torch.equal(b.bG.grad, a.bG.grad), rel_l2(b.bG.grad, a.bG.grad)
    for i, (x, y) in enumerate(zip([a.bG, *a.bD], [b.bG, *b.bD])):
        assert torch.equal(y.flat, x.flat), (i, rel_l2(y.flat, x.flat))
    assert torch.equal(b.bG.avg, a.bG.avg)
    assert int(b.bG.step_dev) == int(a.bG.step_dev) == 1 and b.bG.step == 1


@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
@pytest.mark.parametrize("cls,n_layer", [("OBJ_SS_D_NET", 3), ("OBJ_LS_D_NET", 4)])
def test_obj_d_net_parity(cls, n_layer, engine, l2, mx, monkeypatch):
    """Object discriminators (512x512 bilinear front end, shape code, encoder, RoIAlignAvg, roi code): forward and the
    gradients w.r.t. the fake image and the parameters against the oracle, on the exact-fp32 engine AND on the shipped
    tensor-core engine (f16x3; gradient bounds as in test_pat_d_loss_parity)."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(14)
    net = getattr(model, cls)(80)
    net.apply(model.weights_init)
    net.to(DEV)
    sd = _cpu_sd(net)
    inp = synth.make_inputs(2, seed=6, parity=True)
    x, s, fm = inp["imgs"][2], inp["hmaps"][2], inp["fm_rois"]
    keys = [k for k in O.trainable_keys(sd) if not k.startswith(("COND_DNET", "UNCOND_DNET"))]
    live, leaves = O._with_grad(sd, keys)
    xr = x.clone().requires_grad_(True)
    out_r = O.obj_d_net_forward(live, xr, s, fm.numpy(), n_layer)
    g = torch.randn_like(out_r)
    grads = torch.autograd.grad(out_r, [xr] + [leaves[k] for k in keys], g)
    xg = x.to(DEV).requires_grad_(True)
    out = net(xg, s.to(DEV), fm.to(DEV), inp["num_rois"].to(DEV))
    close(out, out_r.detach(), what="fwd")
    out.backward(g.to(DEV))
    close_grad(xg.grad, grads[0], what="g_image", l2=l2, mx=mx)
    params = dict(net.named_parameters())
    for k, gr in zip(keys, grads[1:]):
        if k == "shp_code.1.bias":
            continue      # bias ahead of InstanceNorm: true gradient is zero
        close_grad(params[k].grad, gr, what=k, l2=l2, mx=mx)


@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
def test_shp_d_net_parity(engine, l2, mx, monkeypatch):
    """SHP_D_NET128 body + UNCOND head: forward and parameter / image gradients against the oracle (both engines)."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(15)
    net = model.SHP_D_NET128(80)
    net.apply(model.weights_init)
    net.to(DEV)
    sd = _cpu_sd(net)
    inp = synth.make_inputs(4, seed=7, parity=True)
    x, seg = inp["imgs"][1], inp["hmaps"][1]
    keys = O.trainable_keys(sd)
    live, leaves = O._with_grad(sd, keys)
    xr = x.clone().requires_grad_(True)
    loss_r = O.bce(O.d_get_logits(O.shp_d_net(xr, seg, live), live, "UNCOND_DNET"), 1)
    grads = torch.autograd.grad(loss_r, [xr] + [leaves[k] for k in keys])
    xg = x.to(DEV).requires_grad_(True)
    loss = ops.bce(net.UNCOND_DNET(net(xg, seg.to(DEV))), 1.0)
    assert abs(float(loss) - float(loss_r)) < 1e-4 * max(1.0, abs(float(loss_r)))
    loss.backward()
    close_grad(xg.grad, grads[0], what="g_image", l2=l2, mx=mx)
    params = dict(net.named_parameters())
    for k, gr in zip(keys, grads[1:]):
        if k == "shp_code.1.bias":
            continue
        close_grad(params[k].grad, gr, what=k, l2=l2, mx=mx)


@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
@pytest.mark.parametrize("cls,n_layer,large", [("OBJ_SS_D_NET", 3, False), ("OBJ_LS_D_NET", 4, True)])
def test_obj_d_loss_parity(cls, n_layer, large, engine, l2, mx, monkeypatch):
    """objD_loss (ref: miscc/losses.py:254-361): device-side roi compaction (feat_select), permuted-shape branch,
    COND / UNCOND heads and the loss weights, value and parameter gradients against the oracle (both engines)."""
    import random
    from objgan_b200 import losses
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(16)
    net = getattr(model, cls)(80)
    net.apply(model.weights_init)
    net.to(DEV)
    sd = _cpu_sd(net)
    inp = synth.make_inputs(3, seed=8, parity=True)
    real, seg, fm, nr = inp["imgs"][2], inp["hmaps"][2], inp["fm_rois"].clone(), inp["num_rois"]
    fm[..., 2:4] *= torch.tensor([1.0, 3.0, 0.2]).view(3, 1, 1)       # boxes on both sides of the size threshold
    fake = torch.tanh(torch.randn_like(real))
    raw_cond = inp["clabels_emb"]
    raw_bt = torch.randn(3, 10, cfg.GAN.GF_DIM)
    keys = O.trainable_keys(sd)
    live, leaves = O._with_grad(sd, keys)
    random.seed(12)
    loss_r = O.obj_d_loss(live, real, fake, seg, raw_cond, raw_bt, fm.numpy(), nr.tolist(), n_layer, is_large_scale=large)
    grads = torch.autograd.grad(loss_r, [leaves[k] for k in keys], allow_unused=True)
    random.seed(12)
    loss = losses.objD_loss(net, real.to(DEV), fake.to(DEV), seg.to(DEV), raw_cond.to(DEV), raw_bt.to(DEV), fm, nr,
                            is_large_scale=large)
    assert abs(float(loss) - float(loss_r)) < 1e-4 * max(1.0, abs(float(loss_r))), (float(loss), float(loss_r))
    loss.backward()
    params = dict(net.named_parameters())
    checked = 0
    for k, gr in zip(keys, grads):
        if gr is None or k == "shp_code.1.bias":
            continue
        close_grad(params[k].grad, gr, what=k, l2=l2, mx=mx)
        checked += 1
    assert checked >= 10


def test_damsm_losses_parity():
    """DAMSM words_loss / sent_loss (ref: miscc/losses.py:22-159) around the fused func_attention: loss values,
    attention maps, accuracy and the gradient reaching the image features / image code against the oracle."""
    from objgan_b200 import losses
    g = torch.Generator().manual_seed(19)
    B, nef, T = 6, 256, 18
    img = torch.randn(B, nef, 17, 17, generator=g)
    words = torch.randn(B, nef, T, generator=g)
    cnn = torch.randn(B, nef, generator=g)
    rnn = torch.randn(B, nef, generator=g)
    cap_lens = torch.tensor([18, 12, 9, 18, 5, 14])
    labels = torch.arange(B)
    class_ids = np.array([3, 7, 3, 1, 7, 9])
    ir = img.clone().requires_grad_(True)
    o0, o1, omaps, oacc = O.words_loss(ir, words, labels, cap_lens.tolist(), class_ids, B)
    go = torch.autograd.grad(o0 + 2.0 * o1, ir)[0]
    ig = img.to(DEV).requires_grad_(True)
    w0, w1, maps, acc = losses.words_loss(ig, words.to(DEV), labels.to(DEV), cap_lens, class_ids, B)
    close(w0, o0.detach(), what="w_loss0")
    close(w1, o1.detach(), what="w_loss1")
    assert abs(float(acc) - oacc) < 1e-4
    for a, b in zip(maps, omaps):
        close(a, b.detach(), what="att_map")
    (w0 + 2.0 * w1).backward()
    close_grad(ig.grad, go, what="g_img_features")
    cr = cnn.clone().requires_grad_(True)
    p0, p1, pacc = O.sent_loss(cr, rnn, labels, class_ids, B)
    gp = torch.autograd.grad(p0 + 0.5 * p1, cr)[0]
    cg = cnn.to(DEV).requires_grad_(True)
    s0, s1, sacc = losses.sent_loss(cg, rnn.to(DEV), labels.to(DEV), class_ids, B)
    close(s0, p0.detach(), what="s_loss0")
    close(s1, p1.detach(), what="s_loss1")
    assert abs(float(sacc) - pacc) < 1e-4
    (s0 + 0.5 * s1).backward()
    close_grad(cg.grad, gp, what="g_cnn_code")


@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
def test_g_loss_full_parity(engine, l2, mx, monkeypatch):
    """The generator's full loss (ref: miscc/losses.py:364-531: patch-D, shape-D, object-D small / large scale and the
    DAMSM word / sentence terms) -- value and the gradients reaching the three fake images and the generator's
    bt_c_code -- against the fixture the reference's own G_loss produced (tests/golden/g_loss.npz).  The image
    encoder is the stock-PyTorch stub of the fixture (the pretrained Inception encoder stays a stock module)."""
    import os
    import sys
    from objgan_b200 import losses
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_golden
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "g_loss.npz"))
    nets, inp, fakes, raw_bt, rois0, fm, class_ids = make_golden.g_loss_case()
    for n in nets["pat"] + nets["shp"] + [nets["ss"], nets["ls"]]:
        n.to(DEV)
    enc = make_golden.StubEncoder().to(DEV)
    fk = [f.to(DEV).requires_grad_(True) for f in fakes]
    bt = raw_bt.to(DEV).requires_grad_(True)
    total, logs = losses.G_loss(nets["pat"], nets["shp"], nets["ss"], nets["ls"], enc, fk,
                                [h.to(DEV) for h in inp["hmaps"]], inp["words_embs"].to(DEV), inp["sent_emb"].to(DEV),
                                inp["clabels_emb"].to(DEV), bt, torch.arange(2, device=DEV), inp["cap_lens"], class_ids,
                                rois0, fm, inp["num_rois"])
    assert {"objss_g_loss", "objls_g_loss", "w_loss", "s_loss"} <= set(logs)
    want = float(gold["total"])
    assert abs(float(total) - want) <= 1e-4 * max(1.0, abs(want)), (float(total), want)
    total.backward()
    close_grad(fk[0].grad, torch.from_numpy(gold["g64"]), what="g_fake64", l2=l2, mx=mx)
    close_grad(fk[1].grad[..., ::2, ::2], torch.from_numpy(gold["g128"]), what="g_fake128", l2=l2, mx=mx)
    close_grad(fk[2].grad[..., ::4, ::4], torch.from_numpy(gold["g256"]), what="g_fake256", l2=l2, mx=mx)
    # unit test of the loss FUNCTION: the reference's G_loss lets a gradient reach bt_c_code when the caller passes a
    # live tensor; the training step never does (trainer.py:393 detaches it -- see test_gpu_zz_step_b.py)
    close_grad(bt.grad, torch.from_numpy(gold["gbt"]), what="g_bt_c_code", l2=l2, mx=mx)
