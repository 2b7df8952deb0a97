"""The convolutions (csrc/conv_tc.cu, conv_simt.cu, wgmma.cuh) against float64, at every layer shape the networks run
(tests/conv_cases.py: CASES, ENC_CASES) and at rows that pin the kernels' code paths (EDGE_CASES), on both engines.

Each CASES / EDGE_CASES row runs through model.Conv2dP (ops.conv2d): forward, input gradient, weight gradient and bias
gradient.  Each ENC_CASES row runs ops.enc_conv_fwd into a channel slice of a NaN-filled destination, or
ops.enc_conv_dgrad.  The reference is torch in float64 on the device, from the same fp32 operands: orthogonal weights
(the networks' initialisation), N(0, 1) activations and output gradients, the layer's bias (the eval BatchNorm folded in
float64 for the encoder).  The LeakyReLU derivative follows the branch the kernel took (the sign of its output): an
element within rounding of 0 may take either.

Metric: per output channel (per input channel for the input gradient), max |got - ref| / max |ref| over that channel, so
an error confined to one N tile or one GLU half cannot hide under a larger channel.  The denominator is at least 1/16 of
the tensor's max |ref|: a channel of one element (the batch-1 linears) may cancel to near 0, and its relative error
says nothing about the kernel.  The bias gradient is compared as one vector.  Padding channels must hold exactly act(0)
(0, or 0.5 after a sigmoid: the epilogue runs over every padded channel, and consumers read the real ones), the padding
channels of the input gradient exactly 0, and an encoder output must leave every destination channel outside its slice
NaN as it was.

Bars, measured on an H100 SXM (80 GB, 700 W power limit) over every row and quantity of the unmodified kernels:
  f16x3  largest error 1.5e-6 on the tensor-core rows (s1 / s2 / encoder), 6.5e-6 on the CUDA-core rows (exact fp32,
         reductions of up to 9216 terms).  With every activation / gradient lo copy zeroed (a kernel that drops a lo
         product, test_zeroed_lo_is_caught) the smallest error over all tensor-core rows is 2.4e-4
         (enc dgrad 16x149x149 32->32 3x3).  BAR 4e-5: 6x the largest error, 1/6 of the smallest mutant.
  simt   exact fp32 FMA everywhere: largest error 8.6e-6 (forward of the 4x4 768->384 roi_code layer).  BAR 5e-5.
The old bar of the tensor-core test was 1e-4 of the global max|ref|, with forward and input gradient only.
"""
import pytest
import torch
import torch.nn.functional as F

from conv_cases import CASES, EDGE_CASES, ENC_CASES
from dry import record
from objgan_b200 import model, ops, synth, trainer
from objgan_b200.lib import ACT_LRELU, ACT_SIGMOID, ACT_TANH, PAD_REFLECT, PAD_ZERO, UPSAMPLE2X

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLOPE = 0.2
BN_EPS = 1e-3
BAR = {"f16x3": 4e-5, "simt": 5e-5}
MUTANT_FLOOR = 4            # a zeroed lo copy must give at least MUTANT_FLOOR x BAR on every tensor-core row
ENGINES = ("f16x3", "simt")
NAMES = {"s1": {"og_conv2d_tc", "og_conv2d_wgrad_tc"}, "s2": {"og_conv2d_tc", "og_conv2d_wgrad_tc"},
         "narrow": {"og_conv2d_narrow_fwd", "og_conv2d_narrow_dgrad", "og_conv2d_narrow_wgrad"},
         "simt": {"og_conv2d_simt", "og_conv2d_wgrad_simt"}}
WORST = {}          # (engine, path) -> largest error;  ("mutant",) -> (smallest zeroed-lo error, row)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST, key=str):
        print(f"\nconv worst {k}: {WORST[k]}")


def _note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), v)


def _rid(r):
    if isinstance(r[0], str):
        d, n, h, w, ci, co, kh, kw, s, ph, pw, relu, b, yoff, cy, path = r
        return f"{d}-{n}x{h}x{w}-{ci}to{co}-k{kh}x{kw}s{s}p{ph}{pw}-y{yoff}of{cy}-{path}"
    n, h, w, ci, co, k, s, p, mode, act, b, split, path = r
    return f"{n}x{h}x{w}-{ci}to{co}-k{k}s{s}p{p}m{mode}-a{act}{'b' if b else ''}-g{split}-{path}"


def _per_channel(got, ref, dim):
    """max |got - ref| / max |ref| per index of ``dim``; the denominator is at least 1/16 of the tensor's max |ref|."""
    dims = [d for d in range(ref.dim()) if d != dim]
    assert torch.isfinite(got).all()
    num = (got.double() - ref).abs().amax(dims)
    den = ref.abs().amax(dims)
    return (num / den.clamp_min(den.max().item() / 16).clamp_min(1e-300)).max().item()


def _act(z, act):
    if act == ACT_LRELU:
        return torch.where(z > 0, z, SLOPE * z)
    if act == ACT_TANH:
        return torch.tanh(z)
    if act == ACT_SIGMOID:
        return torch.sigmoid(z)
    return z


def _dact(z, y_kernel, act):
    if act == ACT_LRELU:
        return torch.where(y_kernel > 0, 1.0, SLOPE).double()
    if act == ACT_TANH:
        return 1 - torch.tanh(z) ** 2
    if act == ACT_SIGMOID:
        s = torch.sigmoid(z)
        return s * (1 - s)
    return torch.ones_like(z)


def _ref_conv(x, w, b, k, stride, pad, mode):
    if mode == PAD_REFLECT:
        return F.conv2d(F.pad(x, (pad,) * 4, mode="reflect"), w, b, stride)
    if mode == UPSAMPLE2X:
        return F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, 1, pad)
    return F.conv2d(x, w, b, stride, pad)


def _convs(calls):
    """The og_conv2d* names among recorded library calls."""
    return {n for n, _ in calls if n.startswith("og_conv2d")}


def _zero_lo(monkeypatch):
    """Every activation / gradient operand pair the tensor cores read gets an all-zero lo copy: the error of a kernel
    that drops the x_lo * w_hi product."""
    def wrap(real):
        def f(*a, **k):
            hi, lo, amax = real(*a, **k)
            z = ops._empty_slack(lo.shape, lo.device)
            z.zero_()
            return hi, z, amax
        return f
    monkeypatch.setattr(ops, "_split", wrap(ops._split))
    monkeypatch.setattr(ops, "_split_s2d_odd", wrap(ops._split_s2d_odd))


def _run_conv(row, engine, monkeypatch, seed=0, sinks=False):
    """Runs the row through model.Conv2dP; returns {quantity: error} and the library calls it issued."""
    N, H, W, Cin, Cout, k, stride, pad, mode, act, bias, split, path = row
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    torch.manual_seed(seed)
    m = model.Conv2dP(Cin, Cout, k, stride, pad, bias, mode, act, split).to(DEV)
    cp = ops.cpad(Cin)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    x = torch.randn(N, H, W, cp, device=DEV, generator=gen)
    x[..., Cin:] = 0
    oh, ow = ops._out_hw(H, W, k, k, stride, pad, mode)
    if split:
        sp = ops.cpad(split)
        kp, real = 2 * sp, list(range(split)) + list(range(sp, sp + split))
    else:
        kp, real = ops.cpad(Cout), list(range(Cout))
    real = torch.tensor(real, device=DEV)
    pad_ch = torch.ones(kp, dtype=torch.bool, device=DEV)
    pad_ch[real] = False
    pad_value = 0.5 if act == ACT_SIGMOID else 0.0          # act(0 + 0): the epilogue runs over every padded channel
    g = torch.randn(N, oh, ow, Cout, device=DEV, generator=gen)
    gfull = torch.zeros(N, oh, ow, kp, device=DEV)
    gfull[..., real] = g
    prefill = {}
    if sinks:
        for p_ in m.parameters():
            prefill[p_] = torch.linspace(-1, 1, p_.numel(), device=DEV).view(p_.shape)
            p_.og_grad_sink = prefill[p_].clone()

    last = []

    def passes():
        for _ in range(2 if sinks else 1):
            xg = x.clone().requires_grad_(True)
            y = m(xg)
            y.backward(gfull)
        last.extend((xg, y))
    calls = record(passes)
    xg, y = last
    assert y.shape == (N, oh, ow, kp)
    assert (y[..., pad_ch] == pad_value).all(), "padding channels of the output are not act(0)"
    assert (xg.grad[..., Cin:] == 0).all(), "padding channels of the input gradient are not 0"

    x64 = x[..., :Cin].permute(0, 3, 1, 2).double().requires_grad_(True)
    w64 = m.weight.detach().double().requires_grad_(True)
    b64 = m.bias.detach().double().requires_grad_(True) if bias else None
    z = _ref_conv(x64, w64, b64, k, stride, pad, mode)
    yk = y[..., real].permute(0, 3, 1, 2)
    gz = g.permute(0, 3, 1, 2).double() * _dact(z.detach(), yk, act)
    grads = torch.autograd.grad(z, [t for t in (x64, w64, b64) if t is not None], gz)
    err = {"fwd": _per_channel(yk, _act(z.detach(), act), 1),
           "dgrad": _per_channel(xg.grad[..., :Cin].permute(0, 3, 1, 2), grads[0], 1)}
    if sinks:
        assert m.weight.grad is None and (not bias or m.bias.grad is None), "a gradient was handed to autograd"
        gw = (m.weight.og_grad_sink.double() - prefill[m.weight]) / 2
        gb = (m.bias.og_grad_sink.double() - prefill[m.bias]) / 2 if bias else None
    else:
        gw, gb = m.weight.grad, m.bias.grad if bias else None
    err["wgrad"] = _per_channel(gw, grads[1], 0)
    if bias:
        err["bgrad"] = (gb.double() - grads[2]).abs().max().item() / grads[2].abs().max().item()
    return err, calls


def _check_path(row, engine, calls):
    """The og_conv2d* names issued are the row's path (f16x3), or the CUDA-core path of the same layer (simt)."""
    N, H, W, Cin, Cout, k, stride, pad, mode, act, bias, split, want = row
    if engine == "simt":
        oh, ow = ops._out_hw(H, W, k, k, stride, pad, mode)
        kp = 2 * ops.cpad(split) if split else ops.cpad(Cout)
        want = "narrow" if kp == 8 and mode == PAD_ZERO and N * oh * ow <= 65536 else "simt"
    assert _convs(calls) == NAMES[want], (_convs(calls), want)
    if want in ("s1", "s2"):                     # the forward's operand split of x
        assert next(a[6] for n, a in calls if n == "og_prep_split") == (want == "s2")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("row", CASES + EDGE_CASES, ids=_rid)
def test_conv(row, engine, monkeypatch):
    err, calls = _run_conv(row, engine, monkeypatch)
    _check_path(row, engine, calls)
    worst = max(err.values())
    _note((engine, row[-1]), worst)
    assert worst <= BAR[engine], err


def _enc_layer(row, seed):
    d, N, H, W, Cin, Cout, kh, kw, stride, padh, padw, relu, bias, yoff, Cy, path = row
    torch.manual_seed(seed)
    w = torch.empty(Cout, Cin, kh, kw)
    torch.nn.init.orthogonal_(w)
    w = w.to(DEV)
    bn = None
    if bias:
        gen = torch.Generator(device=DEV).manual_seed(seed + 2)
        bn = (torch.rand(Cout, device=DEV, generator=gen) + 0.5, torch.randn(Cout, device=DEV, generator=gen) * 0.1,
              torch.randn(Cout, device=DEV, generator=gen) * 0.1, torch.rand(Cout, device=DEV, generator=gen) + 0.5)
    layer = ops.EncConv([w], [bn] if bias else None, kh, kw, stride, padh, padw, BN_EPS, relu)
    w64 = w.double()
    b64 = None
    if bias:
        g, b, m, v = (t.double() for t in bn)
        s = g / torch.sqrt(v + BN_EPS)
        w64, b64 = w64 * s[:, None, None, None], b - m * s
    return layer, w64, b64


def _run_enc(row, engine, monkeypatch, seed=0):
    d, N, H, W, Cin, Cout, kh, kw, stride, padh, padw, relu, bias, yoff, Cy, path = row
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    layer, w64, b64 = _enc_layer(row, seed)
    oh, ow = layer.out_hw(H, W)
    cp = ops.cpad(Cin)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    if d == "fwd":
        x = torch.randn(N, H, W, cp, device=DEV, generator=gen)
        x[..., Cin:] = 0
        y = torch.full((N, oh, ow, Cy), float("nan"), device=DEV)
        calls = record(lambda: ops.enc_conv_fwd(layer, x, y, yoff))
        outside = torch.ones(Cy, dtype=torch.bool, device=DEV)
        outside[yoff:yoff + Cout] = False
        assert torch.isnan(y[..., outside]).all(), "a channel outside the output slice was written"
        z = F.conv2d(x[..., :Cin].permute(0, 3, 1, 2).double(), w64, b64, stride, (padh, padw))
        ref = z.clamp_min(0) if relu else z
        err = {"fwd": _per_channel(y[..., yoff:yoff + Cout].permute(0, 3, 1, 2), ref, 1)}
    else:
        gp = torch.randn(N, oh, ow, Cout, device=DEV, generator=gen)
        out = []
        calls = record(lambda: out.append(ops.enc_conv_dgrad(layer, gp, H, W)))
        gx, = out
        assert gx.shape == (N, H, W, cp) and (gx[..., Cin:] == 0).all()
        x64 = torch.zeros(N, Cin, H, W, device=DEV, dtype=torch.float64, requires_grad=True)
        z = F.conv2d(x64, w64, None, stride, (padh, padw))
        ref, = torch.autograd.grad(z, x64, gp.permute(0, 3, 1, 2).double())
        err = {"dgrad": _per_channel(gx[..., :Cin].permute(0, 3, 1, 2), ref, 1)}
    return err, calls


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("row", ENC_CASES, ids=_rid)
def test_enc_conv(row, engine, monkeypatch):
    err, calls = _run_enc(row, engine, monkeypatch)
    want = "og_conv2d_tc" if engine == "f16x3" and row[-1] == "tc" else "og_conv2d_simt"
    assert _convs(calls) == {want}
    worst = max(err.values())
    _note((engine, "enc_" + row[-1]), worst)
    assert worst <= BAR[engine], err


TC_ROWS = [r for r in CASES + EDGE_CASES if r[-1] in ("s1", "s2")] + [r for r in ENC_CASES if r[-1] == "tc"]


@pytest.mark.parametrize("row", TC_ROWS, ids=_rid)
def test_zeroed_lo_is_caught(row, monkeypatch):
    """With the activation / gradient lo copies zeroed, the tensor-core rows fail the f16x3 bar by MUTANT_FLOOR at least:
    the bar sits well below the error of a kernel that drops a lo product."""
    _zero_lo(monkeypatch)
    err, _ = (_run_enc if isinstance(row[0], str) else _run_conv)(row, "f16x3", monkeypatch)
    worst = max(v for k, v in err.items() if k != "bgrad")
    prev = WORST.get(("mutant",))
    if prev is None or worst < prev[0]:
        WORST[("mutant",)] = (worst, _rid(row))
    assert worst >= MUTANT_FLOOR * BAR["f16x3"], err


SINK_ROWS = [
    (2, 16, 16, 32, 40, 3, 1, 1, PAD_REFLECT, ACT_TANH, True, 0, "s1"),
    (2, 32, 32, 64, 16, 3, 1, 1, 0, 0, False, 0, "s1"),
    (4, 32, 32, 16, 64, 4, 2, 1, 0, ACT_SIGMOID, True, 0, "s2"),
    (4, 64, 64, 96, 192, 4, 2, 1, 0, 0, False, 0, "s2"),
    (3, 8, 8, 96, 48, 3, 1, 1, UPSAMPLE2X, 0, False, 24, "s1"),
    (4, 8, 8, 24, 1, 4, 2, 0, 0, ACT_SIGMOID, True, 0, "narrow"),
    (1, 6, 6, 16, 1, 4, 2, 0, 0, 0, False, 0, "narrow"),
    (2, 6, 6, 40, 20, 3, 1, 1, 0, ACT_LRELU, True, 0, "simt"),
    (2, 6, 6, 40, 24, 3, 1, 1, 0, 0, False, 0, "simt"),
]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("row", SINK_ROWS, ids=_rid)
def test_gradient_sink(row, engine, monkeypatch):
    """``param.og_grad_sink`` set on the weight and the bias: two backward passes accumulate into it (og_unpack_wgrad /
    og_unpack_upsample_wgrad / og_channel_sum with accumulate=1) and hand autograd no gradient."""
    assert row in CASES + EDGE_CASES
    err, calls = _run_conv(row, engine, monkeypatch, sinks=True)
    _check_path(row, engine, calls)
    assert max(err.values()) <= BAR[engine], err


def test_pack_plan_matches_per_layer_pack():
    """After a Step-B step every network re-packs its weights through PackPlan.run (og_amax_multi +
    og_pack_weights_f16_multi): each job's amax word and fp16 hi / lo copies equal, bit for bit, what og_amax +
    og_pack_weights_f16 derive from the same (updated) weights."""
    import random
    t = trainer.StepBTrainer(device=DEV, seed=3)
    inp = synth.make_inputs(2, seed=4, parity=True)
    random.seed(5)
    t.step(t.to_device(inp))
    torch.cuda.synchronize()
    jobs = 0
    assert all(b.step == 1 for b in [t.bG, *t.bD, *t.bShp])
    for b in [t.bG, *t.bD, *t.bShp, *t.bObj]:
        if b.step == 0:          # an object discriminator without rois in this batch: no update, nothing re-packed
            continue
        assert b.plan.jobs
        for cache, w, cip, kp, split, splitp, tr, hi, lo, amax in b.plan.jobs:
            co, ci, kh, kw = w.shape
            a = torch.empty(1, device=DEV, dtype=torch.int32)
            ops._call("og_amax", ops._p(w), w.numel(), ops._p(a))
            h2, l2 = torch.empty_like(hi), torch.empty_like(lo)
            ops._call("og_pack_weights_f16", ops._p(w), co, ci, kh, kw, cip, kp, split, splitp, tr, ops._p(a),
                      ops._p(h2), ops._p(l2))
            assert torch.equal(a, amax)
            assert torch.equal(h2.view(torch.int16), hi.view(torch.int16))
            assert torch.equal(l2.view(torch.int16), lo.view(torch.int16))
            assert cache.hl[tr][0] is hi
            jobs += 1
    assert jobs > 50
