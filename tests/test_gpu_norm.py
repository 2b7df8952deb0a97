"""The normalisation kernels (csrc/norm.cu) against a float64 restatement of their math, at every shape the networks
run them (tests/norm_cases.py: CASES, SPLIT_CASES) and at rows that pin each code path (EDGE_CASES, SPLIT_EDGE_CASES).

The reference is computed on the device in float64 from the same fp32 inputs the kernels get: two-pass biased variance,
eps 1e-5 inside the square root, running statistics with momentum 0.1 and the unbiased variance.  It is NOT the CPU
fp32 oracle.

Inputs per channel: offsets |mu| / sigma in {0, 3, 30, 300} (a conv bias before InstanceNorm), one channel with
sigma^2 = eps (an eps mistake is an O(1) error there), one exactly constant channel (variance 0), GLU gates driven to
+-30 and beyond (sigmoid_fast's exp overflow), and zero pad lanes (the 194-of-200 channel halves of HmapResBlock).

Bounds.  Values are compared per (group, channel): max |got - ref| <= TOL (1 + r) max|ref of the tensor|, TOL = 1e-5,
where r = |mean| / sqrt(var + eps) of the channel.  The (1 + r) is the arithmetic of x - mean in fp32: the mean is
rounded to fp32 (error |mean| 2^-24), which moves xhat by r 2^-24; everything else is a few fp32 roundings of O(1)
values.  A constant channel has r = 0: x - mean is exactly 0 there.  mean and rstd (read back from og_norm_stats) are
held to a few fp32 ulps of the float64 values, plus, for rstd, the one-pass variance's cancellation 7 2^-24 rho / 2
(rho = (mean^2 + var) / (var + eps)) where the kernel keeps the one-pass result (rho < 2048; above 1024 it recomputes the
channel from shifted sums, and those channels -- the constant ones and |mean| / sigma = 300 -- are held to ulps).  That
slack also enters the value bounds, in units of TOL.  The amax words must equal max|out| / max|dx| bitwise; pad lanes
must be exactly 0.  The statistics and the backward are called twice and must repeat bit for bit (the per-CTA sums are
added in a fixed order).

LeakyReLU's derivative is discontinuous at 0: an element whose pre-activation lies within the forward's error band of
0 (2^-18 (1 + r) (|gamma| (1 + |xhat|) + |beta|)) may take either branch, so there the reference follows the branch the
kernel took (read from the sign of its output); measured on an H100, 3.3e-6 of the elements fall in that band.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from norm_cases import CASES, EDGE_CASES, SPLIT_CASES, SPLIT_EDGE_CASES
from objgan_b200 import ops
from objgan_b200.lib import NA_GLU, NA_LRELU, NA_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS, MOM, SLOPE = 1e-5, 0.1, 0.2
TOL = 1e-5
OFFSETS = (0.0, 3.0, 30.0, 300.0)
WORST = {}          # kernel family -> worst observed error / (1 + r) max|ref|, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"norm worst error {k}: {WORST[k]:.3e}")


def _note(name, v):
    WORST[name] = max(WORST.get(name, 0.0), v)


def _call(name, *args):
    ops._call(name, *[ops._p(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _f32_bits(t):
    return t.contiguous().view(torch.int32)


def _real_mask(Cy, act):
    """Channels that carry data: HmapResBlock's 194 of 200 per half (Cy = 200 / 400); every channel otherwise."""
    m = torch.ones(Cy, dtype=torch.bool, device=DEV)
    if Cy in (200, 400):
        for h in range(Cy // 200):
            m[h * 200 + 194:(h + 1) * 200] = False
    return m


def _inputs(kind, G, P, Cy, act, residual, affine, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    Co = Cy // 2 if act == NA_GLU else Cy
    real = _real_mask(Cy, act)
    sigma = torch.exp(torch.rand(Cy, device=DEV, generator=gen) * 1.4 - 0.7)
    sign = torch.where(torch.arange(Cy, device=DEV) % 8 < 4, 1.0, -1.0)
    mu = sign * sigma * torch.tensor(OFFSETS, device=DEV).repeat(Cy // 4 + 1)[:Cy]
    mu = mu[None, :] * (1 + 0.25 * (torch.arange(G, device=DEV)[:, None] % 4))   # groups differ
    y = torch.randn(G, P, Cy, device=DEV, generator=gen) * sigma + mu[:, None, :]
    if Cy > 4:
        y[:, :, 1] = torch.randn(G, P, device=DEV, generator=gen) * math.sqrt(EPS) + 0.01   # sigma^2 = eps
        y[:, :, 2] = 0.3                                                                       # constant channel
    if act == NA_GLU and Co > 4 and P > 1:
        y[:, :, Co + 3] = 0.0               # gate spikes: xhat = -+sqrt(P - 1) at pixel 0 (saturated gates)
        y[:, 0, Co + 3] = -1.0
        if Co > 5:
            y[:, :, Co + 5] = 0.0
            y[:, 0, Co + 5] = 1.0
    y[:, :, ~real] = 0.0
    y = y.float().contiguous()
    gamma = beta = None
    if affine:
        gamma = (torch.rand(Cy, device=DEV, generator=gen) + 0.5) * sign
        beta = torch.randn(Cy, device=DEV, generator=gen) * 0.5
        if act == NA_GLU and Co > 2:
            gamma[Co], beta[Co] = 30.0, -30.0        # gate n = 30 xhat - 30: exp(-n) overflows for xhat < -1.9
            gamma[Co + 2], beta[Co + 2] = 30.0, 30.0
    realo = real[:Co]
    res = None
    if residual:
        res = torch.randn(G, P, Co, device=DEV, generator=gen)
        res[:, :, ~realo] = 0.0
    g = torch.randn(G, P, Co, device=DEV, generator=gen)
    g[:, :, ~realo] = 0.0
    return y, gamma, beta, res, g, real


def _ref_stats(y64):
    m = y64.mean(1)
    var = ((y64 - m[:, None, :]) ** 2).mean(1)
    return m, var


def _act_fwd(n, act, Co):
    if act == NA_GLU:
        return n[..., :Co] * torch.sigmoid(n[..., Co:])
    if act == NA_LRELU:
        return torch.where(n > 0, n, SLOPE * n)
    return n


def _act_bwd(n, g, act, Co, pos=None):
    if act == NA_GLU:
        s = torch.sigmoid(n[..., Co:])
        return torch.cat((g * s, g * n[..., :Co] * s * (1 - s)), -1)
    if act == NA_LRELU:
        return torch.where(n > 0 if pos is None else pos, g, SLOPE * g)
    return g


def _check(family, got, ref, ratio, tol=TOL):
    """per (group, channel): max over pixels |got - ref| <= tol (1 + ratio) max|ref|"""
    got = got.double()
    assert torch.isfinite(got).all(), family
    scale = max(ref.abs().max().item(), 1e-30)
    err = (got - ref).abs().amax(1)
    worst = (err / ((1 + ratio) * scale)).max().item()
    _note(family, worst)
    assert worst <= tol, (family, worst)


def _ulps(a, b):
    """|a - b| in units of the fp32 spacing at max(|a|, |b|)"""
    m = torch.maximum(a.abs(), b.abs()).double()
    _, e = torch.frexp(m)
    sp = torch.ldexp(torch.ones_like(m), (e - 24).clamp(min=-149))
    return ((a.double() - b.double()).abs() / sp).max().item()


def _pair_ratio(ratio, act, Co):
    if act != NA_GLU:
        return ratio
    r = torch.maximum(ratio[:, :Co], ratio[:, Co:])
    return r, torch.cat((r, r), 1)


def _run_case(case, seed=0):
    kind, G, P, Cy, act, residual, affine = case
    Co = Cy // 2 if act == NA_GLU else Cy
    y, gamma, beta, res, g, real = _inputs(*case, seed=seed)
    y64 = y.double()
    if kind == "bn_eval":
        gen = torch.Generator(device=DEV).manual_seed(seed + 1)
        m_all, v_all = _ref_stats(y64)
        rm = (m_all[0] + torch.randn(Cy, device=DEV, generator=gen, dtype=torch.float64) * 0.1).float()
        rv = (v_all[0] * (0.8 + 0.4 * torch.rand(Cy, device=DEV, generator=gen, dtype=torch.float64))).float()
        rv[min(1, Cy - 1)] = 0.0                     # running variance 0: rstd = 1 / sqrt(eps)
        m_ref, rstd_ref = rm.double()[None], (1 / torch.sqrt(rv.double() + EPS))[None]
        mean, rstd = torch.empty(Cy, device=DEV), torch.empty(Cy, device=DEV)
        _call("og_bn_eval_coef", rm, rv, Cy, EPS, mean, rstd)
        assert torch.equal(mean, rm)
        assert _ulps(rstd, rstd_ref[0].float()) <= 1
        var_ref = None
    else:
        m_ref, var_ref = _ref_stats(y64)
        rstd_ref = 1 / torch.sqrt(var_ref + EPS)
        stats = torch.empty(G * Cy * 2, device=DEV, dtype=torch.float64)
        mean, rstd = torch.empty(G * Cy, device=DEV), torch.empty(G * Cy, device=DEV)
        bufs = (None, None, None)
        if kind == "bn":
            gen = torch.Generator(device=DEV).manual_seed(seed + 2)
            rm0 = torch.randn(Cy, device=DEV, generator=gen)
            rv0 = torch.rand(Cy, device=DEV, generator=gen) + 0.5
            bufs = (rm0.clone(), rv0.clone(), torch.full((), 5, dtype=torch.long, device=DEV))
        _call("og_norm_stats", y, G, P, Cy, EPS, stats, mean, rstd, *bufs[:2], MOM, Cy, bufs[2])
        # mean: the fp32 pair sums (<= 2 roundings of |x| <= |mean| + spread) and the final fp32 rounding
        dm = (mean.view(G, Cy).double() - m_ref).abs()
        assert (dm <= 2.0 ** -22 * (m_ref.abs() + var_ref.sqrt())).all(), dm.max().item()
        # the one-pass variance: sumsq is off by <= 3 U sumsq (fp32 squares and pair sums), mean^2 by <= 4 U sumsq, so
        # var + eps by <= 7 U rho (var + eps), rho = (mean^2 + var) / (var + eps); the kernel recomputes every channel
        # with rho > 1024 exactly, so only rho < 2048 (both sides of the switch, with the kernel's own rounding) has it
        rho = (m_ref ** 2 + var_ref) / (var_ref + EPS)
        cancel = torch.where(rho < 2048, 7 * 2.0 ** -24 * rho, torch.zeros_like(rho))
        rel = (rstd.view(G, Cy).double() - rstd_ref).abs() / rstd_ref
        _note("og_norm_stats rstd (relative)", rel.max().item())
        _note("og_norm_stats rstd (relative, exactly recomputed channels)", rel[rho >= 2048].max().item()
              if (rho >= 2048).any() else 0.0)
        assert (rel <= 2.0 ** -20 + cancel / 2).all(), (rel - cancel / 2).max().item()
        if kind == "bn":
            unb = var_ref[0] * P / (P - 1) if P > 1 else var_ref[0]
            want_m = (1 - MOM) * rm0.double() + MOM * m_ref[0]
            want_v = (1 - MOM) * rv0.double() + MOM * unb
            slack = (0.0, MOM * (P / (P - 1) if P > 1 else 1) * cancel[0] * (var_ref[0] + EPS))
            for (got, want), sl in zip(((bufs[0], want_m), (bufs[1], want_v)), slack):
                r = ((got.double() - want).abs() - sl).max().item() / want.abs().max().item()
                _note("og_norm_stats running buffers", r)
                assert r <= 1e-6, r
            assert int(bufs[2]) == 6
        # a second run: the per-CTA sums are added in a fixed order, so the statistics repeat bitwise
        mean2, rstd2 = torch.empty_like(mean), torch.empty_like(rstd)
        _call("og_norm_stats", y, G, P, Cy, EPS, stats, mean2, rstd2, None, None, MOM, Cy, None)
        assert torch.equal(mean, mean2) and torch.equal(rstd, rstd2)
    # x - mean is exact for a constant channel: it carries no offset error.  A one-pass rstd error moves xhat by as much,
    # relative: it is added to the ratio in units of TOL
    ratio = (m_ref.abs() * rstd_ref).clone()
    if var_ref is not None:
        ratio[var_ref == 0] = 0
        ratio = ratio + cancel / 2 / TOL
    else:
        ratio = ratio.expand(G, Cy)
    ro, rx = _pair_ratio(ratio, act, Co) if act == NA_GLU else (ratio, ratio)

    # forward
    xhat = (y64 - m_ref[:, None, :]) * rstd_ref[:, None, :]
    n = xhat * (gamma.double() if affine else 1) + (beta.double() if affine else 0)
    out_ref = _act_fwd(n, act, Co) + (res.double() if residual else 0)
    out = torch.empty(G, P, Co, device=DEV)
    amax = torch.empty(1, device=DEV, dtype=torch.int32)
    _call("og_norm_apply", y, G, P, Cy, mean, rstd, gamma, beta, res, act, SLOPE, out, amax)
    _check(f"og_norm_apply {kind}", out, out_ref, ro)
    assert (out[:, :, ~real[:Co]] == 0).all()
    assert int(amax.item()) == int(_f32_bits(out.abs().max().reshape(1)).item())

    # backward.  LeakyReLU's derivative jumps at n = 0: where |n| is within the forward's error band of 0, the reference
    # takes the branch the kernel took (the sign of its output), elsewhere its own
    pos = None
    if act == NA_LRELU and not residual:
        ga = gamma.double().abs() if affine else 1
        band = 2.0 ** -18 * (1 + ratio[:, None, :]) * (ga * (1 + xhat.abs()) + (beta.double().abs() if affine else 0))
        pos = torch.where(n.abs() <= band, out > 0, n > 0)
        _note("LeakyReLU branch taken from the kernel (fraction)", (pos != (n > 0)).double().mean().item())
    dn = _act_bwd(n, g.double(), act, Co, pos)
    dxh = dn * (gamma.double() if affine else 1)
    dx = torch.empty_like(y)
    amax_dx = torch.empty(1, device=DEV, dtype=torch.int32)
    dgam = torch.empty(Cy, device=DEV) if affine else None
    dbet = torch.empty(Cy, device=DEV) if affine else None
    if kind == "bn_eval":
        dx_ref = dxh * rstd_ref[:, None, :]
        _call("og_bn_eval_backward", y, g, P, Cy, mean, rstd, gamma, beta, act, SLOPE, dx, dgam, dbet, 0, amax_dx)
        dx2, dg2, db2 = torch.empty_like(dx), torch.empty_like(dgam), torch.empty_like(dbet)
        _call("og_bn_eval_backward", y, g, P, Cy, mean, rstd, gamma, beta, act, SLOPE, dx2, dg2, db2, 0, None)
        assert torch.equal(dx, dx2) and torch.equal(dgam, dg2) and torch.equal(dbet, db2)   # fixed-order planes
        fam = "og_bn_eval_backward"
    else:
        dx_ref = rstd_ref[:, None, :] * (dxh - dxh.mean(1, keepdim=True)
                                         - xhat * (dxh * xhat).mean(1, keepdim=True))
        bstats = torch.empty(G * Cy * 2, device=DEV, dtype=torch.float64)
        _call("og_norm_backward", y, g, G, P, Cy, mean, rstd, gamma, beta, act, SLOPE, bstats, dx, dgam, dbet, 0,
              amax_dx)
        dx2 = torch.empty_like(dx)
        dg2, db2 = (torch.empty_like(dgam), torch.empty_like(dbet)) if affine else (None, None)
        _call("og_norm_backward", y, g, G, P, Cy, mean, rstd, gamma, beta, act, SLOPE, bstats, dx2, dg2, db2, 0, None)
        assert torch.equal(dx, dx2) and (not affine or (torch.equal(dgam, dg2) and torch.equal(dbet, db2)))
        fam = f"og_norm_backward {kind}"
    _check(f"{fam} dx", dx, dx_ref, rx)
    assert (dx[:, :, ~real] == 0).all()
    assert int(amax_dx.item()) == int(_f32_bits(dx.abs().max().reshape(1)).item())
    if affine:
        # dgamma / dbeta: sums over P of O(1) terms; the per-term error is the xhat error above
        ref_dg, ref_db = (dn * xhat).sum(1)[0], dn.sum(1)[0]
        scale_g = max((dn * xhat).abs().sum(1)[0].max().item(), 1e-30)
        scale_b = max(dn.abs().sum(1)[0].max().item(), 1e-30)
        for name, got, ref, sc in (("dgamma", dgam, ref_dg, scale_g), ("dbeta", dbet, ref_db, scale_b)):
            err = ((got.double() - ref).abs() / ((1 + rx[0]) * sc)).max().item()
            _note(f"{fam} {name}", err)
            assert err <= TOL, (name, err)


@pytest.mark.parametrize("case", CASES + EDGE_CASES, ids=lambda c: "-".join(map(str, c)))
def test_norm_against_float64(case):
    _run_case(case)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------
# producer-side operand split: og_norm_bound + og_norm_apply_split
# ---------------------------------------------------------------------------------------------------
def _scale_exp(bound):
    return 13 - math.floor(math.log2(bound))


def _split_run(instance, N, H, W, Cy, act, residual, pad, y=None, gamma=None, beta=None, res=None):
    Co = Cy // 2 if act == NA_GLU else Cy
    G, P = (N, H * W) if instance else (1, N * H * W)
    if y is None:
        y, gamma, beta, res, _, _ = _inputs("in" if instance else "bn", G, P, Cy, act, residual, not instance, 11)
    y = y.reshape(N, H, W, Cy).contiguous()
    stats = torch.empty(G * Cy * 2, device=DEV, dtype=torch.float64)
    mean, rstd = torch.empty(G * Cy, device=DEV), torch.empty(G * Cy, device=DEV)
    _call("og_norm_stats", y, G, P, Cy, EPS, stats, mean, rstd, None, None, MOM, Cy, None)
    out_apply = torch.empty(N, H, W, Co, device=DEV)
    _call("og_norm_apply", y, G, P, Cy, mean, rstd, gamma, beta, res, act, SLOPE, out_apply, None)
    res_word = None
    if res is not None:
        res = res.reshape(N, H, W, Co).contiguous()
        res_word = _f32_bits(res.abs().max().reshape(1)).clone()
    word = torch.empty(1, device=DEV, dtype=torch.int32)
    _call("og_norm_bound", gamma, beta, Cy if gamma is not None else 0, P, res_word, word)
    bound = word.view(torch.float32).item()
    Hp, Wp = H + 2 * pad, W + 2 * pad
    xh = torch.empty(N, Hp, Wp, Co, device=DEV, dtype=torch.float16)
    xl = torch.empty_like(xh)
    out = torch.empty_like(out_apply)
    _call("og_norm_apply_split", y, N, H, W, Cy, instance, mean, rstd, gamma, beta, res, act, SLOPE, out, word, pad,
          xh, xl)
    return out_apply, out, xh, xl, bound


@pytest.mark.parametrize("case", SPLIT_CASES + SPLIT_EDGE_CASES, ids=lambda c: "-".join(map(str, c)))
def test_norm_apply_split(case):
    instance, N, H, W, Cy, act, residual, pad = case
    out_apply, out, xh, xl, bound = _split_run(*case)
    assert _ulps(out, out_apply) <= 1                        # same arithmetic as og_norm_apply
    assert bound >= out_apply.abs().max().item()
    k = _scale_exp(bound)
    assert torch.isfinite(xh.float()).all() and xh.float().abs().max().item() < 2.0 ** 14
    want = out.permute(0, 3, 1, 2).double()                 # the fp32 values the copies were made from
    if pad:
        want = F.pad(want, (1, 1, 1, 1), mode="reflect")
        hi = xh.permute(0, 3, 1, 2).float()
        assert torch.equal(F.pad(hi[:, :, 1:-1, 1:-1], (1, 1, 1, 1), mode="reflect"), hi)   # halo = reflection
    want = want.permute(0, 2, 3, 1)
    rec = (xh.double() + xl.double()) * 2.0 ** -k
    rel = 2.0 ** -22
    err = ((rec - want).abs() / torch.clamp(want.abs() * rel, min=bound * 2.0 ** -38)).max().item()
    _note("og_norm_apply_split reconstruction (x bound)", err)
    assert err <= 1.0, err


@pytest.mark.parametrize("instance", [0, 1])
@pytest.mark.parametrize("act", [NA_NONE, NA_LRELU, NA_GLU])
def test_norm_bound_adversarial(instance, act):
    """Per channel one pixel at +a, the rest 0: xhat = sqrt(P - 1), the largest value a normalised channel can take,
    at the channel with the largest gamma, plus a residual whose maximum sits on the same pixel.  The a-priori bound
    must still bound max|out|, and the scaled fp16 copies stay finite and below 2^14."""
    N, H, W, Cy = 2, 16, 16, 32
    Co = Cy // 2 if act == NA_GLU else Cy
    G, P = (N, H * W) if instance else (1, N * H * W)
    y = torch.zeros(G, P, Cy, device=DEV)
    y[:, 0, :] = 5.0
    gamma = beta = None
    if not instance:
        gamma = torch.full((Cy,), 0.5, device=DEV)
        gamma[3] = 4.0
        beta = torch.full((Cy,), 0.25, device=DEV)
        beta[3] = 1.0
        if act == NA_GLU:
            gamma[Co:], beta[Co:] = 0.0, 40.0    # gate sigmoid(40) == 1 in fp32: out = the full "a" value
    res = torch.zeros(G, P, Co, device=DEV)
    res[:, 0, :] = 2.0
    res[:, 1, :] = -1.0
    out_apply, out, xh, xl, bound = _split_run(instance, N, H, W, Cy, act, True, 1, y=y, gamma=gamma, beta=beta,
                                               res=res)
    mx = out_apply.abs().max().item()
    assert bound >= mx, (bound, mx)
    if act != NA_GLU or instance:   # (BatchNorm + GLU: the bound counts the gate half's max|beta| too)
        assert mx >= 0.99 * (bound - 2.0) / 1.001, (bound, mx)     # the bound is tight for this input
    for t in (xh, xl):
        assert torch.isfinite(t.float()).all() and t.float().abs().max().item() < 2.0 ** 14
