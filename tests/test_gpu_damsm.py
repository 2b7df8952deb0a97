"""The DAMSM matching kernels (csrc/words_pairs.cu, csrc/damsm.cu) and the image encoder's backward gathers that carry
the DAMSM gradient back to the image (og_bilinear_bwd_gather, og_global_avg_bwd, og_relu_grad_slice in
csrc/inception.cu) against a float64 restatement, at every shape the networks run them (tests/damsm_cases.py: CASES) and
at rows that pin the paths and edges they do not reach (EDGE_CASES).  Every row goes through the public C ABI.

The reference is computed on the device in float64 from the same fp32 inputs the kernels get, with torch autograd for
the gradients.  It restates the reference's expressions: func_attention (GlobalAttention.py:32-70: softmax over the
words, gamma1, softmax over the regions, weighted context), the cosine with its eps clamp (losses.py:13-19, 43-50), the
Eq. (10) pooling and the two cross-entropy directions (losses.py:50-58, 101-139) with the top-1 taken at the first
maximum as torch.max does, and the adjoint of F.interpolate(align_corners=True).  It is NOT the CPU fp32 oracle.

Inputs.  words_pairs: caption lengths 1 .. T and one above T (the kernel clamps it to T), NaN in every word slot past a
caption's length (never read), NaN-filled wc / attn buffers (rows l >= len must stay NaN: the forward leaves them
untouched and the backward never reads them); "zero" rows add an all-zero word column and an all-zero image, where the
cosine's denominator is clamped to eps.  cosine_matrix: "zero" rows put one zero row in each operand.  ce_pair: scores
on a grid with no near-ties (adjacent values 2 / B^2 apart, 10 / B^2 after gamma3), except one row and one column
holding an exact tie for their maximum at the label and at a later index, so that top-1 must take the first maximum.

Bounds.  The smooth outputs are held to max |got - ref| <= BAR max |ref| (per image for words_pairs' g_ctx, per row for
cosine_matrix's gradient: a zero image or row has gradients of size 1 / eps that would hide every other one).  The bars
(BAR) are about 4x the worst errors measured on an H100 80GB HBM3 at its 700 W power limit (the errors are printed at
the end of the module); the arithmetic they cover is fp32 dot products over ndf = 256 channels, two softmaxes, a
log-sum-exp.  Element-wise bounds where the arithmetic is a few operations: ce_pair_bwd (g0 G0 + g1 G1) to
2^-23 (|g0 G0| + |g1 G1|), two roundings (measured: 0.66 of it); the bilinear gather to 2^-21 sum |w g| over its terms
(w the product of the two axis weights; measured: 0.57 of it), so a dropped or misplaced contribution is an O(1) error
at its element, not noise.  The gather's reference is built from the same fp32 coordinates the kernels use:
r = (IS - 1) / (OS - 1) in fp32, f = r o in fp32, a = (int) f, b = a + (a < IS - 1), l = f - a.  global_avg_bwd (one fp32 division) and relu_grad_slice (selection) are
compared bit for bit; `correct` of ce_pair must equal the float64 top-1 count exactly.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from damsm_cases import (BL_BWD, CASES, CE, CE_BWD, COS_BWD, COS_FWD, EDGE_CASES, ENTRIES, GAP_BWD, REFUSED,
                         RELU_SLICE, WP_BWD, WP_FWD)
from objgan_b200 import ops
from objgan_b200.config import cfg

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
EPS = 1e-8
GAMMA1, GAMMA2, GAMMA3 = cfg.TRAIN.SMOOTH.GAMMA1, cfg.TRAIN.SMOOTH.GAMMA2, cfg.TRAIN.SMOOTH.GAMMA3
SENTINEL = 777.0
# max |got - ref| / max |ref| (see the module docstring): about 4x the worst error measured over every row on an
# H100 80GB HBM3 at its 700 W power limit, which is given in each comment
BAR = {
    "words_pairs sim": 8e-7,          # 1.93e-7
    "words_pairs wc": 6e-6,           # 1.47e-6
    "words_pairs attn": 8e-6,         # 1.91e-6
    "words_pairs g_ctx": 1.2e-5,      # 2.83e-6
    "cosine_matrix out": 3e-6,        # 6.91e-7
    "cosine_matrix ga": 1.3e-6,       # 3.18e-7
    "ce_pair loss": 1.5e-6,           # 3.55e-7
    "ce_pair G": 2.3e-6,              # 5.58e-7
}
WORST = {}                  # family -> worst observed error (relative, or error / bound for the bounded ones)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        bar = f"  (bar {BAR[k]:.1e})" if k in BAR else ""
        print(f"damsm worst error {k}: {WORST[k]:.3e}{bar}")


def _note(name, v):
    WORST[name] = max(WORST.get(name, 0.0), v)


def _call(name, *args):
    ops._call(name, *[ops._p(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rel(got, ref, dims=None):
    """max |got - ref| / max |ref|, over the whole tensor or per slice along the leading `dims` dimensions"""
    err, mag = (got.double() - ref).abs(), ref.abs()
    if dims is not None:
        err, mag = err.flatten(dims).amax(-1), mag.flatten(dims).amax(-1)
    else:
        err, mag = err.max(), mag.max()
    return (err / mag.clamp(min=1e-300)).max().item()


def _check_rel(name, got, ref, dims=None):
    assert torch.isfinite(got).all(), name
    worst = _rel(got, ref, dims)
    _note(name, worst)
    assert worst <= BAR[name], (name, worst)


def _check_bound(name, got, ref, bound):
    """max |got - ref| / bound <= 1 elementwise"""
    assert torch.isfinite(got).all(), name
    err = (got.double() - ref).abs()
    worst = (err / bound.clamp(min=1e-300)).max().item() if err.numel() else 0.0
    _note(name, worst)
    assert worst <= 1.0, (name, worst)


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------
# words_pairs
# ---------------------------------------------------------------------------------------------------
def _wp_inputs(B, NC, ndf, T, S, kind, seed):
    """words (NC, ndf, T) with NaN past each caption's length, ctx (B, ndf, S), lens (NC,) int64 on the device"""
    gen = _gen(seed)
    lens = [1 + (i * 5 + seed) % T for i in range(NC)]
    lens[0] = T
    if NC >= 3:
        lens[1] = 1
    lens[-1] = T + 3                                       # above T: the kernel reads the first T words
    words = torch.randn(NC, ndf, T, device=DEV, generator=gen) * 0.1
    for i, n in enumerate(lens):
        words[i, :, n:] = float("nan")
    ctx = torch.randn(B, ndf, S, device=DEV, generator=gen)
    if kind == "zero":
        words[0, :, 2] = 0.0                               # a word with |q| = 0
        ctx[1] = 0.0                                       # an image whose contexts are all 0
    return words.contiguous(), ctx.contiguous(), torch.tensor(lens, device=DEV, dtype=torch.int64), lens


def _wp_ref(words, ctx64, lens, T):
    """float64 func_attention + cosine + Eq. (10) of every (image, caption) pair: sim (B, NC), wc (B, NC, ndf, T) and
    attn (B, NC, T, S), NaN past each caption's length"""
    B, ndf, S = ctx64.shape
    NC = words.shape[0]
    sims = []
    wc = torch.full((B, NC, ndf, T), float("nan"), device=DEV, dtype=F64)
    attn = torch.full((B, NC, T, S), float("nan"), device=DEV, dtype=F64)
    for i in range(NC):
        n = min(lens[i], T)
        q = words[i, :, :n].double()[None].expand(B, ndf, n)
        a = torch.bmm(ctx64.transpose(1, 2), q)                       # (B, S, n)
        a = F.softmax(a, dim=2).transpose(1, 2) * GAMMA1               # softmax over the words
        a = F.softmax(a, dim=2)                                        # (B, n, S): softmax over the regions
        w = torch.bmm(ctx64, a.transpose(1, 2))                        # (B, ndf, n)
        w12 = (q * w).sum(1)
        nrm = torch.linalg.vector_norm(q, dim=1) * torch.linalg.vector_norm(w, dim=1)
        cos = w12 / nrm.clamp(min=EPS)
        sims.append(torch.log(torch.exp(cos * GAMMA2).sum(1)))
        wc[:, i, :, :n] = w.detach()
        attn[:, i, :n] = a.detach()
    return torch.stack(sims, 1), wc, attn


def _live(lens, T):
    return torch.arange(T, device=DEV)[None, :] < torch.tensor([min(n, T) for n in lens], device=DEV)[:, None]


def _run_wp_fwd(B, NC, ndf, T, S, kind, seed=0):
    words, ctx, lens_dev, lens = _wp_inputs(B, NC, ndf, T, S, kind, seed)
    outs = []
    for _ in range(2):
        wc = torch.full((B * NC, ndf, T), float("nan"), device=DEV)
        attn = torch.full((B * NC, T, S), float("nan"), device=DEV)
        sim = torch.full((B, NC), float("nan"), device=DEV)
        _call(WP_FWD, words, ctx, lens_dev, B, NC, ndf, T, S, GAMMA1, GAMMA2, EPS, wc, attn, sim)
        outs.append((wc, attn, sim))
    (wc, attn, sim), again = outs[0], outs[1]
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(outs[0], again)), "forward not deterministic"
    with torch.no_grad():
        sim_r, wc_r, attn_r = _wp_ref(words, ctx.double(), lens, T)
    _check_rel("words_pairs sim", sim, sim_r)
    live = _live(lens, T)                                               # (NC, T)
    wc, attn = wc.view(B, NC, ndf, T), attn.view(B, NC, T, S)
    lw = live[None, :, None, :].expand_as(wc)
    la = live[None, :, :, None].expand_as(attn)
    _check_rel("words_pairs wc", wc[lw], wc_r[lw])
    _check_rel("words_pairs attn", attn[la], attn_r[la])
    assert torch.isnan(wc[~lw]).all() and torch.isnan(attn[~la]).all(), "rows past a caption's length were written"


def _run_wp_bwd(B, NC, ndf, T, S, kind, seed=0):
    words, ctx, lens_dev, lens = _wp_inputs(B, NC, ndf, T, S, kind, seed)
    wc = torch.full((B * NC, ndf, T), float("nan"), device=DEV)
    attn = torch.full((B * NC, T, S), float("nan"), device=DEV)
    sim = torch.empty((B, NC), device=DEV)
    _call(WP_FWD, words, ctx, lens_dev, B, NC, ndf, T, S, GAMMA1, GAMMA2, EPS, wc, attn, sim)
    g_sim = torch.randn(B, NC, device=DEV, generator=_gen(seed + 1))
    g_ctx = torch.full((B, ndf, S), float("nan"), device=DEV)
    _call(WP_BWD, words, ctx, lens_dev, wc, attn, g_sim, B, NC, ndf, T, S, GAMMA1, GAMMA2, EPS, g_ctx)
    ctx64 = ctx.double().requires_grad_(True)
    sim_r = _wp_ref(words, ctx64, lens, T)[0]
    ref = torch.autograd.grad((sim_r * g_sim.double()).sum(), ctx64)[0]
    _check_rel("words_pairs g_ctx", g_ctx, ref, dims=1)                # per image


# ---------------------------------------------------------------------------------------------------
# cosine_matrix
# ---------------------------------------------------------------------------------------------------
def _cos_inputs(Ba, Bb, D, kind, seed):
    gen = _gen(seed)
    a = torch.randn(Ba, D, device=DEV, generator=gen)
    b = torch.randn(Bb, D, device=DEV, generator=gen) * 0.5
    if kind == "zero":
        a[1] = 0.0
        b[2] = 0.0
    return a.contiguous(), b.contiguous()


def _cos_ref(a64, b64):
    nrm = torch.linalg.vector_norm(a64, dim=1)[:, None] * torch.linalg.vector_norm(b64, dim=1)[None, :]
    return (a64 @ b64.T) / nrm.clamp(min=EPS)


def _run_cos_fwd(Ba, Bb, D, kind, seed=0):
    a, b = _cos_inputs(Ba, Bb, D, kind, seed)
    out = torch.full((Ba, Bb), float("nan"), device=DEV)
    _call(COS_FWD, a, b, Ba, Bb, D, EPS, out)
    _check_rel("cosine_matrix out", out, _cos_ref(a.double(), b.double()))


def _run_cos_bwd(Ba, Bb, D, kind, seed=0):
    a, b = _cos_inputs(Ba, Bb, D, kind, seed)
    g = torch.randn(Ba, Bb, device=DEV, generator=_gen(seed + 1))
    ga = torch.full((Ba, D), float("nan"), device=DEV)
    _call(COS_BWD, a, b, g, Ba, Bb, D, EPS, ga)
    a64 = a.double().requires_grad_(True)
    ref = torch.autograd.grad((_cos_ref(a64, b.double()) * g.double()).sum(), a64)[0]
    _check_rel("cosine_matrix ga", ga, ref, dims=1)                     # per row


# ---------------------------------------------------------------------------------------------------
# ce_pair
# ---------------------------------------------------------------------------------------------------
def _ce_inputs(B, mask_kind, labels_kind, tie, seed):
    """sim (B, B) on a grid of distinct values, labels, mask (uint8 or None) and the tie cells (kept unmasked)"""
    g = torch.Generator().manual_seed(seed)
    sim = (torch.randperm(B * B, generator=g).double() * (2.0 / (B * B)) - 1.0).float().view(B, B)
    labels = torch.randperm(B, generator=g) if labels_kind == "perm" else torch.arange(B)
    keep = [(i, int(labels[i])) for i in range(B)] + [(int(labels[i]), i) for i in range(B)]
    if tie:
        # row t: its maximum at the label column j1 and again at a later column j2
        t = next(i for i in range(B) if labels[i] < B - 2)
        j1 = int(labels[t])
        j2 = B - 1
        sim[t, j1] = sim[t, j2] = 1.5
        # column u: its maximum at the label row r1 and again at a later row r2 (cells apart from row t's)
        u = next(i for i in range(B) if i not in (j1, j2) and labels[i] < B - 2 and int(labels[i]) != t)
        r1 = int(labels[u])
        r2 = next(r for r in range(B - 1, r1, -1) if r != t)
        sim[r1, u] = sim[r2, u] = 1.25
        keep += [(t, j1), (t, j2), (r1, u), (r2, u)]
    mask = None
    if mask_kind == "zero":
        mask = torch.zeros(B, B, dtype=torch.uint8)
    elif mask_kind == "class":
        ids = (torch.arange(B) * 7 % max(B // 3, 1)).numpy()            # about three samples per class
        m = (ids.reshape(-1, 1) == ids.reshape(1, -1)).astype(np.uint8)
        np.fill_diagonal(m, 0)                                          # losses._class_masks
        mask = torch.from_numpy(m)
        for i, j in keep:                                               # never mask a label or a tie cell
            mask[i, j] = 0
        assert mask.sum() > 0
    dev = lambda t: None if t is None else t.to(DEV).contiguous()      # noqa: E731
    return dev(sim), dev(mask), dev(labels)


def _first_max(s):
    """index of the first maximum of each row"""
    idx = torch.arange(s.shape[1], device=s.device).expand_as(s)
    return torch.where(s == s.amax(1, keepdim=True), idx, s.shape[1]).amin(1)


def _run_ce(B, mask_kind, labels_kind, tie, seed=0):
    sim, mask, labels = _ce_inputs(B, mask_kind, labels_kind, tie, seed)
    out = torch.full((3,), float("nan"), device=DEV)
    G0, G1 = (torch.full((B, B), float("nan"), device=DEV) for _ in range(2))
    _call(CE, sim, mask, labels, B, GAMMA3, out[0:1], out[1:2], G0, G1, out[2:3])
    s64 = sim.double().requires_grad_(True)
    sc = s64 * GAMMA3
    if mask is not None:
        sc = sc.masked_fill(mask.bool(), -float("inf"))
    l0 = F.cross_entropy(sc, labels)
    l1 = F.cross_entropy(sc.T, labels)
    G0r = torch.autograd.grad(l0, s64, retain_graph=True)[0]
    G1r = torch.autograd.grad(l1, s64)[0]
    _check_rel("ce_pair loss", out[0:2], torch.stack((l0, l1)).detach())
    _check_rel("ce_pair G", G0, G0r)
    _check_rel("ce_pair G", G1, G1r)
    hits = (_first_max(sc.detach()) == labels).sum() + (_first_max(sc.detach().T) == labels).sum()
    assert out[2].item() == float(hits.item()), (out[2].item(), hits.item())


def _run_ce_bwd(n, g0_on, g1_on, seed=0):
    gen = _gen(seed)
    G0, G1 = torch.randn(n, device=DEV, generator=gen), torch.randn(n, device=DEV, generator=gen)
    g0 = torch.randn((), device=DEV, generator=gen) * 100 if g0_on else None
    g1 = torch.randn((), device=DEV, generator=gen) * 100 if g1_on else None
    gsim = torch.full((n,), float("nan"), device=DEV)
    _call(CE_BWD, G0, G1, g0, g1, n, gsim)
    t0 = g0.double() * G0.double() if g0_on else torch.zeros(n, device=DEV, dtype=F64)
    t1 = g1.double() * G1.double() if g1_on else torch.zeros(n, device=DEV, dtype=F64)
    _check_bound("ce_pair_bwd (error / bound)", gsim, t0 + t1, 2.0 ** -23 * (t0.abs() + t1.abs()) + 2.0 ** -149)


# ---------------------------------------------------------------------------------------------------
# the encoder's backward gathers
# ---------------------------------------------------------------------------------------------------
def _bl_weights(IS, OS):
    """(OS, IS) float64 weights of og_bilinear_fwd's align_corners=True resize, from its fp32 coordinates"""
    r = np.float32(IS - 1) / np.float32(OS - 1) if OS > 1 else np.float32(0.0)
    o = np.arange(OS, dtype=np.float32)
    f = (r * o).astype(np.float32)
    a = f.astype(np.int64)
    b = a + (a < IS - 1)
    lam = (f - a.astype(np.float32)).astype(np.float64)
    w = np.zeros((OS, IS))
    np.add.at(w, (np.arange(OS), a), 1.0 - lam)
    np.add.at(w, (np.arange(OS), b), lam)
    return torch.from_numpy(w).to(DEV)


def _run_bl_bwd(N, IH, IW, C, OH, OW, seed=0):
    g = torch.randn(N, OH, OW, C, device=DEV, generator=_gen(seed))
    gx = torch.full((N, IH, IW, C), float("nan"), device=DEV)
    _call(BL_BWD, g, N, IH, IW, C, OH, OW, gx)
    wh, ww = _bl_weights(IH, OH), _bl_weights(IW, OW)
    g64 = g.double()
    ref = torch.einsum("oi,pj,nopc->nijc", wh, ww, g64)
    bound = 2.0 ** -21 * torch.einsum("oi,pj,nopc->nijc", wh.abs(), ww.abs(), g64.abs())
    _check_bound("bilinear_bwd_gather (error / bound)", gx, ref, bound + 2.0 ** -149)


def _run_gap_bwd(N, P, C, seed=0):
    g = torch.randn(N, C, device=DEV, generator=_gen(seed))
    gx = torch.full((N, P, C), float("nan"), device=DEV)
    _call(GAP_BWD, g, N, P, C, gx)
    want = (g.double() / P).float()            # the correctly rounded fp32 quotient (53 >= 2 * 24 + 2 bits)
    assert torch.equal(_bits(gx), _bits(want[:, None, :].expand(N, P, C)))
    _note("global_avg_bwd (bitwise)", 0.0)


def _run_relu_slice(ldy, yoff, ldg, goff, ldo, ooff, nch, P, relu, seed=0):
    gen = _gen(seed)
    y = torch.randn(P, ldy, device=DEV, generator=gen)
    y.view(-1)[0::7] = 0.0
    y.view(-1)[3::7] = -0.0
    g = torch.randn(P, ldg, device=DEV, generator=gen)
    g.view(-1)[5::11] = -0.0
    out = torch.full((P, ldo), SENTINEL, device=DEV)
    _call(RELU_SLICE, y, ldy, yoff, g, ldg, goff, out, ldo, ooff, nch, P, relu)
    gs = g[:, goff:goff + nch]
    want = torch.where(y[:, yoff:yoff + nch] > 0, gs, torch.zeros_like(gs)) if relu else gs
    assert torch.equal(_bits(out[:, ooff:ooff + nch]), _bits(want))
    assert (out[:, :ooff] == SENTINEL).all() and (out[:, ooff + nch:] == SENTINEL).all()
    _note("relu_grad_slice (bitwise)", 0.0)


RUN = {WP_FWD: _run_wp_fwd, WP_BWD: _run_wp_bwd, COS_FWD: _run_cos_fwd, COS_BWD: _run_cos_bwd, CE: _run_ce,
       CE_BWD: _run_ce_bwd, BL_BWD: _run_bl_bwd, GAP_BWD: _run_gap_bwd, RELU_SLICE: _run_relu_slice}
ROWS = [(e, r) for table in (CASES, EDGE_CASES) for e in ENTRIES for r in table[e]]


@pytest.mark.parametrize("entry,row", ROWS, ids=[f"{e}-" + "-".join(map(str, r)) for e, r in ROWS])
def test_damsm_against_float64(entry, row):
    RUN[entry](*row)
    torch.cuda.synchronize()


@pytest.mark.parametrize("entry,row", REFUSED, ids=[f"{e}-" + "-".join(map(str, r)) for e, r in REFUSED])
def test_damsm_refuses(entry, row):
    """Argument checks: the call raises and writes nothing (the buffers are sized for the refused shape, so not even
    a missing check could reach outside them)."""
    if entry == CE:
        B = row[0]
        n = max(B, 1)
        sim = torch.zeros(n, n, device=DEV)
        labels = torch.zeros(n, device=DEV, dtype=torch.int64)
        out = torch.full((3,), SENTINEL, device=DEV)
        G = torch.full((2, n, n), SENTINEL, device=DEV)
        with pytest.raises(RuntimeError):
            _call(CE, sim, None, labels, B, GAMMA3, out[0:1], out[1:2], G[0], G[1], out[2:3])
        torch.cuda.synchronize()
        assert (out == SENTINEL).all() and (G == SENTINEL).all()
        return
    B, NC, ndf, T, S = row
    words = torch.zeros(NC, ndf, T, device=DEV)
    ctx = torch.zeros(B, ndf, S, device=DEV)
    lens = torch.full((NC,), T, device=DEV, dtype=torch.int64)
    wc = torch.full((B * NC, ndf, T), SENTINEL, device=DEV)
    attn = torch.full((B * NC, T, S), SENTINEL, device=DEV)
    sim = torch.full((B, NC), SENTINEL, device=DEV)
    g_ctx = torch.full((B, ndf, S), SENTINEL, device=DEV)
    with pytest.raises(RuntimeError):
        if entry == WP_FWD:
            _call(WP_FWD, words, ctx, lens, B, NC, ndf, T, S, GAMMA1, GAMMA2, EPS, wc, attn, sim)
        else:
            _call(WP_BWD, words, ctx, lens, wc, attn, sim, B, NC, ndf, T, S, GAMMA1, GAMMA2, EPS, g_ctx)
    torch.cuda.synchronize()
    for t in (wc, attn, sim, g_ctx):
        assert (t == SENTINEL).all()
