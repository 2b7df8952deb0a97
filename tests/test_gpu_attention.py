"""The attention, mask-paint and word-projection kernels (csrc/attention.cu, csrc/attention_tc.cu) against a float64
restatement of their math, at every shape the networks run them (tests/attention_cases.py: CASES) and at rows that pin
each dispatch branch (EDGE_CASES).  Every row goes through the public C ABI.

The reference is computed on the device in float64 from the same fp32 inputs the kernels get, including the
reference's mask-row quirk (grid attention: query (b, q) uses the caption mask of sample (b Q + q) mod B; bottom-up
attention: roi (b, r) uses sample (b R + r) mod B) and the paint backward's rule that the gradient goes to the first
maximal roi.  It is NOT the CPU fp32 oracle.

Bounds.  No fixed relative tolerance: every output element gets its own bound, built from the absolute values of the
operands, and the check is max |got - ref| / bound <= 1.  A K-term product sum sum_k a_k b_k is held to
    k u sum_k |a_k| |b_k|   (+ the scaling floors below, tensor-core rows only)
  Tensor cores: u = 2^-22, k = 8.  Each operand is split into an fp16 pair hi + lo of 22 significant bits
  (representation error 2^-22 |x|), the dropped lo * lo term is below 2^-22 |a| |b|, and the accumulation adds fp32
  roundings (2^-24 each, i.e. 1/4 in units of u).  k = 8 covers those: bound 2^-19 relative to sum |a| |b|.
  SIMT: u = 2^-24, k = 16.  The error is the fp32 roundings of sequential FMA chains of K <= 256 terms; they have both
  signs on these inputs and add like a random walk, sqrt(K) <= 16 (the worst case (K - 1) u, all roundings one way, is
  not reached).  Bound 2^-20 relative to sum |a| |b|.
  The tensor-core kernels scale each operand by a power of two before the split, so that its amax lands in
  [2^13, 2^14); a value far below that amax loses bits to fp16 subnormals (spacing 2^-24 after scaling), an absolute
  error of at most 2^-37 amax per operand (FLOOR).  The amax is taken per WARP (32 query rows) for h in the forward,
  per CTA tile (128 query rows) for g_wc, h and gS in the backward, per image for the word projections; the
  probabilities enter at the fixed scale 2^13, so their floor is 2^-24 2^-13 = 2^-37 absolute (PFLOOR).
The softmax carries the score errors ds_l through: |dp_l| <= p_l (e_l + sum_l' p_l' e_l'), e_l = ds_l plus its own
  fp32 rounding 2^-24 (L + 8 + 2 |s_l - max s|) (exp of a rounded argument, the L-term sum, the reciprocal, the scale).
The softmax backward carries the gP errors the same way: gS_l = P_l (gP_l - sum P gP), so
  |dgS_l| <= P_l (dgP_l + sum_l' P_l' dgP_l') + (L + 3) 2^-24 P_l (|gP|_l + sum P |gP|)  (|gP| the absolute-value sum).
Outputs computed from an already-checked kernel output (the context from the kernel's own probabilities) are held to
the bound of that one step, which isolates each MMA.  The mask paint forward is a max of fp32 products: it must equal
max_r (f m) computed in fp32 exactly.  Output lanes a kernel must not write are filled with a sentinel beforehand and
checked to be unchanged; lanes it must zero, checked to be 0.

Inputs: rows of h and g_wc whose magnitudes spread over 2^-7 .. 2^3 inside every warp and tile, one row per tile
2^-27 below its warp's max (its lo copy is subnormal), one warp-aligned block of 32 all-zero h rows (its scores are 0:
the probabilities must be exactly uniform over the unmasked words), ragged caption masks, NaN in the pad lanes of the
inputs (never read) and in the unused roi slots of the paint masks.

Determinism: the tensor-core forward, every grid-attention backward (per-CTA g_src planes added in a fixed order) and
the paint backward (per-block planes) are called twice on the same inputs and must agree bit for bit.
"""
import pytest
import torch

from attention_cases import (BU_BWD, BU_FWD, BWD, CASES, EDGE_CASES, ENTRIES, FWD, PAINT_BWD, PAINT_FWD, PROJ,
                             PROJ_BWD, batch_for)
from objgan_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
U32 = 2.0 ** -24             # fp32 rounding
KU_TC, KU_SIMT = 8 * 2.0 ** -22, 16 * 2.0 ** -24   # k u of a product sum (see above)
FLOOR = 2.0 ** -37          # per operand, times its scaling amax
PFLOOR = 2.0 ** -37         # probabilities (fixed scale 2^13), absolute
SENTINEL = 777.0
EPS_BU = 1e-8
WORST = {}                  # output -> worst observed error / bound, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"attention worst error/bound {k}: {WORST[k]:.3e}")


def _note(name, v):
    WORST[name] = max(WORST.get(name, 0.0), v)


def _call(name, *args):
    ops._call(name, *[ops._p(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _check(name, got, ref, bound):
    """max |got - ref| / bound <= 1 elementwise (bound 0: exact)"""
    assert torch.isfinite(got).all(), name
    err = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    worst = ratio.max().item() if ratio.numel() else 0.0
    _note(name, worst)
    assert worst <= 1.0, (name, worst)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rows_spread(B, Q, shift):
    """per-(image, query) magnitudes 2^-7 .. 2^3 varying inside every warp, one row per tile at 2^-27 below its warp"""
    q = torch.arange(Q, device=DEV)
    e = ((q[None, :] * 7 + torch.arange(B, device=DEV)[:, None] * 3 + shift) % 11) - 7
    e = torch.where((q % 128 == 37)[None, :], torch.full_like(e, -24), e)
    return torch.exp2(e.double()).float()


def _caption_mask(B, L, shift=0):
    """ragged caption masks (1 = padding word), at least one real word per caption"""
    lens = 1 + (torch.arange(B, device=DEV) * 5 + shift) % L
    lens[0] = L
    return (torch.arange(L, device=DEV)[None, :] >= lens[:, None]).to(torch.uint8).contiguous()


def _softmax_bound(p, s, ds, live, L):
    """|dp_l| <= p_l (e_l + sum p e), e_l = ds_l + 2^-24 (L + 8 + 2 |s_l - max s|), over the live words"""
    mx = torch.where(live, s, torch.full_like(s, -float("inf"))).amax(-1, keepdim=True)
    e = torch.where(live, ds + U32 * (L + 8 + 2 * (s - mx).abs()), torch.zeros_like(s))
    return p * (e + (p * e).sum(-1, keepdim=True)) + 2.0 ** -140


def _group_amax(x, group):
    """amax over groups of `group` consecutive queries (dim 1) and all channels, broadcast back to (B, Q, 1)"""
    B, Q = x.shape[:2]
    a = x.abs().amax(-1).view(B, Q // group, group).amax(-1)
    return a.repeat_interleave(group, 1)[..., None]


# ---------------------------------------------------------------------------------------------------
# grid attention
# ---------------------------------------------------------------------------------------------------
def _fwd_on_tc(B, Q, idf, cs, L):
    return Q >= 4096 and Q % 128 == 0 and idf == 48 and cs == 48 and 1 <= L <= 32 and B <= 128


def _bwd_on_tc(B, Q, idf, cs, L):
    return Q >= 4096 and Q % 128 == 0 and idf == 48 and cs == 48 and 1 <= L <= 32


def _att_inputs(B, Q, idf, cs, L, seed):
    gen = _gen(seed)
    h = torch.full((B, Q, cs), float("nan"), device=DEV)
    h[..., :idf] = torch.randn(B, Q, idf, device=DEV, generator=gen) * _rows_spread(B, Q, seed)[..., None]
    if Q >= 192:
        h[0, 160:192, :idf] = 0.0                       # warp 1 of tile 1: all-zero rows
    # word projections: channel magnitudes spread over 2^0 .. 2^-4
    src = torch.randn(B, idf, L, device=DEV, generator=gen) * 0.3
    src = src * torch.exp2(-(torch.arange(idf, device=DEV) % 5).float())[None, :, None]
    return h.contiguous(), src.contiguous()


def _mask_rows(mask, B, Q):
    """(B, Q, L) bool: the caption mask query (b, q) uses -- sample (b Q + q) mod B (GlobalAttention.py:108)"""
    idx = (torch.arange(B, device=DEV)[:, None] * Q + torch.arange(Q, device=DEV)[None, :]) % B
    return mask.bool()[idx]


def _run_fwd(B, Q, idf, cs, L, mask_on, seed=0):
    tc = _fwd_on_tc(B, Q, idf, cs, L)
    ku = KU_TC if tc else KU_SIMT
    h, src = _att_inputs(B, Q, idf, cs, L, seed)
    mask = _caption_mask(B, L, seed) if mask_on else None
    wc = torch.full((B, Q, cs), float("nan"), device=DEV)
    attn = torch.full((B, L, Q), float("nan"), device=DEV)
    _call(FWD, h, src, mask, B, Q, idf, cs, L, wc, attn)
    tag = "tc" if tc else "simt"

    # scores, probabilities
    h64, src64 = h[..., :idf].double(), src.double()
    s = torch.einsum("bqc,bcl->bql", h64, src64)
    sabs = torch.einsum("bqc,bcl->bql", h64.abs(), src64.abs())
    ds = ku * sabs
    if tc:
        ah = _group_amax(h64, 32)                                     # per-warp scale of h
        asrc = src64.abs().amax((1, 2))[:, None, None]                # per-image scale of src
        ds = ds + FLOOR * (ah * src64.abs().sum(1)[:, None, :] + asrc * h64.abs().sum(-1, keepdim=True))
    live = ~_mask_rows(mask, B, Q) if mask_on else torch.ones_like(s, dtype=torch.bool)
    p = torch.softmax(torch.where(live, s, torch.full_like(s, -float("inf"))), -1)
    got_p = attn.permute(0, 2, 1)
    _check(f"{FWD} attn ({tag})", got_p, p, _softmax_bound(p, s, ds, live, L))
    # the zero rows: scores 0, probabilities exactly uniform over the unmasked words
    if Q >= 192:
        z, zl = got_p[0, 160:192], live[0, 160:192]
        n = zl.sum(-1, keepdim=True)
        assert torch.equal(torch.where(zl, z, 0.0), torch.where(zl, (1.0 / n.float()).expand_as(z), 0.0))

    # context from the kernel's own probabilities: MMA 2 / the second SIMT sum
    pk = got_p.double()
    ref = torch.einsum("bql,bcl->bqc", pk, src64)
    bound = ku * torch.einsum("bql,bcl->bqc", pk, src64.abs())
    if tc:
        bound = bound + PFLOOR * src64.abs().sum(-1)[:, None, :] + FLOOR * asrc
    _check(f"{FWD} wc ({tag})", wc[..., :idf], ref, bound)
    assert (wc[..., idf:] == 0).all()
    if tc:
        wc2, attn2 = torch.empty_like(wc), torch.empty_like(attn)
        _call(FWD, h, src, mask, B, Q, idf, cs, L, wc2, attn2)
        assert torch.equal(wc, wc2) and torch.equal(attn, attn2)


def _run_bwd(B, Q, idf, cs, L, mask_on, seed=0):
    tc = _bwd_on_tc(B, Q, idf, cs, L)
    ku = KU_TC if tc else KU_SIMT
    tag = "tc" if tc else "simt"
    h, src = _att_inputs(B, Q, idf, cs, L, seed)
    gen = _gen(seed + 1)
    g_wc = torch.full((B, Q, cs), float("nan"), device=DEV)
    g_wc[..., :idf] = torch.randn(B, Q, idf, device=DEV, generator=gen) * _rows_spread(B, Q, seed + 5)[..., None]
    g_wc = g_wc.contiguous()
    # saved probabilities: a masked softmax of random scores (the kernel reads them as given)
    s = torch.randn(B, Q, L, device=DEV, generator=gen, dtype=F64) * 2
    if mask_on:
        s = torch.where(_mask_rows(_caption_mask(B, L, seed), B, Q), -float("inf"), s)
    P = torch.softmax(s, -1).float()
    attn = P.permute(0, 2, 1).contiguous()
    g_h = torch.full((B, Q, cs), float("nan"), device=DEV)
    g_src = torch.full((B, idf, L), float("nan"), device=DEV)
    _call(BWD, h, src, attn, g_wc, B, Q, idf, cs, L, g_h, g_src)

    h64, src64, gw64, P64 = h[..., :idf].double(), src.double(), g_wc[..., :idf].double(), P.double()
    asrc = src64.abs().amax((1, 2))[:, None, None]
    gP = torch.einsum("bqc,bcl->bql", gw64, src64)
    gP_abs = torch.einsum("bqc,bcl->bql", gw64.abs(), src64.abs())
    dgP = ku * gP_abs
    if tc:
        dgP = dgP + FLOOR * (_group_amax(gw64, 128) * src64.abs().sum(1)[:, None, :]
                             + asrc * gw64.abs().sum(-1, keepdim=True))
    gS = P64 * (gP - (P64 * gP).sum(-1, keepdim=True))
    gS_abs = P64 * (gP_abs + (P64 * gP_abs).sum(-1, keepdim=True))
    dgS = P64 * (dgP + (P64 * dgP).sum(-1, keepdim=True)) + (L + 3) * U32 * gS_abs

    # g_h = gS . src^T
    ref = torch.einsum("bql,bcl->bqc", gS, src64)
    bound = torch.einsum("bql,bcl->bqc", dgS, src64.abs()) + ku * torch.einsum("bql,bcl->bqc", gS_abs,
                                                                                          src64.abs())
    if tc:
        ags = gS_abs.amax(-1, keepdim=True).view(B, Q // 128, 128).amax(-1).repeat_interleave(128, 1)[..., None]
        bound = bound + FLOOR * (ags * src64.abs().sum(-1)[:, None, :] + asrc * gS_abs.sum(-1, keepdim=True))
    _check(f"{BWD} g_h ({tag})", g_h[..., :idf], ref, bound)
    assert (g_h[..., idf:] == 0).all()

    # g_src = g_wc^T . P + h^T . gS
    ref = torch.einsum("bqc,bql->bcl", gw64, P64) + torch.einsum("bqc,bql->bcl", h64, gS)
    bound = (torch.einsum("bqc,bql->bcl", h64.abs(), dgS)
             + ku * (torch.einsum("bqc,bql->bcl", gw64.abs(), P64)
                              + torch.einsum("bqc,bql->bcl", h64.abs(), gS_abs)))
    if tc:
        agw, ah = _group_amax(gw64, 128)[..., 0], _group_amax(h64, 128)[..., 0]
        ags = ags[..., 0]
        bound = bound + FLOOR * (torch.einsum("bq,bql->bl", agw, P64)[:, None, :]
                                 + torch.einsum("bq,bql->bl", ah, gS_abs)[:, None, :]
                                 + torch.einsum("bq,bqc->bc", ags, h64.abs())[..., None]) \
            + PFLOOR * gw64.abs().sum(1)[..., None]
    _check(f"{BWD} g_src ({tag})", g_src, ref, bound)
    g_h2, g_src2 = torch.empty_like(g_h), torch.empty_like(g_src)       # per-CTA planes added in a fixed order
    _call(BWD, h, src, attn, g_wc, B, Q, idf, cs, L, g_h2, g_src2)
    assert torch.equal(g_h, g_h2) and torch.equal(g_src, g_src2)


# ---------------------------------------------------------------------------------------------------
# bottom-up attention
# ---------------------------------------------------------------------------------------------------
def _run_bu_fwd(B, E, R, L, idf, norm, seed=0):
    gen = _gen(seed)
    labels = torch.randn(B, E, R, device=DEV, generator=gen)
    if R > 2:
        labels[0, :, R - 2:] = 0.0                      # padded roi slots: zero label vectors (norm 0 -> eps)
    glove = torch.randn(B, E, L, device=DEV, generator=gen) * 0.5
    src = torch.randn(B, idf, L, device=DEV, generator=gen) * 0.3
    mask = _caption_mask(B, L, seed + 3)
    wc = torch.full((B, idf, R), float("nan"), device=DEV)
    attn = torch.full((B, L, R), float("nan"), device=DEV)
    _call(BU_FWD, labels, glove, src, mask, B, E, R, L, idf, 1 if norm else 0, EPS_BU, wc, attn)

    lab64, gl64, src64 = labels.double(), glove.double(), src.double()
    S = torch.einsum("ber,bel->brl", lab64, gl64)
    dS = KU_SIMT * torch.einsum("ber,bel->brl", lab64.abs(), gl64.abs())
    if norm:
        # norms: E-term sums of squares and a square root each, their product: k u relative in all
        N = (lab64.norm(dim=1)[:, :, None] * gl64.norm(dim=1)[:, None, :]).clamp(min=EPS_BU)
        dS = (dS + KU_SIMT * S.abs()) / N
        S = S / N
    # mask row of roi (b, r): sample (b R + r) mod B (GlobalAttention.py:160)
    idx = (torch.arange(B, device=DEV)[:, None] * R + torch.arange(R, device=DEV)[None, :]) % B
    live = ~mask.bool()[idx]
    p = torch.softmax(torch.where(live, S, torch.full_like(S, -float("inf"))), -1)
    got_p = attn.permute(0, 2, 1)
    _check(f"{BU_FWD} attn", got_p, p, _softmax_bound(p, S, dS, live, L))
    pk = got_p.double()
    ref = torch.einsum("bcl,brl->bcr", src64, pk)
    _check(f"{BU_FWD} wc", wc, ref, KU_SIMT * torch.einsum("bcl,brl->bcr", src64.abs(), pk))


def _run_bu_bwd(B, _E, R, L, idf, _norm, seed=0):
    gen = _gen(seed)
    attn = torch.softmax(torch.randn(B, R, L, device=DEV, generator=gen) * 2, -1).permute(0, 2, 1).contiguous()
    g_wc = torch.randn(B, idf, R, device=DEV, generator=gen)
    g_src = torch.full((B, idf, L), float("nan"), device=DEV)
    _call(BU_BWD, attn, g_wc, B, R, L, idf, g_src)
    a64, g64 = attn.double(), g_wc.double()
    ref = torch.einsum("bcr,blr->bcl", g64, a64)
    _check(f"{BU_BWD} g_src", g_src, ref, KU_SIMT * torch.einsum("bcr,blr->bcl", g64.abs(), a64))


# ---------------------------------------------------------------------------------------------------
# mask paint
# ---------------------------------------------------------------------------------------------------
def _paint_inputs(B, num, R, Rtot, P, seed):
    """f: roi features (both signs); m: roi masks in [0, 1], zero outside the boxes, NaN in the unused slots R..Rtot.
    Ties: channels k even have f[k, 0] == f[k, 1] above every other roi, and masks 0 and 1 are equal (and nonzero) on
    every third pixel, so there the maximum is attained at r = 0 and r = 1."""
    gen = _gen(seed)
    f = torch.randn(B, num, R, device=DEV, generator=gen)
    m = torch.full((B, Rtot, P), float("nan"), device=DEV)
    mr = torch.rand(B, R, P, device=DEV, generator=gen)
    mr[mr < 0.4] = 0.0
    if R >= 2:
        f[:, 0::2, 0] = 3.0 + f[:, 0::2, 0].abs()
        f[:, 0::2, 1] = f[:, 0::2, 0]
        tie = torch.arange(P, device=DEV) % 3 == 0
        mr[:, 0, tie] = 0.5 + 0.5 * torch.rand(B, int(tie.sum()), device=DEV, generator=gen)
        mr[:, 1, tie] = mr[:, 0, tie]
    m[:, :R] = mr
    return f.contiguous(), m.contiguous()


def _paint_products(f, m, R):
    """(B, num, R, P) fp32 products f[b, k, r] * m[b, r, p]"""
    return f[:, :, :, None] * m[:, None, :R, :]


def _run_paint_fwd(B, num, R, Rtot, P, stride, off, seed=0):
    f, m = _paint_inputs(B, num, R, Rtot, P, seed)
    out = torch.full((B, P, stride), SENTINEL, device=DEV)
    _call(PAINT_FWD, f, m, B, num, R, Rtot, P, out, stride, off)
    ref = _paint_products(f, m, R).amax(2) if R > 0 else torch.zeros(B, num, P, device=DEV)
    assert torch.equal(out[..., off:off + num], ref.permute(0, 2, 1)), "paint forward != max_r f m in fp32"
    _note(f"{PAINT_FWD} (exact)", 0.0)
    # the vectorised kernel writes whole quads: lanes [num, 4 ceil(num / 4)) are zeroed; every other path and every
    # other lane leaves the row untouched
    nq4 = (num + 3) // 4
    vec = (R > 0 and stride % 4 == 0 and off % 4 == 0 and 4 * nq4 + off <= stride and nq4 <= 256
           and 4 * (R * 4 * nq4 + R * 128) <= 48 * 1024)
    pad = out[..., off + num:off + 4 * nq4]
    assert (pad == (0.0 if vec else SENTINEL)).all()
    rest = torch.cat((out[..., :off], out[..., off + 4 * nq4:]), -1)
    assert (rest == SENTINEL).all()


def _run_paint_bwd(B, num, R, Rtot, P, stride, off, seed=0):
    f, m = _paint_inputs(B, num, R, Rtot, P, seed)
    gen = _gen(seed + 1)
    g = torch.full((B, P, stride), float("nan"), device=DEV)
    g[..., off:off + num] = torch.randn(B, P, num, device=DEV, generator=gen)
    g = g.contiguous()
    g_f = torch.full((B, num, R), float("nan"), device=DEV)
    _call(PAINT_BWD, f, m, g, stride, off, B, num, R, Rtot, P, g_f)
    if R == 0:
        assert g_f.numel() == 0
        return
    prod = _paint_products(f, m, R)
    is_max = prod == prod.amax(2, keepdim=True)
    first = is_max & (is_max.cumsum(2) == 1)                              # the first maximal roi
    gk = g[..., off:off + num].permute(0, 2, 1).double()                  # (B, num, P)
    term = gk[:, :, None, :] * m[:, None, :R, :].double() * first         # (B, num, R, P)
    ref = term.sum(-1)
    _check(f"{PAINT_BWD} g_f", g_f, ref, KU_SIMT * term.abs().sum(-1))
    g_f2 = torch.empty_like(g_f)
    _call(PAINT_BWD, f, m, g, stride, off, B, num, R, Rtot, P, g_f2)
    assert torch.equal(g_f, g_f2)


# ---------------------------------------------------------------------------------------------------
# word projections
# ---------------------------------------------------------------------------------------------------
def _proj_inputs(B, idf, cdf, L, seed):
    gen = _gen(seed)
    words = torch.randn(B, cdf, L, device=DEV, generator=gen)
    W = torch.randn(idf, cdf, device=DEV, generator=gen) * 0.1
    return words, W


def _run_proj(B, idf, cdf, L, seed=0):
    words, W = _proj_inputs(B, idf, cdf, L, seed)
    src = torch.full((B, idf, L), float("nan"), device=DEV)
    _call(PROJ, words, W, B, idf, cdf, L, src)
    w64, W64 = words.double(), W.double()
    _check(f"{PROJ} src", src, torch.einsum("ck,bkl->bcl", W64, w64),
           KU_SIMT * torch.einsum("ck,bkl->bcl", W64.abs(), w64.abs()))


def _run_proj_bwd(B, idf, cdf, L, seed=0):
    words, W = _proj_inputs(B, idf, cdf, L, seed)
    gsrc = torch.randn(B, idf, L, device=DEV, generator=_gen(seed + 1))
    gW = torch.full((idf, cdf), float("nan"), device=DEV)
    gwords = torch.full((B, cdf, L), float("nan"), device=DEV)
    _call(PROJ_BWD, words, W, gsrc, B, idf, cdf, L, gW, 0, gwords)
    w64, W64, g64 = words.double(), W.double(), gsrc.double()
    _check(f"{PROJ_BWD} gW", gW, torch.einsum("bcl,bkl->ck", g64, w64),
           KU_SIMT * torch.einsum("bcl,bkl->ck", g64.abs(), w64.abs()))
    _check(f"{PROJ_BWD} gwords", gwords, torch.einsum("ck,bcl->bkl", W64, g64),
           KU_SIMT * torch.einsum("ck,bcl->bkl", W64.abs(), g64.abs()))


RUN = {FWD: _run_fwd, BWD: _run_bwd, BU_FWD: _run_bu_fwd, BU_BWD: _run_bu_bwd, PAINT_FWD: _run_paint_fwd,
       PAINT_BWD: _run_paint_bwd, PROJ: _run_proj, PROJ_BWD: _run_proj_bwd}
ROWS = [(e, r) for table in (CASES, EDGE_CASES) for e in ENTRIES for r in table[e]]


@pytest.mark.parametrize("entry,row", ROWS, ids=[f"{e}-" + "-".join(map(str, r)) for e, r in ROWS])
def test_attention_against_float64(entry, row):
    if entry in (FWD, BWD):
        row = (batch_for(row[0], row[1], _sms()),) + tuple(row[1:])
    RUN[entry](*row)
    torch.cuda.synchronize()
