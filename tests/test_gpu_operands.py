"""Every writer of the tensor-core operand format (csrc/operand.cuh) against a numpy restatement, bit for bit.

The format: x * 2^k as an fp16 pair hi = fp16(x * 2^k), lo = fp16(x * 2^k - hi), with k = og_scale_exp of a scale word
(the float bits of max|x|, or of an upper bound of it).  The writers are the activation splits (og_prep_split,
og_prep_split_s2d, og_norm_apply_split), the weight packers (og_pack_weights_f16, og_pack_upsample_weights and the
multi-job og_pack_weights_f16_multi), and the scale words (og_amax, og_amax_multi).  The restatement rounds like the
kernels: np.float16 of the fp32 product, np.float16 of the fp32 difference, upsample pre-sums in fp32 in kh-then-kw order.
"""
import numpy as np
import pytest
import torch

from objgan_b200 import ops
from objgan_b200.lib import NA_GLU, NA_LRELU, NA_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLOPE = 0.2


def _word():
    return torch.empty(1, device=DEV, dtype=torch.int32)


def _bits(f):
    return int(np.array([f], dtype=np.float32).view(np.uint32)[0])


def _set_word(t, f):
    t.copy_(torch.tensor([np.array([f], dtype=np.float32).view(np.int32)[0]], dtype=torch.int32))


def _get_word(t):
    return int(t.cpu().numpy().view(np.uint32)[0])


def _scale(word):
    word &= 0x7FFFFFFF
    if word == 0:
        return np.float32(1.0)
    k = min(110, max(-110, 13 - ((word >> 23) - 127)))
    return np.float32(2.0 ** k)


def _encode(v, word):
    v = np.asarray(v, dtype=np.float32) * _scale(word)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def _h16(t):
    return t.detach().cpu().numpy().view(np.uint16)


def _assert_pair(xh, xl, want):
    hi, lo = want
    np.testing.assert_array_equal(_h16(xh), hi.view(np.uint16))
    np.testing.assert_array_equal(_h16(xl), lo.view(np.uint16))


def _nan_f16(shape):
    return torch.full(shape, float("nan"), device=DEV, dtype=torch.float16)


def _amax_bits(a):
    return _bits(np.abs(np.asarray(a, dtype=np.float32)).max())


def _rand(shape, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


# ---------------------------------------------------------------------------------------------------------------
# activation splits
# ---------------------------------------------------------------------------------------------------------------
def _s2d_ref(x):
    """[4N][ceil(H/2)][ceil(W/2)][C]: phase block a*2+b = x[:, a::2, b::2], zero past an odd edge."""
    n, h, w, c = x.shape
    out = np.zeros((4, n, (h + 1) // 2, (w + 1) // 2, c), np.float32)
    for a in range(2):
        for b in range(2):
            blk = x[:, a::2, b::2]
            out[a * 2 + b, :, :blk.shape[1], :blk.shape[2]] = blk
    return out.reshape(4 * n, (h + 1) // 2, (w + 1) // 2, c)


@pytest.mark.parametrize("ready", [0, 1])
@pytest.mark.parametrize("mode", ["pad0", "pad1", "s2d"])
def test_prep_split_bits(mode, ready):
    """og_prep_split: the scale word it computes (amax_ready 0) is max|x|, the one it is given (amax_ready 1) is kept
    and used; hi / lo are the encoding of x, of its reflection halo, or of its four space-to-depth phase blocks."""
    n, h, w, c = 2, 6, 10, 16
    x = _rand((n, h, w, c), 11)
    xn = x.cpu().numpy()
    pad, s2d = (1 if mode == "pad1" else 0), (1 if mode == "s2d" else 0)
    if s2d:
        want = _s2d_ref(xn)
    else:
        want = np.pad(xn, ((0, 0), (pad, pad), (pad, pad), (0, 0)), mode="reflect")
    amax = _word()
    word = _amax_bits(xn)
    if ready:
        word = _bits(np.float32(5.5) * np.abs(xn).max())
        _set_word(amax, np.array([word], np.uint32).view(np.float32)[0])
    xh, xl = _nan_f16(want.shape), _nan_f16(want.shape)
    ops._call("og_prep_split", ops._p(x), n, h, w, c, pad, s2d, ops._p(amax), ready, ops._p(xh), ops._p(xl))
    assert _get_word(amax) == word
    _assert_pair(xh, xl, _encode(want, word))


@pytest.mark.parametrize("ready", [0, 1])
@pytest.mark.parametrize("shape", [(2, 6, 10, 16), (2, 7, 5, 8), (1, 6, 5, 16), (3, 9, 4, 8)], ids=str)
def test_prep_split_s2d_bits(shape, ready):
    """og_prep_split_s2d at even and odd H, W: the phase blocks on the ceil(H/2) x ceil(W/2) grid, zero past an odd
    edge.  At even sizes it writes the same bytes as og_prep_split(s2d=1)."""
    n, h, w, c = shape
    x = _rand(shape, 12)
    xn = x.cpu().numpy()
    want = _s2d_ref(xn)
    amax = _word()
    word = _amax_bits(xn)
    if ready:
        word = _bits(np.float32(0.75) * np.abs(xn).max())
        _set_word(amax, np.array([word], np.uint32).view(np.float32)[0])
    xh, xl = _nan_f16(want.shape), _nan_f16(want.shape)
    ops._call("og_prep_split_s2d", ops._p(x), n, h, w, c, ops._p(amax), ready, ops._p(xh), ops._p(xl))
    assert _get_word(amax) == word
    _assert_pair(xh, xl, _encode(want, word))
    if h % 2 == 0 and w % 2 == 0:
        a2 = _word()
        if ready:
            a2.copy_(amax)
        yh, yl = _nan_f16(want.shape), _nan_f16(want.shape)
        ops._call("og_prep_split", ops._p(x), n, h, w, c, 0, 1, ops._p(a2), ready, ops._p(yh), ops._p(yl))
        assert torch.equal(a2, amax)
        assert np.array_equal(_h16(yh), _h16(xh)) and np.array_equal(_h16(yl), _h16(xl))


@pytest.mark.parametrize("pad", [0, 1])
@pytest.mark.parametrize("act", [NA_NONE, NA_LRELU, NA_GLU], ids=["none", "lrelu", "glu"])
def test_norm_apply_split_bits(act, pad):
    """og_norm_apply_split: hi / lo are the encoding, with the bound word, of the fp32 output the kernel wrote (with its
    reflection halo when pad = 1).  InstanceNorm with a residual (none), BatchNorm affine (lrelu), InstanceNorm (glu)."""
    n, h, w = 2, 6, 5
    co = 16
    cy = 2 * co if act == NA_GLU else co
    instance = 0 if act == NA_LRELU else 1
    groups = n if instance else 1
    y = _rand((n, h, w, cy), 13, 1.0)
    mean = _rand((groups * cy,), 14, 0.1)
    rstd = (torch.rand(groups * cy, generator=torch.Generator().manual_seed(15)) + 0.5).to(DEV)
    gamma = beta = res = None
    if act == NA_LRELU:
        gamma = 1 + _rand((cy,), 16, 0.1)
        beta = _rand((cy,), 17, 0.1)
    if act == NA_NONE:
        res = _rand((n, h, w, co), 18, 1.0)
    bound = _word()
    _set_word(bound, 40.0)
    out = torch.full((n, h, w, co), float("nan"), device=DEV)
    shape = (n, h + 2 * pad, w + 2 * pad, co)
    xh, xl = _nan_f16(shape), _nan_f16(shape)
    ops._call("og_norm_apply_split", ops._p(y), n, h, w, cy, instance, ops._p(mean), ops._p(rstd), ops._p(gamma),
              ops._p(beta), ops._p(res), act, SLOPE, ops._p(out), ops._p(bound), pad, ops._p(xh), ops._p(xl))
    o = out.cpu().numpy()
    assert np.isfinite(o).all()
    want = np.pad(o, ((0, 0), (pad, pad), (pad, pad), (0, 0)), mode="reflect")
    _assert_pair(xh, xl, _encode(want, _bits(40.0)))


# ---------------------------------------------------------------------------------------------------------------
# weight packers and scale words
# ---------------------------------------------------------------------------------------------------------------
def _cm(co, split, splitp):
    return co if split == 0 or co < split else co + splitp - split


def _pack_ref(w, cip, kp, split, splitp, transposed):
    """[tap][ci][cm] (or [tap][cm][ci] transposed) fp32, GLU halves at cm = 0 and splitp, zero elsewhere."""
    co_n, ci_n, kh, kw = w.shape
    taps = kh * kw
    wt = w.reshape(co_n, ci_n, taps)
    out = np.zeros((taps, cip, kp), np.float32)
    for co in range(co_n):
        out[:, :ci_n, _cm(co, split, splitp)] = wt[co].T
    return out.transpose(0, 2, 1).copy() if transposed else out


PACKS = [  # (Co, Ci, KH, KW, Cip, Kp, split, splitp)
    (12, 5, 3, 3, 8, 16, 0, 0),
    (20, 9, 3, 3, 16, 32, 10, 16),
    (8, 8, 1, 1, 8, 8, 0, 0),
    (64, 48, 4, 4, 48, 64, 0, 0),
    (96, 40, 3, 3, 40, 96, 48, 48),
]


def _amax(t):
    a = _word()
    _set_word(a, np.float32(123.0))
    ops._call("og_amax", ops._p(t), t.numel(), ops._p(a))
    return a


@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("row", PACKS, ids=str)
def test_pack_weights_bits(row, transposed):
    """og_pack_weights_f16 (and the fp32 og_pack_weights it mirrors): the packed matrix in either layout, GLU halves
    moved to their padded positions, scaled by the og_amax word of the OIHW parameter."""
    co, ci, kh, kw, cip, kp, split, splitp = row
    w = _rand((co, ci, kh, kw), 21, 0.2)
    wn = w.cpu().numpy()
    want = _pack_ref(wn, cip, kp, split, splitp, transposed)
    a = _amax(w)
    assert _get_word(a) == _amax_bits(wn)
    hi, lo = _nan_f16(want.shape), _nan_f16(want.shape)
    ops._call("og_pack_weights_f16", ops._p(w), co, ci, kh, kw, cip, kp, split, splitp, transposed, ops._p(a),
              ops._p(hi), ops._p(lo))
    _assert_pair(hi, lo, _encode(want, _get_word(a)))
    f = torch.full(want.shape, float("nan"), device=DEV)
    ops._call("og_pack_weights", ops._p(w), co, ci, kh, kw, cip, kp, split, splitp, transposed, ops._p(f))
    np.testing.assert_array_equal(f.cpu().numpy().view(np.uint32), want.view(np.uint32))


def _up_row(p, k):
    return int(k >= 1) if p == 0 else int(k >= 2)


@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("row", [(12, 5, 8, 16, 0, 0), (20, 9, 16, 32, 10, 16)], ids=str)
def test_pack_upsample_weights_bits(row, transposed):
    """og_pack_upsample_weights: the 2x2 phase pre-sums (fp32, kh then kw) at their packed positions, scaled by the
    word 4 * amax(w) that it also writes to amax_up."""
    co_n, ci_n, cip, kp, split, splitp = row
    w = _rand((co_n, ci_n, 3, 3), 22, 0.2)
    wn = w.cpu().numpy()
    out = np.zeros((16, cip, kp), np.float32)
    for t in range(16):
        b, a, q, p = t & 1, (t >> 1) & 1, (t >> 2) & 1, (t >> 3) & 1
        v = np.zeros((co_n, ci_n), np.float32)
        for kh in range(3):
            if _up_row(p, kh) != a:
                continue
            for kw in range(3):
                if _up_row(q, kw) == b:
                    v = (v + wn[:, :, kh, kw]).astype(np.float32)
        for co in range(co_n):
            out[t, :ci_n, _cm(co, split, splitp)] = v[co]
    want = out.transpose(0, 2, 1).copy() if transposed else out
    a = _amax(w)
    up = _word()
    word = _bits(np.float32(4.0) * np.abs(wn).max())
    hi, lo = _nan_f16(want.shape), _nan_f16(want.shape)
    ops._call("og_pack_upsample_weights", ops._p(w), co_n, ci_n, cip, kp, split, splitp, transposed, ops._p(a),
              ops._p(up), ops._p(hi), ops._p(lo))
    assert _get_word(up) == word
    _assert_pair(hi, lo, _encode(want, word))


@pytest.mark.parametrize("n", [1, 3, 6, 1021, 300003])
def test_amax_bits(n):
    """og_amax at lengths that are not a multiple of 4: the float bits of max|x|, the maximum placed in the tail."""
    x = _rand((n,), 23, 1.0)
    x[n - 1] = -9.75
    assert _get_word(_amax(x)) == _bits(9.75)
    x[n - 1] = 0.0
    assert _get_word(_amax(x)) == _amax_bits(x.cpu().numpy())


def test_multi_tables_match_single_calls():
    """One og_amax_multi + og_pack_weights_f16_multi table over several layers, two layouts sharing one amax word:
    every word and hi / lo pair equals, bit for bit, the single-layer og_amax + og_pack_weights_f16 (and numpy)."""
    CH = 4096
    ws = [_rand(r[:4], 30 + i, 0.2) for i, r in enumerate(PACKS)]
    words = [_word() for _ in ws]
    for wd in words:
        _set_word(wd, np.float32(77.0))
    arows, prows, bufs, ab, pb = [], [], [], 0, 0
    for w, wd in zip(ws, words):
        arows.append([w.data_ptr(), w.numel(), wd.data_ptr(), ab])
        ab += (w.numel() + CH - 1) // CH
    for row, w, wd in zip(PACKS, ws, words):
        co, ci, kh, kw, cip, kp, split, splitp = row
        total = kh * kw * cip * kp
        for tr in (0, 1):
            hi, lo = _nan_f16((total,)), _nan_f16((total,))
            bufs.append((row, w, wd, tr, hi, lo))
            prows.append([w.data_ptr(), hi.data_ptr(), lo.data_ptr(), wd.data_ptr(), co, ci, kh * kw, cip, kp, split,
                          splitp, tr, total, pb])
            pb += (total + CH - 1) // CH
    at = torch.tensor(arows, dtype=torch.int64, device=DEV)
    pt = torch.tensor(prows, dtype=torch.int64, device=DEV)
    ops._call("og_amax_multi", ops._p(at), len(arows), ab)
    ops._call("og_pack_weights_f16_multi", ops._p(pt), len(prows), pb)
    for w, wd in zip(ws, words):
        assert torch.equal(_amax(w), wd)
        assert _get_word(wd) == _amax_bits(w.cpu().numpy())
    for row, w, wd, tr, hi, lo in bufs:
        co, ci, kh, kw, cip, kp, split, splitp = row
        h2, l2 = _nan_f16(hi.shape), _nan_f16(lo.shape)
        ops._call("og_pack_weights_f16", ops._p(w), co, ci, kh, kw, cip, kp, split, splitp, tr, ops._p(wd),
                  ops._p(h2), ops._p(l2))
        assert np.array_equal(_h16(h2), _h16(hi)) and np.array_equal(_h16(l2), _h16(lo))
        want = _pack_ref(w.cpu().numpy(), cip, kp, split, splitp, tr).reshape(-1)
        _assert_pair(hi, lo, _encode(want, _get_word(wd)))
