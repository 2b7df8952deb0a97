"""GPU tests of the row-run forward kernel (conv_tc_rows_kernel in conv_tc.cu).

A tap list that splits into runs of taps differing only in dh (the column-by-column order of conv2d's 3x3 stride-1
layers) takes conv_tc_rows_kernel, which loads one haloed A box per run instead of one A tile per tap.  Its consumers
walk the stages, partial sums and order of conv_tc_kernel, so its outputs must be bitwise those of conv_tc_kernel.

The conv_tc_kernel reference comes from the same library: the source is passed stacked twice (SN = 2N, the two
copies identical) and dn alternates between 0 and N along each run.  Every tap reads the same values in the same
order, but no run qualifies, so og_conv2d_tc launches conv_tc_kernel.  Both are also checked against float64 at the
1e-4 of max|out| bound of test_gpu_tc.py."""
import pytest
import torch
import torch.nn.functional as F

from conv_cases import CASES, EDGE_CASES
from objgan_b200 import ops
from objgan_b200.lib import ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, PAD_REFLECT, UPSAMPLE2X

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _layer_rows():
    """The 3x3 stride-1 tensor-core rows of conv_cases whose taps run column by column (no upsampling), deduplicated
    on what a launch sees."""
    seen, out = set(), []
    for r in CASES + EDGE_CASES:
        n, h, w, cin, cout, k, stride, pad, mode, act, bias, split, path = r
        if path != "s1" or k != 3 or mode == UPSAMPLE2X:
            continue
        key = (n, h, w, cin, cout, mode, act, bias, split)
        if key not in seen:
            seen.add(key)
            out.append(r)
    return out


def _kp(cout, split):
    return 2 * ops.cpad(split) if split else ops.cpad(cout)


def _launch(d, r):
    """_Problem arguments (oh, ow, taps, source channels, source h, w, reflection halo of the source copy, output
    channels, bias, act) of direction d of the row r."""
    n, h, w, cin, cout, k, stride, pad, mode, act, bias, split, _ = r
    plan = ops._tc_plan(d, *ops._conv2d_geo(n, h, w, k, k, stride, pad, mode))
    taps, oh, ow, _, _, _ = plan.launches[0]
    c, kp = ops.cpad(cin), _kp(cout, split)
    if d == ops.FPROP:
        return oh, ow, taps, c, h, w, plan.xsplit[0], kp, bias, act
    return oh, ow, taps, kp, h, w, 0, c, False, ACT_NONE


# hand-picked geometry: partial last tiles in h and w, the last chunk 1..4 k-steps deep (C = 200 / 88 / 104 / 128),
# one to four chunks, stacked tiles (<= 32 output channels), N tiles of 48 / 104 / 128 columns, TW = 8 patches, the
# fullest shared memory (4 slots of 40 KB + 2 B stages of 32 KB) and the descending run order of an input gradient.
# These maps have few output tiles: without a bias or an activation og_conv2d_tc would split their reduction, which
# the row-run kernel does not take, so every row has one (_check asserts the kernel each form launched).
EDGES = [
    # taps, n, h, w, c, halo, k, bias, act
    ("fprop", 2, 20, 36, 200, 1, 400, True, ACT_NONE),       # 4 chunks, klast 1, BN 104, partial tiles in h and w
    ("fprop", 2, 24, 40, 88, 0, 48, True, ACT_LRELU),        # 2 chunks, klast 2, BN 48
    ("fprop", 3, 16, 24, 104, 1, 128, True, ACT_NONE),       # 2 chunks, klast 3, BN 128
    ("fprop", 2, 32, 32, 128, 0, 256, True, ACT_TANH),       # 2 chunks, klast 4, BN 128
    ("fprop", 2, 40, 8, 192, 0, 104, False, ACT_LRELU),      # 3 chunks, TW = 8, TH = 16
    ("fprop", 2, 30, 30, 256, 0, 128, True, ACT_NONE),       # 4 chunks, BN 128 (2 B stages)
    ("fprop", 2, 24, 24, 48, 1, 12, True, ACT_NONE),         # stacked, 16 rows
    ("fprop", 2, 24, 24, 80, 0, 24, True, ACT_SIGMOID),      # stacked, 32 rows
    ("dgrad", 2, 20, 36, 200, 1, 200, True, ACT_NONE),       # descending runs, 4 chunks
    ("dgrad", 3, 16, 16, 8, 0, 48, False, ACT_NONE),         # descending runs, 1 chunk of one k-step
]


def _taps(d, halo):
    """conv2d's 3x3 tap order (ops._tc_plan, cols=True) for a source with `halo` rows and columns of padding."""
    geo = (1, 8, 8, 3, 3, 1, 1, 1, PAD_REFLECT if halo else 0, True)
    (taps, *_), = ops._tc_plan(ops.FPROP if d == "fprop" else ops.DGRAD, *geo).launches
    return taps


def _apply(v, act):
    if act == ACT_LRELU:
        return F.leaky_relu(v, ops.LRELU_SLOPE)
    if act == ACT_TANH:
        return torch.tanh(v)
    if act == ACT_SIGMOID:
        return torch.sigmoid(v)
    return v


class _Problem:
    """Random source and packed weights of one og_conv2d_tc launch over an (sh, sw) source (copied with a reflection
    halo of `halo` pixels); runs it as given and in the reference form."""

    def __init__(self, n, oh, ow, taps, c, sh, sw, halo, k, bias, act, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.n, self.oh, self.ow, self.taps, self.k, self.act = n, oh, ow, tuple(taps), k, act
        x = torch.randn(n, sh, sw, c, generator=g, device=DEV)
        self.src = F.pad(x.permute(0, 3, 1, 2), (halo,) * 4, mode="reflect").permute(0, 2, 3, 1) if halo else x
        self.w = torch.randn(9, k, 1, c, generator=g, device=DEV) * 0.05
        self.bias = torch.randn(k, generator=g, device=DEV) * 0.1 if bias else None
        self.xs = ops._split(x, halo)
        self.ws = ops._split(self.w)

    def run(self, reference):
        xh, xl, ax = self.xs
        taps = self.taps
        if reference:
            xh, xl = torch.cat((xh, xh)), torch.cat((xl, xl))
            taps = tuple((dh, dw, dn + (i % 2) * self.n, t) for i, (dh, dw, dn, t) in enumerate(taps))
        y = torch.full((self.n, self.oh, self.ow, self.k), float("nan"), device=DEV)
        plan = ops._Plan(None, None, False, 9, (self.oh, self.ow), ((taps, self.oh, self.ow, 1, 0, 0),))
        ops._tc_launch((xh, xl, ax), self.n, self.ws, plan, y, self.k, self.bias, self.act)
        torch.cuda.synchronize()
        return y

    def float64(self):
        """out[n, h, w] = act(sum_t src[n + dn, h + dh, w + dw] W[t]^T + b), out-of-range source pixels zero."""
        src = self.src.double()
        p = 3
        srcp = F.pad(src, (0, 0, p, p, p, p))
        out = torch.zeros(self.n, self.oh, self.ow, self.k, device=DEV, dtype=torch.float64)
        w = self.w.double()[:, :, 0, :]
        for dh, dw, dn, t in self.taps:
            s = srcp[dn:dn + self.n, p + dh:p + dh + self.oh, p + dw:p + dw + self.ow]
            out += torch.einsum("nhwc,kc->nhwk", s, w[t])
        if self.bias is not None:
            out += self.bias.double()
        return _apply(out, self.act)


def _check(prob, rows=None):
    """prob's launch bitwise equal to its conv_tc_kernel form, and within 1e-4 of max|out| of float64.  rows = True:
    also assert from profiler traces that the launch took conv_tc_rows_kernel and the reference conv_tc_kernel."""
    out = {}
    if rows:
        k_got = _kernels_launched(lambda: out.setdefault("got", prob.run(False)))
        k_ref = _kernels_launched(lambda: out.setdefault("ref", prob.run(True)))
        assert len(k_got) == 1 and "conv_tc_rows_kernel" in next(iter(k_got)), k_got
        assert len(k_ref) == 1 and "conv_tc_rows_kernel" not in next(iter(k_ref)), k_ref
    got, ref = out.get("got"), out.get("ref")
    if got is None:
        got, ref = prob.run(False), prob.run(True)
    assert torch.isfinite(got).all()
    assert torch.equal(got, ref), (got - ref).abs().max().item()
    want = prob.float64()
    err = (got.double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 1e-4, err


@pytest.mark.parametrize("d", [ops.FPROP, ops.DGRAD])
@pytest.mark.parametrize("row", _layer_rows(), ids=lambda r: "x".join(map(str, r[:5])) + "-m%d-a%d-b%d-s%d" % (r[8], r[9], r[10], r[11]))
def test_rows_kernel_bitwise_at_layer_shapes(row, d):
    # which kernel each of these launches takes is pinned by test_which_kernel_each_layer_takes
    args = _launch(d, row)
    _check(_Problem(row[0], *args, seed=row[1] + row[3] + args[-3]))


@pytest.mark.parametrize("edge", EDGES, ids=lambda e: "%s-%dx%dx%dx%d-k%d" % (e[0], *e[1:5], e[6]))
def test_rows_kernel_bitwise_at_edges(edge):
    d, n, h, w, c, halo, k, bias, act = edge
    taps = _taps(d, halo)
    if d == "dgrad":    # the input gradient of a reflection-padded layer is computed on the padded grid
        prob = _Problem(n, h + 2 * halo, w + 2 * halo, taps, c, h, w, 0, k, bias, act, seed=h * w + c + k)
    else:
        prob = _Problem(n, h, w, taps, c, h, w, halo, k, bias, act, seed=h * w + c + k)
    assert _takes_rows(n, prob.oh, prob.ow, c, k, bias, act)
    _check(prob, True)


# ---------------------------------------------------------------- which kernel each layer takes
TC_BN_SET = (32, 48, 64, 96, 104, 112, 128)
SMEM_LIMIT = 227 * 1024 - 1024


def _takes_rows(n, oh, ow, c, k, bias, act):
    """og_conv2d_tc's choice for a 3x3 column-order tap list, restated: a TN = 1 patch with TW % 8 == 0, no reduction
    split, and every chunk's A slot plus two B stages in the shared memory."""
    tw = 1
    while tw * 2 <= ow and tw * 2 <= 16:
        tw *= 2
    th = 1
    while th * 2 <= oh and tw * th * 2 <= 128:
        th *= 2
    if 128 // (tw * th) != 1 or tw % 8:
        return False
    ntile = -(-k // 128)
    bn = next(b for b in TC_BN_SET if b >= (-(-k // ntile) + 7) // 8 * 8)
    tiles = n * -(-oh // th) * -(-ow // tw) * -(-k // bn)
    cch = -(-c // 64)
    nk = 9 * cch
    if tiles < 100 and nk >= 16 and not bias and act == ACT_NONE:
        s = min(-(-2 * torch.cuda.get_device_properties(0).multi_processor_count // tiles), nk // 8)
        if s > 1 and -(-nk // -(-nk // s)) > 1:
            return False
    brows = (16 if k <= 16 else 32) if (bn == 32 and k <= 32) else bn
    return cch * 2 * (th + 2) * tw * 128 + 2 * 2 * brows * 128 + 1024 <= SMEM_LIMIT


def _kernels_launched(fn):
    """Names of the forward tensor-core conv kernels fn launches (every og_conv2d_tc launch runs one).  fn must be
    repeatable: a short profiler session now and then delivers none of the kernel's records, and fn is then run
    again (at most three times)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if "conv_tc" in e.name and "wgrad" not in e.name}
        if names:
            break
    return names


def test_which_kernel_each_layer_takes():
    """Every 3x3 tensor-core row of conv_cases, forward and input gradient: the row-run kernel where og_conv2d_tc's
    predicate holds, conv_tc_kernel otherwise; the upsample phases keep conv_tc_kernel.  The layers named in DESIGN
    §3.1 are pinned by name."""
    took = {}
    for r in CASES + EDGE_CASES:
        n, h, w, cin, cout, k, stride, pad, mode, act, bias, split, path = r
        if path != "s1" or k != 3:
            continue
        for d in (ops.FPROP, ops.DGRAD):
            args = _launch(d, r)     # the upsample forms: the first of their launches (phase 0, row-major taps)
            oh, ow, taps, c, _, _, _, kk, b, a = args
            want = mode != UPSAMPLE2X and _takes_rows(n, oh, ow, c, kk, b, a)
            prob = _Problem(n, *args, seed=1)
            names = _kernels_launched(lambda: prob.run(False))
            assert len(names) == 1, (r, d, names)
            got = "conv_tc_rows_kernel" in next(iter(names))
            assert got == want, (r, d, names)
            took[(n, h, w, cin, cout, mode, d)] = got
            del prob
    # Step-A at batch 16: both res-block convs' forward at 64^2 and 128^2, conv2's input gradient, G_HMAP's
    # reflect convs, the image heads; conv1's input gradient (400 channels) and the upsample phases do not
    for hw in (64, 128):
        assert took[(16, hw, hw, 194, 388, PAD_REFLECT, ops.FPROP)]
        assert took[(16, hw, hw, 194, 194, PAD_REFLECT, ops.FPROP)]
        assert took[(16, hw, hw, 194, 194, PAD_REFLECT, ops.DGRAD)]
        assert not took[(16, hw, hw, 194, 388, PAD_REFLECT, ops.DGRAD)]
        assert not took[(16, hw, hw, 194, 96, UPSAMPLE2X, ops.FPROP)]
    for hw in (64, 128, 256):
        assert took[(16, hw, hw, 80, 24, PAD_REFLECT, ops.FPROP)]
        assert took[(16, hw, hw, 48, 3, 0, ops.FPROP)]
    assert not took[(16, 8, 8, 1024, 768, 0, ops.FPROP)]   # split reduction on a small map


def test_other_run_lengths_keep_conv_tc_kernel():
    """Tap lists that split into runs of a length other than three keep conv_tc_kernel: the 2-tap runs of the 3x3
    stride-2 input-gradient phases (conv_cases rows 24 -> 48 and the like) and the 7-tap runs of a 7x1 convolution
    (INCEPTION_V3 at 17 x 17)."""
    seen = 0
    for r in CASES + EDGE_CASES:
        n, h, w, cin, cout, k, stride, pad, mode, act, bias, split, path = r
        if path != "s2" or k != 3:
            continue
        plan = ops._tc_plan(ops.DGRAD, *ops._conv2d_geo(n, h, w, k, k, stride, pad, mode))
        for taps, oh, ow, *_ in plan.launches:
            prob = _Problem(n, oh, ow, taps, _kp(cout, split), h // 2, w // 2, 0, ops.cpad(cin), False, ACT_NONE, 1)
            names = _kernels_launched(lambda: prob.run(False))
            assert len(names) == 1 and "conv_tc_rows_kernel" not in next(iter(names)), (r, taps, names)
            seen += len(taps) == 2 and taps[0][1] == taps[1][1]
    assert seen, "no 2-tap run among the stride-2 input-gradient phases"
    taps = [(i - 3, 0, 0, i) for i in range(7)]
    prob = _Problem(16, 17, 17, taps, 128, 17, 17, 0, 192, False, ACT_NONE, seed=2)
    names = _kernels_launched(lambda: prob.run(False))
    assert len(names) == 1 and "conv_tc_rows_kernel" not in next(iter(names)), names
