"""Autograd-aware Python operators over the C ABI of libobjgan_b200.so.

PyTorch is plumbing here: device memory (``torch.empty``), the autograd tape and streams.  Every
arithmetic step is a kernel of this repo's library, reached through ``lib.call`` (ctypes); there is no
torch / cuDNN / cuBLAS compute path and no CPU fallback -- CPU tensors raise.

Internal activation layout: NHWC fp32, shape (N, H, W, Cp) with Cp = channels rounded up to 8 and the
pad lanes kept at exactly zero.
"""
from __future__ import annotations

from collections import namedtuple

import torch

from . import lib as _lib
from .lib import (ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, NA_GLU, NA_LRELU, NA_NONE, PAD_REFLECT, PAD_ZERO,
                  TRANSPOSED, UPSAMPLE2X)

LRELU_SLOPE = 0.2
NORM_EPS = 1e-5
BN_MOMENTUM = 0.1


def cpad(c: int) -> int:
    return (c + 7) // 8 * 8


def _chk(*ts):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda and not _lib.DRY_RUN:
            raise RuntimeError("objgan_b200 kernels need CUDA tensors (no CPU fallback)")
        if t.dtype not in (torch.float32, torch.uint8, torch.float64, torch.int64):
            raise RuntimeError(f"unsupported dtype {t.dtype}")


def _p(t):
    return 0 if t is None else t.data_ptr()


def _call(name, *args):
    if _lib.DRY_RUN:  # host-logic tracing only (tests): kernels are NOT executed, outputs stay uninitialised
        lib = _lib.get()
        want = len(lib.protos[name]) - 1          # every prototype ends with the stream
        if len(args) != want:
            raise TypeError(f"{name}: {len(args)} arguments passed, the header declares {want} (+ stream)")
        lib.launches += 1
        return
    _lib.get().call(name, *args, _lib.stream())


# weights change only through the optimiser / load_state_dict; both bump this epoch so cached packed copies
# are rebuilt.  In-place torch ops on a Parameter are caught through Tensor._version.
_param_epoch = [0]


def bump_param_epoch():
    _param_epoch[0] += 1


def _epoch_of(w):
    """(global epoch, epoch of the network that owns w): a network's optimiser step only invalidates ITS operand
    copies (a trainer attaches ``og_epoch`` = its bucket's counter to every parameter)."""
    own = getattr(w, "og_epoch", None)
    return (_param_epoch[0], own[0] if own is not None else 0)


class PackedWeights:
    """Cache of kernel-native copies (fprop and dgrad operand) of one OIHW parameter."""

    def __init__(self):
        self.key = None
        self.f = None
        self.t = None
        self.hl = {}
        self.amax = None

    @staticmethod
    def _key(w, cip, kp, split):
        """What the cached copies were derived from: the parameter's storage, its version and epochs, and the layout."""
        return (w.data_ptr(), w._version, _epoch_of(w), cip, kp, split)

    def _refresh(self, w, cip, kp, split):
        key = self._key(w, cip, kp, split)
        if key != self.key:
            self.key, self.f, self.t, self.hl, self.amax = key, None, None, {}, None

    def install(self, w, cip, kp, split, amax, hl):
        """Re-validate the cache for the current w with the fp16 copies PackPlan.run re-packed in place
        (hl: {transposed: (hi, lo, amax)}); every other copy is dropped."""
        self.key, self.f, self.t, self.hl, self.amax = self._key(w, cip, kp, split), None, None, hl, amax

    def _amax(self, w):
        """Device word with the float bits of max|w| (the power-of-two scale of the fp16 operand copies)."""
        if self.amax is None:
            self.amax = torch.empty(1, device=w.device, dtype=torch.int32)
            _call("og_amax", _p(w), w.numel(), _p(self.amax))
        return self.amax

    def get(self, w, cip, kp, split, splitp, need_t):
        self._refresh(w, cip, kp, split)
        co, ci, kh, kw = w.shape
        if self.f is None:
            self.f = torch.empty(kh * kw * cip * kp, device=w.device, dtype=torch.float32)
            _call("og_pack_weights", _p(w), co, ci, kh, kw, cip, kp, split, splitp, 0, _p(self.f))
        if need_t and self.t is None:
            self.t = torch.empty(kh * kw * cip * kp, device=w.device, dtype=torch.float32)
            _call("og_pack_weights", _p(w), co, ci, kh, kw, cip, kp, split, splitp, 1, _p(self.t))
        return self.f, self.t

    def get_up_hilo(self, w, cip, kp, split, splitp, transposed):
        """Pre-summed 2x2 phase weights of an upsample+conv3x3 layer as (fp16 hi, fp16 lo, scale word), laid out
        [16][co][ci] (transposed) or [16][ci][co]."""
        self._refresh(w, cip, kp, split)
        key = ("up", transposed)
        if key not in self.hl:
            co, ci, _, _ = w.shape
            hi = torch.empty(16 * cip * kp, device=w.device, dtype=torch.float16)
            lo = torch.empty_like(hi)
            amax_up = torch.empty(1, device=w.device, dtype=torch.int32)
            _call("og_pack_upsample_weights", _p(w), co, ci, cip, kp, split, splitp, transposed, _p(self._amax(w)),
                  _p(amax_up), _p(hi), _p(lo))
            self.hl[key] = (hi, lo, amax_up)
        return self.hl[key]

    def get_hilo(self, w, cip, kp, split, splitp, transposed):
        """(fp16 hi, fp16 lo, scale word) of the packed matrix ([tap][co][ci] when transposed else [tap][ci][co])."""
        self._refresh(w, cip, kp, split)
        if transposed not in self.hl:
            co, ci, kh, kw = w.shape
            # hi and lo live back to back in one buffer
            nel = kh * kw * cip * kp
            buf = torch.empty(2 * nel, device=w.device, dtype=torch.float16)
            hi = buf[:nel]
            lo = buf[nel:]
            _call("og_pack_weights_f16", _p(w), co, ci, kh, kw, cip, kp, split, splitp, transposed,
                  _p(self._amax(w)), _p(hi), _p(lo))
            self.hl[transposed] = (hi, lo, self._amax(w))
            plan = getattr(w, "og_pack_plan", None)
            if plan is not None:            # the owner re-packs all of its weights in one launch after its Adam step
                plan.record(self, w, cip, kp, split, splitp, transposed, hi, lo, self._amax(w))
        return self.hl[transposed]


_PackJob = namedtuple("_PackJob", "cache w cip kp split splitp transposed hi lo amax")


class PackPlan:
    """All (weight, layout) fp16 operand copies of ONE network, re-derived by two launches (og_amax_multi +
    og_pack_weights_f16_multi) right after the network's optimiser step instead of lazily, layer by layer, at the next
    use (~300 tiny launches per training step).  Jobs are recorded the first time a layer asks for a copy; from then on
    ``run`` refreshes the SAME buffers and re-validates the layers' caches."""

    def __init__(self):
        self.jobs = []              # _PackJob
        self._tables = None
        self._n_built = 0

    def record(self, cache, w, cip, kp, split, splitp, transposed, hi, lo, amax):
        job = _PackJob(cache, w, cip, kp, split, splitp, transposed, hi, lo, amax)
        for i, j in enumerate(self.jobs):
            if j.cache is cache and j.transposed == transposed:      # same layer and layout packed again: new buffers
                self.jobs[i] = job
                self._tables = None
                return
        self.jobs.append(job)

    def _build(self, device):
        CH = 4096
        arows, prows, ab, pb, seen = [], [], 0, 0, {}
        for j in self.jobs:
            w = j.w
            if id(j.amax) not in seen:
                seen[id(j.amax)] = True
                arows.append([w.data_ptr(), w.numel(), j.amax.data_ptr(), ab])
                ab += (w.numel() + CH - 1) // CH
            co, ci, kh, kw = w.shape
            total = kh * kw * j.cip * j.kp
            prows.append([w.data_ptr(), j.hi.data_ptr(), j.lo.data_ptr(), j.amax.data_ptr(), co, ci,
                          kh * kw, j.cip, j.kp, j.split, j.splitp, j.transposed, total, pb])
            pb += (total + CH - 1) // CH
        mk = lambda rows: h2d(rows, device, torch.int64)
        self._tables = (mk(arows), len(arows), ab, mk(prows), len(prows), pb)
        self._n_built = len(self.jobs)

    def run(self):
        """Call after the weights changed (and after the parameter epoch was bumped)."""
        if not self.jobs:
            return
        if self._tables is None or self._n_built != len(self.jobs):
            self._build(self.jobs[0].w.device)
        at, an, ab, pt, pn, pb = self._tables
        _call("og_amax_multi", _p(at), an, ab)
        _call("og_pack_weights_f16_multi", _p(pt), pn, pb)
        per_cache = {}              # id(cache) -> (its first job, {transposed: (hi, lo, amax)})
        for j in self.jobs:
            per_cache.setdefault(id(j.cache), (j, {}))[1][j.transposed] = (j.hi, j.lo, j.amax)
        for j, hl in per_cache.values():
            j.cache.install(j.w, j.cip, j.kp, j.split, j.amax, hl)


# Contraction engine for the convolutions: "f16x3" = wgmma tensor cores with the error-compensated
# three-product fp16 hi/lo split (22-bit operands, fp32-level accuracy: the default), "simt" = exact fp32 FMA on the
# CUDA cores.
import ctypes
import functools
import os as _os
CONV_ENGINE = _os.environ.get("OBJGAN_CONV", "f16x3")
if CONV_ENGINE not in ("f16x3", "simt"):
    raise ValueError("OBJGAN_CONV=%r: the convolution engine is 'f16x3' or 'simt'" % CONV_ENGINE)
TC_MIN_PIXELS = 256        # smaller problems go to the exact-fp32 SIMT kernels (the tc kernel splits K on small maps)


def _int_array(rows):
    flat = [int(v) for r in rows for v in r]
    return (ctypes.c_int * len(flat))(*flat)


def _empty_slack(shape, device):
    """fp16 buffer with 512 bytes of readable slack after the last element."""
    n = 1
    for d in shape:
        n *= d
    flat = torch.empty(n + 256, device=device, dtype=torch.float16)
    return flat[:n].view(shape)


def _split(x, pad=0, s2d=False):
    """(fp16 hi, fp16 lo, scale word) of an NHWC tensor scaled by a power of two from its max|x|; pad=1 adds the
    reflection halo; s2d gives the four space-to-depth phase blocks [4N, ceil(H/2), ceil(W/2), C] (_split_s2d_odd at
    an odd size)."""
    n, h, w, c = x.shape
    ready_made = getattr(x, "og_split", None)          # the producer already wrote them (og_norm_apply_split)
    if ready_made is not None and ready_made[3:] == (pad, bool(s2d), x._version):
        return ready_made[:3]
    if getattr(x, "og_f32_invalid", False):
        raise RuntimeError("this activation exists only as tensor-core operand copies (pad=%s); a consumer asked for "
                           "another layout" % (ready_made[3] if ready_made else None))
    if s2d and (h % 2 or w % 2):
        return _split_s2d_odd(x)
    shape = (4 * n, h // 2, w // 2, c) if s2d else (n, h + 2 * pad, w + 2 * pad, c)
    xh = _empty_slack(shape, x.device)
    xl = _empty_slack(shape, x.device)
    amax = _known_amax(x)
    ready = amax is not None
    if not ready:
        amax = torch.empty(1, device=x.device, dtype=torch.int32)
    _call("og_prep_split", _p(x), n, h, w, c, pad, 1 if s2d else 0, _p(amax), 1 if ready else 0, _p(xh), _p(xl))
    return xh, xl, amax


def _split_s2d_odd(x):
    """_split(x, s2d=True) at an odd H or W: og_prep_split_s2d zero-fills the phase blocks past the odd edge (at even
    sizes it writes what og_prep_split(s2d=1) does)."""
    n, h, w, c = x.shape
    shape = (4 * n, (h + 1) // 2, (w + 1) // 2, c)
    xh = _empty_slack(shape, x.device)
    xl = _empty_slack(shape, x.device)
    amax = torch.empty(1, device=x.device, dtype=torch.int32)
    _call("og_prep_split_s2d", _p(x), n, h, w, c, _p(amax), 0, _p(xh), _p(xl))
    return xh, xl, amax


def _tag_amax(t):
    """Attach a fresh max|t| word to a tensor some kernel is about to produce (the kernel fills it); a consuming
    convolution then skips its own amax pass.  The tag is void once the tensor is modified in place."""
    word = torch.empty(1, device=t.device, dtype=torch.int32)
    t.og_amax = (word, t._version)
    return word


def _known_amax(t):
    tag = getattr(t, "og_amax", None)
    if tag is not None and tag[1] == t._version:
        return tag[0]
    return None


def _out_hw(h, w, kh, kw, stride, pad, mode, padw=None):
    if mode == UPSAMPLE2X:
        return 2 * h, 2 * w
    padw = pad if padw is None else padw
    return (h + 2 * pad - kh) // stride + 1, (w + 2 * padw - kw) // stride + 1


def conv_path(n, h, w, kh, kw, stride, padh, padw, mode, kp, engine, general=False):
    """The path a convolution of an (n, h, w) source with kp (padded) output channels takes under ``engine``: "s1" /
    "s2" (tensor cores; "s2" on the space-to-depth phases of a stride-2 layer), "narrow" (og_conv2d_narrow_*: 8 padded
    output channels, zero padding, small maps) or "simt" (og_conv2d_simt / og_conv2d_wgrad_simt).

    general: the layer has the tensor-core form at every zero-padded shape of stride 1 or 2 and no narrow form (the
    Inception trunks).  Otherwise the tensor cores take the 3x3 pad-1 layers of any mode, the 4x4 stride-1 zero-padded
    roi_code layer, and the 3x3 / 4x4 stride-2 pad-1 zero-padded layers on even maps.  Either way they need
    TC_MIN_PIXELS output pixels; the batch need not fill the last pixel tile (rows past it are never stored)."""
    oh, ow = _out_hw(h, w, kh, kw, stride, padh, mode, padw)
    if engine == "f16x3" and n * oh * ow >= TC_MIN_PIXELS:
        if general:
            return "s%d" % stride
        if kh == kw and padh == padw == 1:
            if stride == 1 and (kh == 3 or (kh == 4 and mode == PAD_ZERO)):
                return "s1"
            if stride == 2 and kh in (3, 4) and mode == PAD_ZERO and h % 2 == 0 and w % 2 == 0:
                return "s2"
    if not general and kp == 8 and mode == PAD_ZERO and n * oh * ow <= 65536:
        return "narrow"
    return "simt"


def _tc_kind(n, h, w, c, kh, kw, stride, pad, mode):
    """The tensor-core form ("s1" / "s2") conv2d takes for this layer under CONV_ENGINE (conv_path), or None.  c, the
    input channels, decides nothing: only the narrow form looks at channels, and it is not a tensor-core form."""
    path = conv_path(n, h, w, kh, kw, stride, pad, pad, mode, 0, CONV_ENGINE)
    return path if path in ("s1", "s2") else None


FPROP, DGRAD, WGRAD = "fprop", "dgrad", "wgrad"
_UP_OFF = ((-1, 0), (0, 1))   # low-res row/col offsets read by output phase 0 / 1 of upsample + conv3x3
_Plan = namedtuple("_Plan", "xsplit gsplit up ntaps out launches")


@functools.lru_cache(maxsize=None)
def _tc_plan(d, n, h, w, kh, kw, stride, padh, padw, mode, cols=False):
    """The tensor-core launches of one direction (FPROP, DGRAD or WGRAD) of a convolution over an (n, h, w) source.
    Tap order is summation order: these lists fix the bits of the results.

      xsplit, gsplit  the (pad, s2d) layouts _split makes of x and of the output gradient g
      up              the weights are an upsample layer's pre-summed phase weights (get_up_hilo)
      ntaps           taps of the packed weights and of the packed weight gradient
      out             (rows, cols) of the buffer FPROP / DGRAD writes: y, or the input gradient (with the halo of a
                      reflection-padded layer); for WGRAD the grid of g's copies
      launches        FPROP / DGRAD: per og_conv2d_tc launch (taps, oh, ow, osy, opy, opx), taps (dh, dw, dn, widx);
                      WGRAD: one (entries, oh, ow, 1, 0, 0), entries (gdn, dh, dw, xdn, output tap)

    cols: the forward taps of a stride-1 layer without upsampling run column by column, and the input gradient's
    column by column with the kernel rows descending (conv2d's 3x3 layers); otherwise every list runs row by row."""
    oh, ow = _out_hw(h, w, kh, kw, stride, padh, mode, padw)
    halo = padh if mode == PAD_REFLECT else 0             # reflect: x's copies carry the halo; zero pad: TMA fills
    if mode == UPSAMPLE2X:      # 3x3 pad 1 on the 2x map: output phases p = (py, px) of 2x2 taps at low resolution
        xsplit, gsplit, up, ntaps = (0, False), (0, True), True, 16
        phases = [[(_UP_OFF[p // 2][a], _UP_OFF[p % 2][b], 0, (p * 2 + a) * 2 + b) for a in range(2) for b in range(2)]
                  for p in range(4)]
    else:
        xsplit, gsplit, up, ntaps = (halo, stride == 2), (0, False), False, kh * kw
        rows = [(i, j) for i in range(kh) for j in range(kw)]
        if stride == 2:         # x as its four space-to-depth phases: tap (i, j) reads phase (a, b) at offset (dh, dw)
            phases = [[(dh, dw, (a * 2 + b) * n, i * kw + j) for i, j in rows
                       for (dh, a), (dw, b) in [(divmod(i - padh, 2), divmod(j - padw, 2))]]]
        else:
            phases = [[(i - padh + halo, j - padw + halo, 0, i * kw + j) for i, j in rows]]
    cols = cols and stride == 1 and not up
    if d == FPROP:
        out = (oh, ow)
        if up:
            launches = [(taps, h, w, 2, p // 2, p % 2) for p, taps in enumerate(phases)]
        else:
            taps = phases[0]
            if cols:
                taps = [taps[i * kw + j] for j in range(kw) for i in range(kh)]
            launches = [(taps, oh, ow, 1, 0, 0)]
    elif d == DGRAD and stride == 2:    # input pixel (2y + a, 2x + b) <- the taps i = a + padh, j = b + padw (mod 2)
        out = (h, w)
        launches = [([((a + padh - i) // 2, (b + padw - j) // 2, 0, i * kw + j)
                      for i in range(kh) if (a + padh - i) % 2 == 0 for j in range(kw) if (b + padw - j) % 2 == 0],
                     (h + 1) // 2, (w + 1) // 2, 2, a, b) for a in range(2) for b in range(2)]
    elif d == DGRAD:            # the adjoint of every phase in one launch, phase p of g at block dn = p n
        out = (h + 2 * halo, w + 2 * halo)
        taps = [(-dh, -dw, p * n, t) for p, ts in enumerate(phases) for dh, dw, _, t in ts]
        if cols:
            taps = [taps[i * kw + j] for j in range(kw) for i in reversed(range(kh))]
        launches = [(taps, *out, 1, 0, 0)]
    else:                       # dW[t] = sum g[gdn + m, y, x] x[xdn + m, y + dh, x + dw] over the grid of g's copies
        out = (h, w) if up else (oh, ow)
        launches = [([(p * n,) + tap for p, ts in enumerate(phases) for tap in ts], *out, 1, 0, 0)]
    return _Plan(xsplit, gsplit, up, ntaps, out, tuple((tuple(taps), *rest) for taps, *rest in launches))


def _tc_launch(xs, n, ws, plan, y, k, bias=None, act=ACT_NONE, yoff=0, slope=LRELU_SLOPE):
    """The og_conv2d_tc launches of a FPROP / DGRAD plan.  xs / ws: (hi, lo, scale word) operand triples; the source
    is [SN, SH, SW, C] with SN = n or 4n (space-to-depth).  The k output channels start at channel yoff of y."""
    xh, xl, ax = xs
    wh, wl, aw = ws
    sn, sh, sw, c = xh.shape
    _, ohf, owf, kc = y.shape
    for taps, oh, ow, osy, opy, opx in plan.launches:
        arr = _int_array(taps)
        _call("og_conv2d_tc", _p(xh), _p(xl), _p(ax), n, sn, sh, sw, c, _p(wh), _p(wl), _p(aw), plan.ntaps, k,
              _p(y) + 4 * yoff, oh, ow, k, ohf * owf * kc, owf * kc, kc, ohf, owf, osy, osy, opy, opx,
              ctypes.addressof(arr), len(taps), _p(bias), act, slope)


def _simt_conv(x, wp, y, k, kh, kw, stride, padh, padw, mode, bias=None, act=ACT_NONE, slope=LRELU_SLOPE,
               splitk=True, yoff=0):
    """og_conv2d_simt from the contiguous NHWC x into k channels of y (N, OH, OW, Cy) from channel yoff; returns y."""
    n, h, w, c = x.shape
    _, oh, ow, cy = y.shape
    _call("og_conv2d_simt", _p(x), n, h, w, c, h * w * c, w * c, c, _p(wp), _p(y) + 4 * yoff, oh, ow, k, oh * ow * cy,
          ow * cy, cy, kh, kw, stride, padh, padw, mode, _p(bias), act, slope, 1 if splitk else 0)
    return y


def _grad_sink(param):
    """Persistent gradient buffer a trainer attached to a parameter (``param.og_grad_sink``): the backward kernels
    then accumulate into it directly and hand autograd no gradient (one kernel and one temporary less per use)."""
    sink = getattr(param, "og_grad_sink", None)
    if sink is not None and sink.shape == param.shape and sink.is_contiguous():
        return sink
    return None


def _unpack_wgrad(dwp, weight, c, kp, split, splitp, sink, transposed=0, up=False):
    """The OIHW gradient of a packed weight gradient ([tap][kp][c] when transposed, else [tap][c][kp]; up: the 16
    phase taps of an upsample layer), added to the sink if there is one (then None is returned)."""
    co, ci, kh, kw = weight.shape
    gw = torch.empty_like(weight) if sink is None else sink
    acc = 0 if sink is None else 1
    if up:
        _call("og_unpack_upsample_wgrad", _p(dwp), co, ci, c, kp, split, splitp, _p(gw), acc)
    else:
        _call("og_unpack_wgrad", _p(dwp), co, ci, kh, kw, c, kp, split, splitp, _p(gw), acc, transposed)
    return gw if sink is None else None


def _conv2d_geo(n, h, w, kh, kw, stride, pad, mode):
    """The layer arguments of _tc_plan for a conv2d layer: its 3x3 layers' stride-1 taps run column by column."""
    return n, h, w, kh, kw, stride, pad, pad, mode, kh == 3


def _tc_fprop(x, cache, weight, kp, split, splitp, geo, bias_p, act):
    """Returns (y, xs): the output and the fp16 operand triple of x (reused by the weight gradient)."""
    plan = _tc_plan(FPROP, *geo)
    ws = (cache.get_up_hilo if plan.up else cache.get_hilo)(weight, x.shape[3], kp, split, splitp, 1)
    xs = _split(x, *plan.xsplit)
    y = torch.empty((x.shape[0], *plan.out, kp), device=x.device, dtype=torch.float32)
    _tc_launch(xs, x.shape[0], ws, plan, y, kp, bias_p, act)
    return y, xs


def _tc_dgrad(gs, cache, weight, c, kp, split, splitp, geo):
    """Input gradient (N, h, w, c) on the tensor cores from gs, the hi/lo copies of g in the plan's gsplit layout."""
    plan = _tc_plan(DGRAD, *geo)
    n, h, w = geo[:3]
    ws = (cache.get_up_hilo if plan.up else cache.get_hilo)(weight, c, kp, split, splitp, 0)
    gx = torch.empty((n, *plan.out, c), device=gs[0].device, dtype=torch.float32)
    _tc_launch(gs, n, ws, plan, gx, c)
    if plan.out != (h, w):      # the reflection halo folds back onto the border
        gpad, gx = gx, torch.empty((n, h, w, c), device=gx.device, dtype=torch.float32)
        _call("og_reflect_pad_bwd", _p(gpad), n, h, w, c, _p(gx))
    return gx


def _tc_wgrad(xs, gs, weight, c, kp, split, splitp, geo, sink=None):
    """Weight gradient on the tensor cores (og_conv2d_wgrad_tc) from the hi/lo copies of x and g; returns the OIHW
    gradient (None with a sink)."""
    plan = _tc_plan(WGRAD, *geo)
    xh, xl, ax = xs
    gh, gl, ag = gs
    (ents, oh, ow, _, _, _), = plan.launches
    arr = _int_array(ents)
    dwp = torch.empty(plan.ntaps * kp * c, device=xh.device, dtype=torch.float32)
    _call("og_conv2d_wgrad_tc", _p(gh), _p(gl), _p(ag), geo[0], gh.shape[0], oh, ow, kp, _p(xh), _p(xl), _p(ax),
          xh.shape[0], xh.shape[1], xh.shape[2], c, _p(dwp), plan.ntaps, ctypes.addressof(arr), len(ents))
    return _unpack_wgrad(dwp, weight, c, kp, split, splitp, sink, 1, plan.up)


class _Conv2d(torch.autograd.Function):
    """y = act(conv(x, W) + b) on NHWC tensors; W, b are the reference's OIHW / (Co,) parameters."""

    @staticmethod
    def forward(ctx, x, weight, bias, cache, stride, pad, mode, act, split):
        _chk(x, weight, bias)
        x = x.contiguous()
        n, h, w, c = x.shape
        co, ci, kh, kw = weight.shape
        assert c == cpad(ci), (c, ci)
        if split:
            assert co == 2 * split
            splitp = cpad(split)
            kp = 2 * splitp
        else:
            splitp, kp = 0, cpad(co)
        need_t = ctx.needs_input_grad[0]
        oh, ow = _out_hw(h, w, kh, kw, stride, pad, mode)
        kind = _tc_kind(n, h, w, c, kh, kw, stride, pad, mode)
        path = kind or conv_path(n, h, w, kh, kw, stride, pad, pad, mode, kp, "simt")    # narrow or simt
        tc = kind is not None
        geo = _conv2d_geo(n, h, w, kh, kw, stride, pad, mode)
        bias_p = None
        if bias is not None:
            if kp == co:
                bias_p = bias.detach()
            else:
                assert not split
                bias_p = torch.zeros(kp, device=x.device, dtype=torch.float32)
                bias_p[:co] = bias.detach()
        f32_missing = getattr(x, "og_f32_invalid", False)
        if f32_missing and not tc:
            raise RuntimeError("input exists only as tensor-core operand copies, but this convolution runs on the CUDA cores")
        xs = None
        if tc:
            y, xs = _tc_fprop(x, cache, weight, kp, split, splitp, geo, bias_p, act)
            if not ctx.needs_input_grad[1] and not f32_missing:
                xs = None
        elif path == "narrow":
            wf, _ = cache.get(weight, c, kp, split, splitp, False)
            y = torch.empty((n, oh, ow, 8), device=x.device, dtype=torch.float32)
            _call("og_conv2d_narrow_fwd", _p(x), n, h, w, c, _p(wf), _p(y), oh, ow, kh, kw, stride, pad, _p(bias_p), act,
                  LRELU_SLOPE)
        else:
            wf, _ = cache.get(weight, c, kp, split, splitp, False)
            y = _simt_conv(x, wf, torch.empty((n, oh, ow, kp), device=x.device, dtype=torch.float32), kp, kh, kw,
                           stride, pad, pad, mode, bias_p, act, splitk=(bias is None and act == ACT_NONE))
        ctx.path, ctx.geo = path, geo
        ctx.wsink = _grad_sink(weight)
        ctx.bsink = _grad_sink(bias) if bias is not None else None
        ctx.xs = xs                      # hi/lo operand copies of x, reused by the weight gradient
        ctx.cfg = (stride, pad, mode, act, split, splitp, kp, need_t)
        ctx.cache = cache
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, weight, y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, g):
        x, weight, y = ctx.saved_tensors
        stride, pad, mode, act, split, splitp, kp, _ = ctx.cfg
        n, h, w, c = x.shape
        co, ci, kh, kw = weight.shape
        g = g.contiguous()
        oh, ow = g.shape[1], g.shape[2]
        if act != ACT_NONE:
            gp = torch.empty_like(g)
            _call("og_act_backward", _p(y), _p(g), g.numel(), act, LRELU_SLOPE, _p(gp))
            g = gp
        gx = gw = gb = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            scratch = torch.empty(kp, device=g.device, dtype=torch.float64)
            if ctx.bsink is not None:
                _call("og_channel_sum", _p(g), n * oh * ow, kp, _p(scratch), _p(ctx.bsink), co, 1)
            else:
                gb = torch.empty(co, device=g.device, dtype=torch.float32)
                _call("og_channel_sum", _p(g), n * oh * ow, kp, _p(scratch), _p(gb), co, 0)
        path, geo, cache = ctx.path, ctx.geo, ctx.cache
        if path == "narrow":
            wf, _ = cache.get(weight, c, kp, split, splitp, False)
            if ctx.needs_input_grad[0]:
                gx = torch.empty_like(x)
                _call("og_conv2d_narrow_dgrad", _p(g), n, h, w, c, _p(wf), _p(gx), oh, ow, kh, kw, stride, pad)
            if ctx.needs_input_grad[1]:
                dwp = torch.empty(kh * kw * c * 8, device=g.device, dtype=torch.float32)
                _call("og_conv2d_narrow_wgrad", _p(x), n, h, w, c, _p(g), _p(dwp), oh, ow, kh, kw, stride, pad)
                gw = _unpack_wgrad(dwp, weight, c, kp, split, splitp, ctx.wsink)
        elif path in ("s1", "s2"):
            gs = None
            if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
                gs = _split(g, *_tc_plan(DGRAD, *geo).gsplit)
            if ctx.needs_input_grad[0]:
                gx = _tc_dgrad(gs, cache, weight, c, kp, split, splitp, geo)
            if ctx.needs_input_grad[1]:
                xs = ctx.xs if ctx.xs is not None else _split(x, *_tc_plan(WGRAD, *geo).xsplit)
                ctx.xs = None
                gw = _tc_wgrad(xs, gs, weight, c, kp, split, splitp, geo, ctx.wsink)
        else:
            if ctx.needs_input_grad[0]:     # the adjoint as a TRANSPOSED convolution onto the padded / 2x extent
                _, wt = cache.get(weight, c, kp, split, splitp, True)
                if mode == PAD_ZERO:
                    gx = _simt_conv(g, wt, torch.empty_like(x), c, kh, kw, stride, pad, pad, TRANSPOSED)
                elif mode == PAD_REFLECT:
                    assert stride == 1 and pad == 1
                    gpad = _simt_conv(g, wt, torch.empty((n, h + 2, w + 2, c), device=g.device, dtype=torch.float32),
                                      c, kh, kw, 1, 0, 0, TRANSPOSED)
                    gx = torch.empty_like(x)
                    _call("og_reflect_pad_bwd", _p(gpad), n, h, w, c, _p(gx))
                else:  # UPSAMPLE2X
                    gu = _simt_conv(g, wt, torch.empty((n, 2 * h, 2 * w, c), device=g.device, dtype=torch.float32),
                                    c, kh, kw, 1, pad, pad, TRANSPOSED)
                    gx = torch.empty_like(x)
                    _call("og_upsample2x_bwd", _p(gu), n, h, w, c, _p(gx))
            if ctx.needs_input_grad[1]:
                dwp = torch.empty(kh * kw * c * kp, device=g.device, dtype=torch.float32)
                _call("og_conv2d_wgrad_simt", _p(x), n, h, w, c, h * w * c, w * c, c, _p(g), oh, ow, kp, oh * ow * kp,
                      ow * kp, kp, _p(dwp), kh, kw, stride, pad, mode)
                gw = _unpack_wgrad(dwp, weight, c, kp, split, splitp, ctx.wsink)
        return gx, gw, gb, None, None, None, None, None, None


def conv2d(x, weight, bias, cache, *, stride=1, pad=1, mode=PAD_ZERO, act=ACT_NONE, split=0):
    return _Conv2d.apply(x, weight, bias, cache, stride, pad, mode, act, split)


# --------------------------------------------------------------------------------------------------
class _NormAct(torch.autograd.Function):
    """InstanceNorm2d (groups = N) or train-mode BatchNorm (groups = 1) + fused activation (+ residual)."""

    @staticmethod
    def forward(ctx, y, gamma, beta, res, bn_buffers, instance, act, split_pad=None, keep_f32=True):
        _chk(y, gamma, beta, res)
        y = y.contiguous()
        n, h, w, cy = y.shape
        groups = n if instance else 1
        P = h * w if instance else n * h * w
        dev = y.device
        stats = torch.empty(groups * cy * 2, device=dev, dtype=torch.float64)
        mean = torch.empty(groups * cy, device=dev, dtype=torch.float32)
        rstd = torch.empty(groups * cy, device=dev, dtype=torch.float32)
        rm = rv = nbt = None
        if bn_buffers is not None:
            rm, rv, nbt = bn_buffers
            assert gamma.numel() == cy, "BatchNorm layers of this model never need channel padding"
        _call("og_norm_stats", _p(y), groups, P, cy, NORM_EPS, _p(stats), _p(mean), _p(rstd), _p(rm), _p(rv),
              BN_MOMENTUM, cy, _p(nbt))
        co = cy // 2 if act == NA_GLU else cy
        out = torch.empty((n, h, w, co), device=dev, dtype=torch.float32)
        if res is not None:
            res = res.contiguous()
            assert res.shape == out.shape
        fused = (split_pad is not None and CONV_ENGINE == "f16x3"
                 and (res is None or _known_amax(res) is not None) and (split_pad == 0 or (h > 1 and w > 1)))
        if fused:
            # the consuming convolution's operand copies straight from this pass, scaled by an a-priori bound of max|out|
            word = torch.empty(1, device=dev, dtype=torch.int32)
            _call("og_norm_bound", _p(gamma), _p(beta), cy if gamma is not None else 0, P,
                  _p(_known_amax(res)) if res is not None else 0, _p(word))
            xh = _empty_slack((n, h + 2 * split_pad, w + 2 * split_pad, co), dev)
            xl = _empty_slack((n, h + 2 * split_pad, w + 2 * split_pad, co), dev)
            _call("og_norm_apply_split", _p(y), n, h, w, cy, 1 if instance else 0, _p(mean), _p(rstd), _p(gamma),
                  _p(beta), _p(res), act, LRELU_SLOPE, _p(out) if keep_f32 else 0, _p(word), split_pad, _p(xh), _p(xl))
            out.og_amax = (word, out._version)          # an upper bound is a valid operand scale for other consumers
            out.og_split = (xh, xl, word, split_pad, False, out._version)
            if not keep_f32:
                out.og_f32_invalid = True               # nothing may read the fp32 tensor: it was never written
        else:
            _call("og_norm_apply", _p(y), groups, P, cy, _p(mean), _p(rstd), _p(gamma), _p(beta), _p(res), act,
                  LRELU_SLOPE, _p(out), _p(_tag_amax(out)))
        ctx.cfg = (groups, P, cy, act, res is not None)
        ctx.sinks = (_grad_sink(gamma), _grad_sink(beta)) if gamma is not None else (None, None)
        ctx.save_for_backward(y, mean, rstd, gamma, beta)
        return out

    @staticmethod
    def backward(ctx, g):
        y, mean, rstd, gamma, beta = ctx.saved_tensors
        groups, P, cy, act, has_res = ctx.cfg
        g = g.contiguous()
        bstats = torch.empty(groups * cy * 2, device=g.device, dtype=torch.float64)
        dy = torch.empty_like(y)
        dgamma = dbeta = None
        want_pg = gamma is not None and ctx.needs_input_grad[1]     # frozen discriminators (G update): no param grads
        direct = want_pg and ctx.sinks[0] is not None and ctx.sinks[1] is not None
        if direct:
            dgamma, dbeta = ctx.sinks
        elif want_pg:
            dgamma = torch.empty_like(gamma)
            dbeta = torch.empty_like(beta)
        _call("og_norm_backward", _p(y), _p(g), groups, P, cy, _p(mean), _p(rstd), _p(gamma), _p(beta), act,
              LRELU_SLOPE, _p(bstats), _p(dy), _p(dgamma), _p(dbeta), 1 if direct else 0, _p(_tag_amax(dy)))
        if direct:
            dgamma = dbeta = None
        return dy, dgamma, dbeta, (g if has_res else None), None, None, None, None, None


def instance_norm_act(y, act, res=None, split_pad=None, keep_f32=True):
    """``split_pad`` (0 / 1): also emit the fp16 hi / lo operand copies the NEXT convolution needs (plain / with the
    reflection halo), so that convolution skips its split pass; ``keep_f32=False``: the fp32 tensor is not written at
    all (only valid when that convolution is the ONLY reader and runs on the tensor cores)."""
    return _NormAct.apply(y, None, None, res, None, True, act, split_pad, keep_f32)


class _BatchNormEvalAct(torch.autograd.Function):
    """Eval-mode BatchNorm (running statistics) + fused activation.  The running buffers are only read: eval() must
    not move them, and the output of a sample must not depend on the other samples of its batch."""

    @staticmethod
    def forward(ctx, y, gamma, beta, running_mean, running_var, act):
        _chk(y, gamma, beta, running_mean, running_var)
        y = y.contiguous()
        n, h, w, cy = y.shape
        assert gamma.numel() == cy, "BatchNorm layers of this model never need channel padding"
        P = n * h * w
        mean = torch.empty(cy, device=y.device, dtype=torch.float32)
        rstd = torch.empty(cy, device=y.device, dtype=torch.float32)
        _call("og_bn_eval_coef", _p(running_mean), _p(running_var), cy, NORM_EPS, _p(mean), _p(rstd))
        co = cy // 2 if act == NA_GLU else cy
        out = torch.empty((n, h, w, co), device=y.device, dtype=torch.float32)
        _call("og_norm_apply", _p(y), 1, P, cy, _p(mean), _p(rstd), _p(gamma), _p(beta), 0, act, LRELU_SLOPE,
              _p(out), _p(_tag_amax(out)))
        ctx.cfg = (P, cy, act)
        ctx.sinks = (_grad_sink(gamma), _grad_sink(beta))
        ctx.save_for_backward(y, mean, rstd, gamma, beta)
        return out

    @staticmethod
    def backward(ctx, g):
        y, mean, rstd, gamma, beta = ctx.saved_tensors
        P, cy, act = ctx.cfg
        g = g.contiguous()
        dy = torch.empty_like(y)
        dgamma = dbeta = None
        want_pg = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        direct = want_pg and ctx.sinks[0] is not None and ctx.sinks[1] is not None
        if direct:
            dgamma, dbeta = ctx.sinks
        elif want_pg:
            dgamma = torch.empty_like(gamma)
            dbeta = torch.empty_like(beta)
        _call("og_bn_eval_backward", _p(y), _p(g), P, cy, _p(mean), _p(rstd), _p(gamma), _p(beta), act, LRELU_SLOPE,
              _p(dy), _p(dgamma), _p(dbeta), 1 if direct else 0, _p(_tag_amax(dy)))
        if direct:
            dgamma = dbeta = None
        return dy, dgamma, dbeta, None, None, None


def batch_norm_act(y, gamma, beta, buffers, act, training=True):
    """BatchNorm (+ fused activation).  ``training``: batch statistics, and the running buffers (running_mean,
    running_var, num_batches_tracked) are updated; otherwise the running statistics normalise and nothing is updated."""
    if not training:
        return _BatchNormEvalAct.apply(y, gamma, beta, buffers[0], buffers[1], act)
    return _NormAct.apply(y, gamma, beta, None, buffers, False, act)


# --------------------------------------------------------------------------------------------------
class _ToNHWC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cp):
        _chk(x)
        x = x.contiguous()
        n, c, h, w = x.shape
        y = torch.empty((n, h, w, cp), device=x.device, dtype=torch.float32)
        _call("og_nchw_to_nhwc", _p(x), n, c, h, w, cp, _p(y))
        ctx.c = c
        return y

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        n, h, w, cp = g.shape
        gx = torch.empty((n, ctx.c, h, w), device=g.device, dtype=torch.float32)
        _call("og_nhwc_to_nchw", _p(g), n, ctx.c, h, w, cp, _p(gx))
        return gx, None


class _ToNCHW(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, c):
        _chk(y)
        y = y.contiguous()
        n, h, w, cp = y.shape
        x = torch.empty((n, c, h, w), device=y.device, dtype=torch.float32)
        _call("og_nhwc_to_nchw", _p(y), n, c, h, w, cp, _p(x))
        ctx.cp = cp
        return x

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        n, c, h, w = g.shape
        gy = torch.empty((n, h, w, ctx.cp), device=g.device, dtype=torch.float32)
        _call("og_nchw_to_nhwc", _p(g), n, c, h, w, ctx.cp, _p(gy))
        return gy, None


# Derived copies of CONSTANT inputs (no gradient: segmentation maps, real images): a step converts / resizes the same
# input tensor for several networks (the 80-channel 256^2 class maps go through NCHW -> NHWC eight times and through the
# 512^2 bilinear resize four times in one Step-B); the copy is kept while the source tensor is the same object at the
# same version.  Never used while a CUDA graph is being captured (a replay must recompute from the static buffers).
_CONST_CACHE = []          # [(weakref to the source, version, key, value)], newest last
_CONST_CACHE_SLOTS = 12


def cached_const(src, key, fn):
    import weakref
    if src.requires_grad or not src.is_cuda or torch.cuda.is_current_stream_capturing():
        return fn()
    for ref, ver, k, val in _CONST_CACHE:
        if k == key and ver == src._version and ref() is src:
            return val
    val = fn()
    _CONST_CACHE[:] = [e for e in _CONST_CACHE if e[0]() is not None][-(_CONST_CACHE_SLOTS - 1):]
    _CONST_CACHE.append((weakref.ref(src), src._version, key, val))
    return val


def to_nhwc(x, cp=None):
    cp = cpad(x.shape[1]) if cp is None else cp
    if not x.requires_grad:
        return cached_const(x, ("nhwc", cp), lambda: _ToNHWC.apply(x, cp))
    return _ToNHWC.apply(x, cp)


def to_nchw(y, c):
    return _ToNCHW.apply(y, c)


class _Add(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        _chk(a, b)
        a, b = a.contiguous(), b.contiguous()
        out = torch.empty_like(a)
        _call("og_add", _p(a), _p(b), _p(out), a.numel())
        return out

    @staticmethod
    def backward(ctx, g):
        return g, g


def add(a, b):
    return _Add.apply(a, b)


class _CatChannels(torch.autograd.Function):
    """torch.cat along channels for NHWC tensors with padded lanes: copies the first reals[i] channels of
    each input back to back and zero-fills the tail up to cpad(sum(reals))."""

    @staticmethod
    def forward(ctx, reals, *xs):
        _chk(*xs)
        xs = [x.contiguous() for x in xs]
        n, h, w, _ = xs[0].shape
        tot = sum(reals)
        cp = cpad(tot)
        out = torch.empty((n, h, w, cp), device=xs[0].device, dtype=torch.float32)
        if cp != tot:
            out.zero_()
        off = 0
        P = n * h * w
        for x, r in zip(xs, reals):
            _call("og_copy_channels", _p(x), x.shape[3], 0, _p(out), cp, off, r, P, 0)
            off += r
        ctx.reals = reals
        ctx.cps = [x.shape[3] for x in xs]
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        n, h, w, cp = g.shape
        P = n * h * w
        outs, off = [], 0
        for i, (r, c) in enumerate(zip(ctx.reals, ctx.cps)):
            if ctx.needs_input_grad[1 + i]:
                gi = torch.empty((n, h, w, c), device=g.device, dtype=torch.float32)
                if c != r:
                    gi.zero_()
                _call("og_copy_channels", _p(g), cp, off, _p(gi), c, 0, r, P, 0)
                outs.append(gi)
            else:
                outs.append(None)
            off += r
        return (None, *outs)


def cat_channels(xs, reals):
    return _CatChannels.apply(tuple(reals), *xs)


class _GatherRows(torch.autograd.Function):
    """out[i] = x[idx[i]] over the leading dimension (idx: int64 device tensor)."""

    @staticmethod
    def forward(ctx, x, idx):
        _chk(x, idx)
        x = x.contiguous()
        n_in = x.shape[0]
        rowlen = x.numel() // max(n_in, 1)
        out = torch.empty((idx.numel(),) + tuple(x.shape[1:]), device=x.device, dtype=torch.float32)
        _call("og_gather_rows", _p(x), _p(idx), idx.numel(), rowlen, _p(out))
        ctx.save_for_backward(idx)
        ctx.shape = tuple(x.shape)
        return out

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        g = g.contiguous()
        gx = torch.empty(ctx.shape, device=g.device, dtype=torch.float32)
        n_in = ctx.shape[0]
        rowlen = gx.numel() // max(n_in, 1)
        _call("og_scatter_rows_add", _p(g), _p(idx), idx.numel(), n_in, rowlen, _p(gx))
        return gx, None


def gather_rows(x, idx):
    return _GatherRows.apply(x, idx)


def cat_rows_const(a, b):
    """torch.cat((a, b), dim=1) for two constant (no-grad) 2-D tensors: two strided row copies."""
    _chk(a, b)
    a, b = a.detach().contiguous(), b.detach().contiguous()
    r, ca, cb = a.shape[0], a.shape[1], b.shape[1]
    assert b.shape[0] == r
    out = torch.empty((r, ca + cb), device=a.device, dtype=torch.float32)
    _call("og_copy_channels", _p(a), ca, 0, _p(out), ca + cb, 0, ca, r, 0)
    _call("og_copy_channels", _p(b), cb, 0, _p(out), ca + cb, ca, cb, r, 0)
    return out


class _BroadcastCat(torch.autograd.Function):
    """D_GET_LOGITS conditioning: cat(h, c_code broadcast over the grid) along channels.  c_code is the detached
    sentence embedding in the patch-D callers (miscc/losses.py:169-190, 375-377); in the object-discriminator terms of
    G_loss it carries the generator's bt_c_code (losses.py:436-452), so its gradient is produced when asked for."""

    @staticmethod
    def forward(ctx, h, c_code):
        _chk(h, c_code)
        h, c_code = h.contiguous(), c_code.contiguous()
        n, hh, ww, ch = h.shape
        cc = c_code.shape[1]
        cp = cpad(ch + cc)
        out = torch.empty((n, hh, ww, cp), device=h.device, dtype=torch.float32)
        if cp != ch + cc:
            out.zero_()
        P = n * hh * ww
        _call("og_copy_channels", _p(h), ch, 0, _p(out), cp, 0, ch, P, 0)
        _call("og_broadcast_channels", _p(c_code), n, cc, _p(out), cp, ch, hh * ww)
        ctx.ch, ctx.cc = ch, cc
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        n, hh, ww, cp = g.shape
        gh = torch.empty((n, hh, ww, ctx.ch), device=g.device, dtype=torch.float32)
        _call("og_copy_channels", _p(g), cp, 0, _p(gh), ctx.ch, 0, ctx.ch, n * hh * ww, 0)
        gc = None
        if ctx.needs_input_grad[1]:
            gc = torch.empty((n, ctx.cc), device=g.device, dtype=torch.float32)
            _call("og_broadcast_channels_bwd", _p(g), n, ctx.cc, cp, ctx.ch, hh * ww, _p(gc))
        return gh, gc


class _CatRows(torch.autograd.Function):
    """torch.cat((a, b), dim=1) of two 2-D tensors where only ``b`` carries a gradient."""

    @staticmethod
    def forward(ctx, a, b):
        ctx.ca = a.shape[1]
        return cat_rows_const(a, b)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        r, c = g.shape
        cb = c - ctx.ca
        gb = torch.empty((r, cb), device=g.device, dtype=torch.float32)
        _call("og_copy_channels", _p(g), c, ctx.ca, _p(gb), cb, 0, cb, r, 0)
        return None, gb


def cat_rows(a_const, b):
    return _CatRows.apply(a_const, b)


def broadcast_cat(h, c_code):
    return _BroadcastCat.apply(h, c_code)


class _GLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _chk(x)
        x = x.contiguous()
        ch = x.shape[-1] // 2
        P = x.numel() // (2 * ch)
        out = torch.empty((*x.shape[:-1], ch), device=x.device, dtype=torch.float32)
        _call("og_glu_fwd", _p(x), P, ch, _p(out))
        ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        ch = x.shape[-1] // 2
        gx = torch.empty_like(x)
        _call("og_glu_bwd", _p(x), _p(g.contiguous()), x.numel() // (2 * ch), ch, _p(gx))
        return gx


def glu(x):
    return _GLU.apply(x)


class _Reparam(torch.autograd.Function):
    """c = eps * exp(0.5 * logvar) + mu with x rows = [mu (D) | logvar (D) | pad]; c rows padded to cpad(D)."""

    @staticmethod
    def forward(ctx, x, eps, d):
        _chk(x, eps)
        x, eps = x.contiguous(), eps.contiguous()
        b = x.shape[0]
        cs = cpad(d)
        c = torch.zeros((b, cs), device=x.device, dtype=torch.float32)
        _call("og_reparam_fwd", _p(x), x.shape[1], _p(eps), b, d, _p(c), cs)
        ctx.d = d
        ctx.save_for_backward(x, eps)
        return c

    @staticmethod
    def backward(ctx, gc):
        x, eps = ctx.saved_tensors
        gc = gc.contiguous()
        gx = torch.zeros_like(x)
        _call("og_reparam_bwd", _p(x), x.shape[1], _p(eps), _p(gc), gc.shape[1], x.shape[0], ctx.d, _p(gx))
        return gx, None, None


def reparam(x, eps, d):
    return _Reparam.apply(x, eps, d)


# --------------------------------------------------------------------------------------------------
# losses: scalar = weight * mean(...)
# --------------------------------------------------------------------------------------------------
class _BCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p, target, weight):
        _chk(p)
        p = p.contiguous()
        loss = torch.zeros((), device=p.device, dtype=torch.float32)
        gp = torch.empty_like(p) if ctx.needs_input_grad[0] else None
        _call("og_bce", _p(p), p.numel(), float(target), float(weight), _p(loss), _p(gp))
        ctx.save_for_backward(gp)
        return loss

    @staticmethod
    def backward(ctx, g):
        (gp,) = ctx.saved_tensors
        return gp * g, None, None


def bce(p, target, weight=1.0):
    """weight * nn.BCELoss()(p, full_like(p, target))."""
    return _BCE.apply(p, target, weight)


class _KL(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, d, weight):
        _chk(x)
        x = x.contiguous()
        loss = torch.zeros((), device=x.device, dtype=torch.float32)
        gx = torch.zeros_like(x)
        _call("og_kl", _p(x), x.shape[1], x.shape[0], d, float(weight), _p(loss), _p(gx))
        ctx.save_for_backward(gx)
        return loss

    @staticmethod
    def backward(ctx, g):
        (gx,) = ctx.saved_tensors
        return gx * g, None, None


def kl_rows(x, d, weight=1.0):
    return _KL.apply(x, d, weight)


# --------------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------------
def mask_bytes(mask):
    if mask is None:
        return None
    return mask.to(torch.uint8).contiguous()


class _WordsProj(torch.autograd.Function):
    @staticmethod
    def forward(ctx, words, w):
        _chk(words, w)
        words = words.contiguous()
        b, cdf, l = words.shape
        idf = w.shape[0]
        src = torch.empty((b, idf, l), device=words.device, dtype=torch.float32)
        _call("og_words_proj", _p(words), _p(w), b, idf, cdf, l, _p(src))
        ctx.save_for_backward(words, w)
        return src

    @staticmethod
    def backward(ctx, g):
        words, w = ctx.saved_tensors
        g = g.contiguous()
        b, cdf, l = words.shape
        idf = w.shape[0]
        gw = torch.empty_like(w) if ctx.needs_input_grad[1] else None
        gwords = torch.empty_like(words) if ctx.needs_input_grad[0] else None
        _call("og_words_proj_bwd", _p(words), _p(w), _p(g), b, idf, cdf, l, _p(gw), 0, _p(gwords))
        return gwords, gw


def words_proj(words, w):
    return _WordsProj.apply(words, w)


class _AttGeneral(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, src, mask_u8, idf):
        _chk(h, src, mask_u8)
        h, src = h.contiguous(), src.contiguous()
        b, ih, iw, cs = h.shape
        l = src.shape[2]
        q = ih * iw
        wc = torch.empty_like(h)
        attn = torch.empty((b, l, ih, iw), device=h.device, dtype=torch.float32)
        _call("og_att_general_fwd", _p(h), _p(src), _p(mask_u8), b, q, idf, cs, l, _p(wc), _p(attn))
        ctx.idf = idf
        ctx.save_for_backward(h, src, attn)
        ctx.mark_non_differentiable(attn)  # visualisation only (trainer.py:390 discards it)
        return wc, attn

    @staticmethod
    def backward(ctx, g_wc, _g_attn):
        h, src, attn = ctx.saved_tensors
        b, ih, iw, cs = h.shape
        l = src.shape[2]
        g_h = torch.empty_like(h)
        g_src = torch.empty_like(src)
        _call("og_att_general_bwd", _p(h), _p(src), _p(attn), _p(g_wc.contiguous()), b, ih * iw, ctx.idf, cs, l,
              _p(g_h), _p(g_src))
        return g_h, g_src, None, None


def att_general(h, src, mask_u8, idf):
    return _AttGeneral.apply(h, src, mask_u8, idf)


class _BuAtt(torch.autograd.Function):
    @staticmethod
    def forward(ctx, labels, glove, src, mask_u8, norm):
        _chk(labels, glove, src, mask_u8)
        labels, glove, src = labels.contiguous(), glove.contiguous(), src.contiguous()
        b, e, r = labels.shape
        l = glove.shape[2]
        idf = src.shape[1]
        wc = torch.empty((b, idf, r), device=src.device, dtype=torch.float32)
        attn = torch.empty((b, l, r), device=src.device, dtype=torch.float32)
        _call("og_bu_att_fwd", _p(labels), _p(glove), _p(src), _p(mask_u8), b, e, r, l, idf, 1 if norm else 0, 1e-8,
              _p(wc), _p(attn))
        ctx.save_for_backward(attn)
        ctx.dims = (b, r, l, idf)
        ctx.mark_non_differentiable(attn)
        return wc, attn

    @staticmethod
    def backward(ctx, g_wc, _g):
        (attn,) = ctx.saved_tensors
        b, r, l, idf = ctx.dims
        g_src = torch.empty((b, idf, l), device=attn.device, dtype=torch.float32)
        _call("og_bu_att_bwd", _p(attn), _p(g_wc.contiguous()), b, r, l, idf, _p(g_src))
        return None, None, g_src, None, None


def bu_att(labels, glove, src, mask_u8, norm=True):
    return _BuAtt.apply(labels, glove, src, mask_u8, norm)


class _PaintMax(torch.autograd.Function):
    """pprocess_bt_attns: out[b, y, x, k] = max_r f[b, k, r] * m[b, r, y, x]; f (B, num, R), m (B, Rtot, ih, iw)."""

    @staticmethod
    def forward(ctx, f, m):
        _chk(f, m)
        f, m = f.contiguous(), m.contiguous()
        b, num, r = f.shape
        _, rtot, ih, iw = m.shape
        cp = cpad(num)
        out = torch.empty((b, ih, iw, cp), device=f.device, dtype=torch.float32)
        if cp != num:
            out.zero_()
        _call("og_paint_max_fwd", _p(f), _p(m), b, num, r, rtot, ih * iw, _p(out), cp, 0)
        ctx.save_for_backward(f, m)
        return out

    @staticmethod
    def backward(ctx, g):
        f, m = ctx.saved_tensors
        g = g.contiguous()
        b, num, r = f.shape
        _, rtot, ih, iw = m.shape
        g_f = torch.empty_like(f)
        _call("og_paint_max_bwd", _p(f), _p(m), _p(g), g.shape[3], 0, b, num, r, rtot, ih * iw, _p(g_f))
        return g_f, None


def paint_max(f, m):
    return _PaintMax.apply(f, m)


class _FuncAttention(torch.autograd.Function):
    """DAMSM attention (reference: GlobalAttention.py:32-70) on the reference's NCHW tensors."""

    @staticmethod
    def forward(ctx, query, context, gamma1):
        _chk(query, context)
        query, context = query.contiguous(), context.contiguous()
        b, ndf, lq = query.shape
        ih, iw = context.shape[2:]
        wc = torch.empty((b, ndf, lq), device=query.device, dtype=torch.float32)
        attn = torch.empty((b, lq, ih, iw), device=query.device, dtype=torch.float32)
        _call("og_func_attention_fwd", _p(query), _p(context), b, ndf, lq, ih * iw, float(gamma1), _p(wc), _p(attn))
        ctx.gamma1 = float(gamma1)
        ctx.save_for_backward(query, context, attn)
        return wc, attn

    @staticmethod
    def backward(ctx, g_wc, g_attn):
        query, context, attn = ctx.saved_tensors
        b, ndf, lq = query.shape
        s = context.shape[2] * context.shape[3]
        g_q = torch.empty_like(query)
        g_c = torch.empty_like(context)
        ga = g_attn.contiguous() if g_attn is not None else None
        _call("og_func_attention_bwd", _p(query), _p(context), _p(attn), _p(g_wc.contiguous()), _p(ga), b, ndf, lq, s,
              ctx.gamma1, _p(g_q), _p(g_c))
        return g_q, g_c, None


def func_attention(query, context, gamma1):
    return _FuncAttention.apply(query, context, gamma1)


def h2d(data, device, dtype=None):
    """Small host table (list / numpy array / CPU tensor) -> device WITHOUT stalling the host: staged in pinned memory
    and copied asynchronously on the current stream (a pageable ``.to(device)`` blocks the calling thread until the GPU
    has drained the stream, which serialises an eager step with its own kernels).  The caching pinned allocator only
    reuses the staging block after the copy has executed."""
    import numpy as np
    if torch.is_tensor(data):
        t = data if dtype is None else data.to(dtype)
    elif isinstance(data, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(data))
        t = t if dtype is None else t.to(dtype)
    else:
        t = torch.tensor(data, dtype=dtype)
    dev = torch.device(device)
    if dev.type != "cuda" or t.device.type == "cuda":
        return t.to(dev)
    return t.contiguous().pin_memory().to(dev, non_blocking=True)


def permute_channels(x, perm):
    """out[b, c] = x[b, perm[b, c]] for an NCHW tensor and a (B, C) int64 table on the device."""
    _chk(x, perm)
    x = x.detach().contiguous()
    b, c, h, w = x.shape
    assert perm.shape == (b, c) and perm.dtype == torch.int64
    out = torch.empty_like(x)
    _call("og_permute_channels", _p(x), _p(perm.contiguous()), b, c, h * w, _p(out))
    return out


def zeros(shape, device):
    """Zero-filled fp32 tensor through cudaMemsetAsync (a memset node inside a captured graph, no library kernel)."""
    t = torch.empty(shape, device=device, dtype=torch.float32)
    _chk(t)
    _call("og_zero_bytes", _p(t), t.numel() * 4)
    return t


def form_hmaps(bt_masks, roi_cls, num_rois, num_classes, clamp_max=0.0, out=None):
    """Class heat maps (B, num_classes, S, S) from the per-roi masks (B, R, S, S) and the roi class ids (B, R) int64:
    what the reference's loader accumulates on the host (ref: miscc/load.py:160-176), rebuilt on the device."""
    _chk(bt_masks, roi_cls, num_rois)
    bt_masks = bt_masks.contiguous()
    b, r, h, w = bt_masks.shape
    assert roi_cls.dtype == torch.int64 and num_rois.dtype == torch.int64 and roi_cls.shape == (b, r)
    if out is None:
        out = torch.empty((b, num_classes, h, w), device=bt_masks.device, dtype=torch.float32)
    _call("og_form_hmaps", _p(bt_masks), _p(roi_cls.contiguous()), _p(num_rois.contiguous()), b, r, h * w, num_classes,
          float(clamp_max), _p(out))
    return out


def form_clabels_feat(clabels_emb, roi_cls, num_rois, rmax, out=None):
    """ref: miscc/utils.py:502-522 on the device: (B, E, rmax, 1) label embeddings of the first num_rois[b] boxes."""
    _chk(clabels_emb, roi_cls, num_rois)
    b, r = roi_cls.shape
    ncls, e = clabels_emb.shape
    if out is None:
        out = torch.empty((b, e, rmax, 1), device=clabels_emb.device, dtype=torch.float32)
    _call("og_form_clabels_feat", _p(clabels_emb.contiguous()), _p(roi_cls.contiguous()), _p(num_rois.contiguous()), b, r,
          rmax, e, ncls, _p(out))
    return out


# --------------------------------------------------------------------------------------------------
# Shape generator stage (SHP_G_NET and the heat maps of its masks).  Inference only: none of these has a backward.
# --------------------------------------------------------------------------------------------------
def inference_only(what, *ts):
    """Raises when autograd would have to record ``what`` (a tensor it reads requires grad and grad mode is on)."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts):
        raise RuntimeError(f"{what} is inference only (it has no backward): run it under torch.no_grad()")


def _i64(t):
    assert t.dtype == torch.int64
    return t.contiguous()


def form_bbox_maps(rois0, fm_rois, roi_cls, num_rois, rmax, num_classes, size=64, fsize=16):
    """The loader's box maps (ref: miscc/load.py:178-189, 625-641) on the device, from the box tables of the batch:
    ``rois0`` / ``fm_rois`` (B, BOXES, >=4) float64 (x, y, w, h at 64 / 32 pixels), ``roi_cls`` (B, BOXES) int64.
    Returns the forward and backward sequences as ONE NHWC tensor (2*B*rmax, size, size, cpad(num_classes)) --
    image b*rmax + t of the forward half, then the backward half, whose slot t is box slot BOXES-1-t -- and
    bbox_fmaps (B, rmax, fsize, fsize)."""
    _chk(rois0, fm_rois, roi_cls, num_rois)
    r0 = rois0.to(torch.float64).contiguous()
    fm = fm_rois.to(torch.float64).contiguous()
    b, boxes = roi_cls.shape
    assert r0.shape[:2] == (b, boxes) and fm.shape[:2] == (b, boxes) and rmax <= boxes
    cp = cpad(num_classes)
    dev = r0.device
    maps = torch.empty((2 * b * rmax, size, size, cp), device=dev, dtype=torch.float32)
    fmaps = torch.empty((b, rmax, fsize, fsize), device=dev, dtype=torch.float32)
    _call("og_form_bbox_maps", _p(r0), r0.shape[2], _p(fm), fm.shape[2], _p(_i64(roi_cls)), _p(_i64(num_rois)), b, boxes,
          rmax, num_classes, cp, size, fsize, _p(maps), _p(fmaps))
    return maps, fmaps


def nchw_rows(xs, cp):
    """NCHW tensors (N_i, C, H, W) -> one NHWC tensor (sum N_i, H, W, cp), stacked along the batch."""
    _chk(*xs)
    n = sum(x.shape[0] for x in xs)
    _, c, h, w = xs[0].shape
    out = torch.empty((n, h, w, cp), device=xs[0].device, dtype=torch.float32)
    off = 0
    for x in xs:
        x = x.detach().contiguous()
        _call("og_nchw_to_nhwc", _p(x), x.shape[0], c, h, w, cp, _p(out[off:]))
        off += x.shape[0]
    return out


def fill_channels(dst, rows, doff):
    """dst[i, :, :, doff:doff+C] = rows[i] for an NHWC tensor dst (N, H, W, Cd) and rows (N, C)."""
    _chk(dst, rows)
    n, h, w, cd = dst.shape
    rows = rows.detach().contiguous().view(n, -1)
    _call("og_broadcast_channels", _p(rows), n, rows.shape[1], _p(dst), cd, doff, h * w)
    return dst


def clstm_cell(gx, gh, c, joint, t):
    """One step of both ConvLSTM directions (ref: model.py:818-863).  gx = (fwd, bwd) x-parts of Gates with bias for all
    steps, NHWC (B*R, H, W, 4*Ch); gh = None at t = 0 (zero state) or the (fwd, bwd) h-parts (B, H, W, 4*Ch); c = (fwd,
    bwd) cell states (B, H, W, Ch), updated in place.  h goes to joint (B*R, H, W, Cj) channels [0, Ch) of slot t
    (forward) and [Ch, 2*Ch) of slot R-1-t (backward); returns (h_fwd, h_bwd)."""
    inference_only("the ConvLSTM cell", *gx, *(gh or ()), *c)
    _chk(*gx, *(gh or ()), *c, joint)
    b, hh, ww, ch = c[0].shape
    r = gx[0].shape[0] // b
    assert gx[0].shape == (b * r, hh, ww, 4 * ch) and joint.shape[:3] == (b * r, hh, ww)
    hf, hb = torch.empty_like(c[0]), torch.empty_like(c[1])
    _call("og_clstm_cell", _p(gx[0]), _p(gx[1]), _p(gh[0]) if gh else 0, _p(gh[1]) if gh else 0, _p(c[0]), _p(c[1]),
          _p(hf), _p(hb), _p(joint), b, r, t, hh * ww, ch, joint.shape[3])
    return hf, hb


def mul_pixels(x, s):
    """x * s broadcast over channels: x NHWC (N, H, W, C), s with N*H*W elements (one factor per pixel)."""
    inference_only("mul_pixels", x, s)
    _chk(x, s)
    x = x.contiguous()
    n, h, w, c = x.shape
    assert s.numel() == n * h * w
    out = torch.empty_like(x)
    _call("og_mul_pixels", _p(x), _p(s.contiguous()), n * h * w, c, _p(out))
    return out


def _resize_nhwc(x, size):
    """F.interpolate(bilinear, align_corners=True) to size x size; the identity when the size does not change."""
    n, h, w, c = x.shape
    if (h, w) == (size, size):
        return x
    y = torch.empty((n, size, size, c), device=x.device, dtype=torch.float32)
    _call("og_bilinear_fwd", _p(x), n, h, w, c, size, size, _p(y))
    return y


def _nchw_of(x, c):
    n, h, w, cp = x.shape
    out = torch.empty((n, c, h, w), device=x.device, dtype=torch.float32)
    _call("og_nhwc_to_nchw", _p(x), n, c, h, w, cp, _p(out))
    return out


def form_gen_hmaps(raw_masks, roi_cls, num_rois, sizes=(64, 128, 256), num_classes=80):
    """form_hmaps (ref: miscc/utils.py:524-584) on the device: the generated masks (B, R, 64, 64) (or (B, R, 1, 64, 64))
    -> (hmaps[len(sizes)], bt_masks[len(sizes)], fm_bt_masks).  hmaps are (B, num_classes, s, s); the per-roi tensors are
    (B, BOXES, s, s) with the slots past R zero, the shapes a batch with ground-truth masks has.  Slots
    num_rois[b] <= t < R are not normalised: they keep the raw sigmoid values, as in the reference."""
    _chk(raw_masks, roi_cls, num_rois)
    inference_only("form_gen_hmaps", raw_masks)
    raw = raw_masks.detach()
    if raw.dim() == 5:
        raw = raw[:, :, 0]
    raw = raw.contiguous()
    b, r, h, w = raw.shape
    boxes = roi_cls.shape[1]
    assert roi_cls.shape[0] == b and r <= boxes
    cs = (boxes + 3) // 4 * 4               # one lane per box slot; lanes >= R are zero
    top = max(sizes)
    dev = raw.device
    x = torch.empty((b, h, w, cs), device=dev, dtype=torch.float32)
    _call("og_nchw_to_nhwc", _p(raw), b, r, h, w, cs, _p(x))
    slots = _resize_nhwc(x, top)            # normalised in place below
    cp = cpad(num_classes)
    hm = torch.empty((b, top, top, cp), device=dev, dtype=torch.float32)
    _call("og_gen_hmaps", _p(slots), b, top * top, cs, _p(_i64(roi_cls)), boxes, _p(_i64(num_rois)), num_classes, cp,
          _p(hm))
    hmaps = [_nchw_of(_resize_nhwc(hm, s), num_classes) for s in sizes]
    bt_masks = [_nchw_of(_resize_nhwc(slots, s), boxes) for s in sizes]
    fm_bt_masks = _nchw_of(_resize_nhwc(slots, sizes[0] // 2), boxes)
    return hmaps, bt_masks, fm_bt_masks


class _WordsPairs(torch.autograd.Function):
    """All B x NC (image, caption) pairs of words_loss in one launch (ref: miscc/losses.py:87-127): func_attention,
    word / attended-context cosine and the Eq. (10) pooling.  ctx_feat (B, ndf, ih, iw) carries the gradient;
    words (NC, ndf, T) and lens (NC,) int64 on the device are constants.  Returns sim (B, NC), attn (B, NC, T, ih, iw)
    (rows beyond a caption's length are zero)."""

    @staticmethod
    def forward(ctx, feat, words, lens, gamma1, gamma2, eps):
        _chk(feat, words, lens)
        feat, words = feat.contiguous(), words.detach().contiguous()
        assert lens.dtype == torch.int64 and lens.is_contiguous()
        b, ndf, ih, iw = feat.shape
        nc, _, t = words.shape
        s = ih * iw
        wc = zeros((b * nc, ndf, t), feat.device)
        attn = zeros((b, nc, t, ih, iw), feat.device)
        sim = torch.empty((b, nc), device=feat.device, dtype=torch.float32)
        _call("og_words_pairs_fwd", _p(words), _p(feat), _p(lens), b, nc, ndf, t, s, float(gamma1), float(gamma2),
              float(eps), _p(wc), _p(attn), _p(sim))
        ctx.cfg = (b, nc, ndf, t, s, float(gamma1), float(gamma2), float(eps))
        ctx.save_for_backward(feat, words, lens, wc, attn)
        ctx.mark_non_differentiable(attn)
        return sim, attn

    @staticmethod
    def backward(ctx, g_sim, _g_attn):
        feat, words, lens, wc, attn = ctx.saved_tensors
        b, nc, ndf, t, s, g1, g2, eps = ctx.cfg
        g_feat = torch.empty_like(feat)
        _call("og_words_pairs_bwd", _p(words), _p(feat), _p(lens), _p(wc), _p(attn), _p(g_sim.contiguous()), b, nc, ndf,
              t, s, g1, g2, eps, _p(g_feat))
        return g_feat, None, None, None, None, None


def words_pairs(feat, words, lens, gamma1, gamma2, eps=1e-8):
    return _WordsPairs.apply(feat, words, lens, gamma1, gamma2, eps)


class _CosineMatrix(torch.autograd.Function):
    """out[i, j] = <a_i, b_j> / max(|a_i| |b_j|, eps) (ref: miscc/losses.py:43-50); ``b`` is a constant."""

    @staticmethod
    def forward(ctx, a, b, eps):
        _chk(a, b)
        a, b = a.contiguous(), b.detach().contiguous()
        out = torch.empty((a.shape[0], b.shape[0]), device=a.device, dtype=torch.float32)
        _call("og_cosine_matrix_fwd", _p(a), _p(b), a.shape[0], b.shape[0], a.shape[1], float(eps), _p(out))
        ctx.eps = float(eps)
        ctx.save_for_backward(a, b)
        return out

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        ga = torch.empty_like(a)
        _call("og_cosine_matrix_bwd", _p(a), _p(b), _p(g.contiguous()), a.shape[0], b.shape[0], a.shape[1], ctx.eps,
              _p(ga))
        return ga, None, None


def cosine_matrix(a, b, eps=1e-8):
    return _CosineMatrix.apply(a, b, eps)


class _CEPair(torch.autograd.Function):
    """(CrossEntropyLoss(scores, labels), CrossEntropyLoss(scores^T, labels), top-1 hits) with scores = gamma3 * sim and
    the masked entries at -inf (ref: miscc/losses.py:50-68, 131-147)."""

    @staticmethod
    def forward(ctx, sim, mask, labels, gamma3):
        _chk(sim, mask, labels)
        sim = sim.contiguous()
        b = sim.shape[0]
        assert sim.shape == (b, b)
        dev = sim.device
        l0 = torch.empty((), device=dev, dtype=torch.float32)
        l1 = torch.empty((), device=dev, dtype=torch.float32)
        hits = torch.empty((), device=dev, dtype=torch.float32)
        g0 = torch.empty((b, b), device=dev, dtype=torch.float32)
        g1 = torch.empty((b, b), device=dev, dtype=torch.float32)
        m = mask.contiguous() if mask is not None else None
        _call("og_ce_pair", _p(sim), _p(m), _p(labels.contiguous()), b, float(gamma3), _p(l0), _p(l1), _p(g0), _p(g1),
              _p(hits))
        ctx.save_for_backward(g0, g1)
        ctx.mark_non_differentiable(hits)
        return l0, l1, hits

    @staticmethod
    def backward(ctx, gl0, gl1, _gc):
        g0, g1 = ctx.saved_tensors
        gsim = torch.empty_like(g0)
        a = gl0.contiguous() if gl0 is not None else None
        b = gl1.contiguous() if gl1 is not None else None
        _call("og_ce_pair_bwd", _p(g0), _p(g1), _p(a), _p(b), g0.numel(), _p(gsim))
        return gsim, None, None, None


def ce_pair(sim, mask, labels, gamma3):
    return _CEPair.apply(sim, mask, labels, gamma3)


class _Bilinear(torch.autograd.Function):
    """F.interpolate(size, mode='bilinear', align_corners=True) on NHWC tensors."""

    @staticmethod
    def forward(ctx, x, oh, ow):
        _chk(x)
        x = x.contiguous()
        n, h, w, c = x.shape
        y = torch.empty((n, oh, ow, c), device=x.device, dtype=torch.float32)
        _call("og_bilinear_fwd", _p(x), n, h, w, c, oh, ow, _p(y))
        ctx.dims = (n, h, w, c, oh, ow)
        return y

    @staticmethod
    def backward(ctx, g):
        n, h, w, c, oh, ow = ctx.dims
        gx = torch.empty((n, h, w, c), device=g.device, dtype=torch.float32)
        _call("og_bilinear_bwd", _p(g.contiguous()), n, h, w, c, oh, ow, _p(gx))
        return gx, None, None


def bilinear(x, oh, ow):
    return _Bilinear.apply(x, oh, ow)


# --------------------------------------------------------------------------------------------------
# ROIAlign (NCHW like the reference op)
# --------------------------------------------------------------------------------------------------
class _RoIAlign(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, rois, ah, aw, scale):
        _chk(features, rois)
        features, rois = features.contiguous(), rois.contiguous()
        assert rois.shape[1] == 5
        b, c, h, w = features.shape
        r = rois.shape[0]
        out = torch.zeros((r, c, ah, aw), device=features.device, dtype=torch.float32)
        _call("ROIAlignForwardLaucher", _p(features), float(scale), r, h, w, c, ah, aw, _p(rois), _p(out))
        ctx.cfg = (b, c, h, w, ah, aw, scale)
        ctx.save_for_backward(rois)
        return out

    @staticmethod
    def backward(ctx, g):
        (rois,) = ctx.saved_tensors
        b, c, h, w, ah, aw, scale = ctx.cfg
        gin = torch.zeros((b, c, h, w), device=g.device, dtype=torch.float32)
        _call("ROIAlignBackwardLaucher", _p(g.contiguous()), float(scale), b, rois.shape[0], h, w, c, ah, aw, _p(rois),
              _p(gin))
        return gin, None, None, None, None


def roi_align(features, rois, ah, aw, scale):
    return _RoIAlign.apply(features, rois, ah, aw, scale)


class _RoIAlignAvg(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, rois, ah, aw, scale):
        _chk(features, rois)
        features, rois = features.contiguous(), rois.contiguous()
        assert rois.shape[1] == 5
        b, c, h, w = features.shape
        r = rois.shape[0]
        out = torch.empty((r, c, ah, aw), device=features.device, dtype=torch.float32)
        _call("og_roi_align_avg_fwd", _p(features), h, w, c, _p(rois), r, ah, aw, float(scale), _p(out))
        ctx.cfg = (b, c, h, w, ah, aw, scale)
        ctx.save_for_backward(rois)
        return out

    @staticmethod
    def backward(ctx, g):
        (rois,) = ctx.saved_tensors
        b, c, h, w, ah, aw, scale = ctx.cfg
        gin = torch.zeros((b, c, h, w), device=g.device, dtype=torch.float32)
        _call("og_roi_align_avg_bwd", _p(g.contiguous()), h, w, c, _p(rois), rois.shape[0], ah, aw, float(scale),
              _p(gin))
        return gin, None, None, None, None


def roi_align_avg(features, rois, ah, aw, scale):
    return _RoIAlignAvg.apply(features, rois, ah, aw, scale)


class _RoIAlignAvgNHWC(torch.autograd.Function):
    """Channels-last fused RoIAlignAvg: features (B, H, W, C) -> (R, ah, aw, C); same values as ``roi_align_avg``."""

    @staticmethod
    def forward(ctx, features, rois, ah, aw, scale):
        _chk(features, rois)
        features, rois = features.contiguous(), rois.contiguous()
        assert rois.shape[1] == 5 and features.shape[3] % 4 == 0
        b, h, w, c = features.shape
        r = rois.shape[0]
        out = torch.empty((r, ah, aw, c), device=features.device, dtype=torch.float32)
        _call("og_roi_align_avg_nhwc_fwd", _p(features), h, w, c, _p(rois), r, ah, aw, float(scale), _p(out))
        ctx.cfg = (b, h, w, c, ah, aw, scale)
        ctx.save_for_backward(rois)
        return out

    @staticmethod
    def backward(ctx, g):
        (rois,) = ctx.saved_tensors
        b, h, w, c, ah, aw, scale = ctx.cfg
        gin = zeros((b, h, w, c), g.device)
        _call("og_roi_align_avg_nhwc_bwd", _p(g.contiguous()), h, w, c, _p(rois), rois.shape[0], ah, aw, float(scale),
              _p(gin))
        return gin, None, None, None, None


def roi_align_avg_nhwc(features, rois, ah, aw, scale):
    return _RoIAlignAvgNHWC.apply(features, rois, ah, aw, scale)


# --------------------------------------------------------------------------------------------------
def adam_ema_(p, g, m, v, avg, step, *, lr=2e-4, b1=0.5, b2=0.999, eps=1e-8, gscale=1.0, decay=0.999, step_dev=None,
              bump=True):
    """Fused Adam (+EMA) over flat fp32 buffers, in place.  ``step_dev`` (int64 device scalar) replaces the host
    step count and is incremented first, which keeps the call replayable from a CUDA graph."""
    _chk(p, g, m, v, avg, step_dev)
    if step_dev is not None:
        _call("og_inc_i64", _p(step_dev))
    _call("og_adam_ema", _p(p), _p(g), _p(m), _p(v), _p(avg), p.numel(), float(lr), float(b1), float(b2), float(eps),
          int(step), _p(step_dev), float(gscale), float(decay))
    if bump:
        bump_param_epoch()


# --------------------------------------------------------------------------------------------------
# Text stage (the text encoder and the word inputs of caption-conditioned sampling).  Inference only.
# --------------------------------------------------------------------------------------------------
def zeros_into(t):
    """t.zero_() through cudaMemsetAsync."""
    _chk(t)
    _call("og_zero_bytes", _p(t), t.numel() * 4)


def copy_channels(src, sstride, dst, dstride, rows):
    """dst[p, :sstride] = src[p, :] for p < rows: row-major src (rows, sstride) into the wider rows of dst."""
    _chk(src, dst)
    _call("og_copy_channels", _p(src.contiguous()), sstride, 0, _p(dst), dstride, 0, sstride, rows, 0)


def add_into(a, b, out):
    """out = a + b elementwise (out: a contiguous view of the same size)."""
    _chk(a, b, out)
    _call("og_add", _p(a.detach().contiguous()), _p(b.detach().contiguous()), _p(out), a.numel())


def linear_rows(x, w, bias, cache):
    """y = x w^T + bias over rows as one 1x1 og_conv2d_simt (exact fp32, no split-K): x (N, cpad(Ci)) with zero pad
    lanes, w (Co, Ci, 1, 1), bias (Co,) -> (N, Co)."""
    _chk(x, w, bias)
    n, c = x.shape
    co, ci = w.shape[:2]
    assert c == cpad(ci) and co % 4 == 0
    wf, _ = cache.get(w, c, co, 0, 0, False)
    y = torch.empty((n, 1, 1, co), device=x.device, dtype=torch.float32)
    return _simt_conv(x.contiguous().view(n, 1, 1, c), wf, y, co, 1, 1, 1, 0, 0, PAD_ZERO, bias,
                      splitk=False).view(n, co)


def lstm_bidir(gx, whh_f, whh_b, cap_lens, max_len):
    """The recurrence of a one-layer bidirectional LSTM (H = 128) in one launch: gx (B*max_len, 8H) x-parts of the gates
    with both biases (og_lstm_bidir), cap_lens (B,) int64 in [1, max_len] on the device -> words_emb (B, 2H, max_len),
    every column t >= cap_lens[b] zero, and sent_emb (B, 2H)."""
    _chk(gx, whh_f, whh_b, cap_lens)
    inference_only("lstm_bidir", gx, whh_f, whh_b)
    h = whh_f.shape[1]
    b = cap_lens.shape[0]
    assert gx.shape == (b * max_len, 8 * h) and whh_f.shape == whh_b.shape == (4 * h, h)
    words = torch.empty((b, 2 * h, max_len), device=gx.device, dtype=torch.float32)
    sent = torch.empty((b, 2 * h), device=gx.device, dtype=torch.float32)
    _call("og_lstm_bidir", _p(gx.contiguous()), _p(whh_f.detach().contiguous()), _p(whh_b.detach().contiguous()),
          _p(_i64(cap_lens)), b, max_len, h, _p(words), _p(sent))
    return words, sent


def text_inputs(captions, glove_captions, glove, max_len):
    """evaluator.py:340-351 on the device: (glove_words_embs (B, E, max_len) = glove[glove_captions[:, :max_len]]
    transposed, mask (B, max_len) bool = (captions == 0)[:, :max_len]) in one launch."""
    _chk(captions, glove_captions, glove)
    c, g = _i64(captions), _i64(glove_captions)
    b, e = c.shape[0], glove.shape[1]
    words = torch.empty((b, e, max_len), device=glove.device, dtype=torch.float32)
    mask = torch.empty((b, max_len), device=glove.device, dtype=torch.uint8)
    _call("og_text_inputs", _p(c), c.shape[1], _p(g), g.shape[1], _p(glove.detach().contiguous()), e, b, max_len,
          _p(words), _p(mask))
    return words, mask.view(torch.bool)


def class_label_emb(glove_weight, cat_labels, cat_label_lens, order):
    """prepare_cat_emb (ref: evaluator.py:148-164, trainer.py:227-241) on the device: over the length-sorted labels
    ``cat_labels`` (N, W) int64 (GloVe ids) and ``cat_label_lens`` (N,) of load.py:305-355, row k is the mean of the
    label's GloVe vectors when it has 1 or 2 tokens and zeros otherwise; the result is indexed by ``order`` (the
    "resort" indices).  Returns (N, E)."""
    lab, lens, order = _i64(cat_labels), _i64(cat_label_lens), _i64(order)
    n, e = order.shape[0], glove_weight.shape[1]
    lab_h, lens_h, order_h = lab.cpu(), lens.cpu(), order.cpu()   # built once per sampler: a host read is cheap here
    read = (torch.arange(lab_h.shape[1]).view(1, -1) < lens_h.view(-1, 1)) & (lens_h <= 2).view(-1, 1)
    if lens_h.shape[0] != lab_h.shape[0] or bool(((lens_h == 2) & (lab_h.shape[1] < 2)).any()):
        raise ValueError("cat_label_lens does not match cat_labels")
    if bool(((lab_h < 0) | (lab_h >= glove_weight.shape[0]))[read].any()):
        raise ValueError("a class label token is outside the GloVe table")
    if bool(((order_h < 0) | (order_h >= lab_h.shape[0])).any()):
        raise ValueError("cat_label_order indexes past the labels")
    _chk(glove_weight, lab, lens, order)
    out = torch.empty((n, e), device=glove_weight.device, dtype=torch.float32)
    _call("og_class_label_emb", _p(glove_weight.detach().contiguous()), e, _p(lab), lab.shape[1], _p(lens), _p(order),
          n, _p(out))
    return out


# --------------------------------------------------------------------------------------------------
# Box stage (the box generator's encoder state, decoder and layout post-processing).  Inference only.
# --------------------------------------------------------------------------------------------------
BOX_NOISE = 6           # per sample and step: u_xy, n1, n2, u_wh, n3, n4


def lstm_bidir_state(gx, whh_f, whh_b, cap_lens, max_len):
    """lstm_bidir that also returns the final cell state: (words_emb (B, 2H, max_len), h (B, 2H), c (B, 2H)), h and c
    with the directions concatenated (forward state after token cap_lens[b]-1, backward state after token 0)."""
    _chk(gx, whh_f, whh_b, cap_lens)
    inference_only("lstm_bidir_state", gx, whh_f, whh_b)
    h = whh_f.shape[1]
    b = cap_lens.shape[0]
    assert gx.shape == (b * max_len, 8 * h) and whh_f.shape == whh_b.shape == (4 * h, h)
    words = torch.empty((b, 2 * h, max_len), device=gx.device, dtype=torch.float32)
    sent = torch.empty((b, 2 * h), device=gx.device, dtype=torch.float32)
    cell = torch.empty((b, 2 * h), device=gx.device, dtype=torch.float32)
    _call("og_lstm_bidir_state", _p(gx.contiguous()), _p(whh_f.detach().contiguous()),
          _p(whh_b.detach().contiguous()), _p(_i64(cap_lens)), b, max_len, h, _p(words), _p(sent), _p(cell))
    return words, sent, cell


def box_label_table(emb, w_ih, b_ih, b_hh):
    """(n_labels, 1024) = b_ih + b_hh + W_ih[:, 100:] emb[l] for every label l (og_box_label_table)."""
    _chk(emb, w_ih, b_ih, b_hh)
    nl = emb.shape[0]
    assert emb.shape[1] == 256 and w_ih.shape == (1024, 356)
    table = torch.empty((nl, 1024), device=emb.device, dtype=torch.float32)
    _call("og_box_label_table", _p(emb.detach().contiguous()), _p(w_ih.detach().contiguous()),
          _p(b_ih.detach().contiguous()), _p(b_hh.detach().contiguous()), nl, _p(table))
    return table


BOX_PACKED = ("table", "wt", "xy_w", "xy_b", "wh_w", "wh_b", "nxy_w", "nxy_b", "lout_t", "lout_b", "xyo_t", "xyo_b",
              "who_t", "who_b")


def box_decode(h0, c0, packed, noise, steps, sos, eos, means, debug=False):
    """Every decoding step of the box decoder in one launch (og_box_decode).  h0 / c0 (B, 256) the encoder state with
    its directions concatenated, ``packed`` the decoder's derived weights (DecoderRNN.packed_weights), noise (B, >=
    steps, 6), ``means`` the first step's (x, y, w, r).  Returns labels (B, steps) int64 (-1 after the end), samples
    (B, steps, 4), steps taken (B,) int64 and, with ``debug``, (B, steps, n_labels + 60): each step's p and both
    mixture parameter sets."""
    nz = noise[:, :steps]
    nz = nz if nz.is_contiguous() else nz.contiguous()
    _chk(h0, c0, nz, *(packed[k] for k in BOX_PACKED))
    inference_only("box_decode", h0, c0)
    b, nl = h0.shape[0], packed["table"].shape[0]
    assert h0.shape == c0.shape == (b, 256) and nz.shape == (b, steps, BOX_NOISE)
    dev = h0.device
    labels = torch.empty((b, steps), device=dev, dtype=torch.int64)
    samples = torch.empty((b, steps, 4), device=dev, dtype=torch.float32)
    taken = torch.empty((b,), device=dev, dtype=torch.int64)
    dbg = torch.empty((b, steps, nl + 60), device=dev, dtype=torch.float32) if debug else None
    _call("og_box_decode", _p(h0.contiguous()), _p(c0.contiguous()), *(_p(packed[k]) for k in BOX_PACKED), _p(nz), b,
          steps, nl, int(sos), int(eos), *(float(m) for m in means), _p(labels), _p(samples), _p(taken), _p(dbg))
    return labels, samples, taken, dbg


def boxes_to_layout(labels, samples, steps, mean_std, label_to_class, count_stats, noise_cnt, boxes_num=10,
                    min_size=10):
    """The evaluator's post-processing of decoder samples and the loader's reading of boxes.txt (ref:
    box_generation/seq2seq/evaluator/evaluator.py:74-139, image_generation/miscc/load.py:653-776) on the device
    (og_box_layout): labels (B, S) int64, samples (B, S, 4) normalised, steps (B,), mean_std (4, 2) float64 (mean, std of
    x, y, w, r), label_to_class (n_labels,) int64 (class row, -1 for the special tokens), count_stats (C, 2) float64
    (mu, sigma of the per-class box count), noise_cnt (B, C) standard normals.  Returns rois (a list of three (B,
    boxes_num, 6) float64 tables at 64, 128 and 256 pixels), fm_rois (B, boxes_num, 6), roi_cls (B, boxes_num) int64 and
    num_rois (B,) int64, zero-padded to boxes_num slots."""
    ms, cs = mean_std.to(torch.float64).contiguous(), count_stats.to(torch.float64).contiguous()
    ncnt = noise_cnt.to(torch.float32).contiguous()
    _chk(labels, samples, steps, ms, label_to_class, cs, ncnt)
    b, s = labels.shape
    nl, c = label_to_class.shape[0], cs.shape[0]
    assert samples.shape == (b, s, 4) and ms.shape == (4, 2) and cs.shape == (c, 2) and ncnt.shape == (b, c)
    dev = labels.device
    rois = torch.empty((3, b, boxes_num, 6), device=dev, dtype=torch.float64)
    fm_rois = torch.empty((b, boxes_num, 6), device=dev, dtype=torch.float64)
    roi_cls = torch.empty((b, boxes_num), device=dev, dtype=torch.int64)
    num_rois = torch.empty((b,), device=dev, dtype=torch.int64)
    _call("og_box_layout", _p(_i64(labels)), _p(samples.contiguous()), _p(_i64(steps)), _p(ms), _p(_i64(label_to_class)),
          _p(cs), _p(ncnt), b, s, nl, c, boxes_num, int(min_size), _p(rois), _p(fm_rois), _p(roi_cls), _p(num_rois))
    return list(rois.unbind(0)), fm_rois, roi_cls, num_rois


def box_records(labels, samples, steps, mean_std, label_to_class, count_stats, noise_cnt):
    """The rows Evaluator.evaluate writes to boxes.txt (ref: box_generation/seq2seq/evaluator/evaluator.py:74-139) on
    the device (og_box_records), from the inputs of ``boxes_to_layout``: rows (B, S, 4) float64 (x, y, w, h, neither
    rounded nor size-filtered, zero after the end), row_cls (B, S) int64 class rows, n_rows (B,), n_valid (B,) the valid
    steps before the last is dropped, and n_special (B,) the boxes dropped for a special label.  All five are views of
    one int64 buffer (``box_records_packed``), so a single copy brings them to the host."""
    return unpack_box_records(box_records_packed(labels, samples, steps, mean_std, label_to_class, count_stats,
                                                 noise_cnt), *labels.shape)


def box_records_packed(labels, samples, steps, mean_std, label_to_class, count_stats, noise_cnt):
    """``box_records``' outputs in one int64 buffer (B*S*5 + 3*B,): the float64 bits of rows, then row_cls, n_rows,
    n_valid and n_special; ``unpack_box_records`` gives the views."""
    ms, cs = mean_std.to(torch.float64).contiguous(), count_stats.to(torch.float64).contiguous()
    ncnt = noise_cnt.to(torch.float32).contiguous()
    _chk(labels, samples, steps, ms, label_to_class, cs, ncnt)
    b, s = labels.shape
    nl, c = label_to_class.shape[0], cs.shape[0]
    assert samples.shape == (b, s, 4) and ms.shape == (4, 2) and cs.shape == (c, 2) and ncnt.shape == (b, c)
    packed = torch.empty((b * s * 5 + 3 * b,), device=labels.device, dtype=torch.int64)
    rows, row_cls, n_rows, n_valid, n_special = unpack_box_records(packed, b, s)
    _call("og_box_records", _p(_i64(labels)), _p(samples.contiguous()), _p(_i64(steps)), _p(ms), _p(_i64(label_to_class)),
          _p(cs), _p(ncnt), b, s, nl, c, _p(rows), _p(row_cls), _p(n_rows), _p(n_valid), _p(n_special))
    return packed


def unpack_box_records(packed, b, s):
    """(rows, row_cls, n_rows, n_valid, n_special) as views of box_records' int64 buffer (on any device)."""
    rows = packed[:b * s * 4].view(torch.float64).view(b, s, 4)
    row_cls = packed[b * s * 4:b * s * 5].view(b, s)
    n_rows, n_valid, n_special = packed[b * s * 5:].view(3, b).unbind(0)
    return rows, row_cls, n_rows, n_valid, n_special


def box_noise(seed, first, b, steps, num_classes, device):
    """The box stage's noise of captions first .. first + b - 1 (og_box_noise): noise_box (b, steps, 6) with uniforms
    in columns 0 and 3 and standard normals elsewhere, noise_cnt (b, num_classes) standard normals.  Each caption's
    values depend only on (seed, its index), not on b or first."""
    if not 0 <= int(seed) < 2 ** 63:
        raise ValueError(f"seed must lie in [0, 2**63), got {seed}")
    nb = torch.empty((b, steps, BOX_NOISE), device=device, dtype=torch.float32)
    nc = torch.empty((b, num_classes), device=device, dtype=torch.float32)
    _call("og_box_noise", int(seed), int(first), b, steps, num_classes, _p(nb), _p(nc))
    return nb, nc


# --------------------------------------------------------------------------------------------------
# Inception-v3 image encoder (CNN_ENCODER, ref: model.py:182-287).  Its convolutions take the tensor cores at every
# kernel shape (1x1, 1xN, Nx1, 3x3, 5x5, valid 3x3 stride 2; conv_path's general form), the exact-fp32 SIMT kernel
# under TC_MIN_PIXELS output pixels or with CONV_ENGINE = "simt".  Eval BatchNorm is folded into the weights and the
# bias (og_bn_fold), ReLU is the LeakyReLU epilogue with slope 0.  The backward computes the input gradient only; the
# encoder is frozen.
# --------------------------------------------------------------------------------------------------
class EncConv:
    """One BasicConv2d (conv without bias -> BatchNorm2d(eps=0.001) in eval mode -> ReLU), or several that read the
    same input fused along N (their weights concatenated), or a plain bias-free conv (``bns`` None, no ReLU).
    ``weights``: OIHW parameters; ``bns``: (gamma, beta, running_mean, running_var) per weight."""

    def __init__(self, weights, bns, kh, kw, stride=1, padh=0, padw=0, eps=1e-3, relu=True):
        self.weights, self.bns = list(weights), (list(bns) if bns is not None else None)
        self.kh, self.kw, self.stride, self.padh, self.padw, self.eps = kh, kw, stride, padh, padw, eps
        self.act = ACT_LRELU if relu else ACT_NONE
        self.cin = self.weights[0].shape[1]
        self.couts = [w.shape[0] for w in self.weights]
        self.cout = sum(self.couts)
        assert self.cout % 8 == 0
        self._key = None
        self.wf = self.bias = self.cache = None

    def folded(self):
        """(folded OIHW weight, folded bias, PackedWeights); recomputed when any source tensor changed."""
        srcs = list(self.weights) + [t for bn in (self.bns or ()) for t in bn]
        key = (_param_epoch[0],) + tuple((t.data_ptr(), t._version) for t in srcs)
        if key != self._key:
            w0 = self.weights[0]
            if self.bns is None and len(self.weights) == 1:
                self.wf, self.bias = w0.detach(), None
            else:
                r = self.cin * self.kh * self.kw
                self.wf = torch.empty((self.cout, self.cin, self.kh, self.kw), device=w0.device, dtype=torch.float32)
                self.bias = torch.empty(self.cout, device=w0.device, dtype=torch.float32)
                off = 0
                for w, (g, b, m, v) in zip(self.weights, self.bns):
                    _chk(w, g, b, m, v)
                    co = w.shape[0]
                    _call("og_bn_fold", _p(w.detach().contiguous()), co, r, _p(g), _p(b), _p(m), _p(v), self.eps,
                          self.wf.data_ptr() + off * r * 4, self.bias.data_ptr() + off * 4)
                    off += co
            self.cache = PackedWeights()          # a new fold is a new operand: its packed copies start empty
            self._key = key
        return self.wf, self.bias, self.cache

    def out_hw(self, h, w):
        return ((h + 2 * self.padh - self.kh) // self.stride + 1, (w + 2 * self.padw - self.kw) // self.stride + 1)

    def macs(self, h, w):
        oh, ow = self.out_hw(h, w)
        return oh * ow * self.cout * self.cin * self.kh * self.kw


def enc_conv_fwd(layer, x, y, yoff=0):
    """y[..., yoff:yoff + layer.cout] = act(conv(x) * s + b): x (N, H, W, cpad(cin)) contiguous, y (N, OH, OW, Cy)."""
    n, h, w, c = x.shape
    assert c == cpad(layer.cin) and y.is_contiguous()
    oh, ow = layer.out_hw(h, w)
    cy = y.shape[3]
    assert y.shape[1:3] == (oh, ow) and yoff + layer.cout <= cy
    wf, bias, cache = layer.folded()
    k = layer.cout
    geo = (n, h, w, layer.kh, layer.kw, layer.stride, layer.padh, layer.padw, PAD_ZERO)
    if conv_path(*geo, k, CONV_ENGINE, general=True) == "simt":
        wp, _ = cache.get(wf, c, k, 0, 0, False)
        _simt_conv(x, wp, y, k, *geo[3:], bias, layer.act, 0.0,
                   bias is None and layer.act == ACT_NONE and yoff == 0 and cy == k, yoff)
    else:
        plan = _tc_plan(FPROP, *geo)
        ws = cache.get_hilo(wf, c, k, 0, 0, 1)                    # [tap][co][ci]
        _tc_launch(_split(x, *plan.xsplit), n, ws, plan, y, k, bias, layer.act, yoff, 0.0)


def enc_conv_dgrad(layer, gp, h, w):
    """Input gradient of the convolution (the epilogue's ReLU already applied to gp (N, OH, OW, cout)); (N, h, w, cpad(cin))."""
    n, oh, ow, k = gp.shape
    c = cpad(layer.cin)
    wf, _, cache = layer.folded()
    gx = torch.empty((n, h, w, c), device=gp.device, dtype=torch.float32)
    geo = (n, h, w, layer.kh, layer.kw, layer.stride, layer.padh, layer.padw, PAD_ZERO)
    if conv_path(*geo, k, CONV_ENGINE, general=True) == "simt":
        _, wt = cache.get(wf, c, k, 0, 0, True)
        _simt_conv(gp, wt, gx, c, *geo[3:8], TRANSPOSED, slope=0.0)
    else:
        plan = _tc_plan(DGRAD, *geo)
        ws = cache.get_hilo(wf, c, k, 0, 0, 0)                    # [tap][ci][co]
        _tc_launch(_split(gp, *plan.gsplit), n, ws, plan, gx, c, slope=0.0)
    return gx


class InceptionProgram:
    """The encoder as a list of steps over named NHWC buffers, run forward and, for the input gradient, backward.

    Steps: ("input", src, dst, size, mode) (og_inception_input: NCHW images to the trunk's NHWC input; forward
    only), ("interp", src, dst, size), ("conv", layer, src, dst, off), ("copy", src, soff, dst, doff, nch),
    ("maxpool", src, dst, off), ("avgpool", src, dst), ("gap", src, dst).  ``chans[name]`` is a buffer's channel
    count (its concatenated width for a block output)."""

    def __init__(self, steps, chans, outputs):
        self.steps, self.chans, self.outputs = steps, chans, outputs

    def forward(self, x):
        bufs = {"x": x}
        for st in self.steps:
            op = st[0]
            if op == "input":
                _, s, d, size, mode = st
                src = bufs[s]
                _chk(src)
                n, c, h, w = src.shape
                assert c == 3 and src.is_contiguous()
                bufs[d] = torch.empty((n, size, size, 8), device=src.device, dtype=torch.float32)
                _call("og_inception_input", _p(src), n, h, w, size, mode, _p(bufs[d]))
            elif op == "interp":
                _, s, d, size = st
                src = bufs[s]
                n, h, w, c = src.shape
                y = torch.empty((n, size, size, c), device=src.device, dtype=torch.float32)
                _call("og_bilinear_fwd", _p(src), n, h, w, c, size, size, _p(y))
                bufs[d] = y
            elif op == "conv":
                _, layer, s, d, off = st
                src = bufs[s]
                if d not in bufs:
                    oh, ow = layer.out_hw(src.shape[1], src.shape[2])
                    bufs[d] = torch.empty((src.shape[0], oh, ow, self.chans[d]), device=src.device, dtype=torch.float32)
                enc_conv_fwd(layer, src, bufs[d], off)
            elif op == "copy":
                _, s, soff, d, doff, nch = st
                src = bufs[s]
                n, h, w, cs = src.shape
                if d not in bufs:
                    bufs[d] = torch.empty((n, h, w, self.chans[d]), device=src.device, dtype=torch.float32)
                _call("og_copy_channels", _p(src), cs, soff, _p(bufs[d]), self.chans[d], doff, nch, n * h * w, 0)
            elif op == "maxpool":
                _, s, d, off = st
                src = bufs[s]
                n, h, w, c = src.shape
                if d not in bufs:
                    bufs[d] = torch.empty((n, (h - 3) // 2 + 1, (w - 3) // 2 + 1, self.chans[d]), device=src.device,
                                          dtype=torch.float32)
                _call("og_maxpool3s2_fwd", _p(src), n, h, w, c, _p(bufs[d]), self.chans[d], off)
            elif op == "avgpool":
                _, s, d = st
                src = bufs[s]
                bufs[d] = torch.empty_like(src)
                n, h, w, c = src.shape
                _call("og_avgpool3s1_fwd", _p(src), n, h, w, c, _p(bufs[d]))
            elif op == "gap":
                _, s, d = st
                src = bufs[s]
                n, h, w, c = src.shape
                bufs[d] = torch.empty((n, c), device=src.device, dtype=torch.float32)
                _call("og_global_avg_fwd", _p(src), n, h * w, c, _p(bufs[d]))
        return bufs

    def backward(self, bufs, grads):
        """grads: {output name: gradient}; returns the gradient of "x".  Each step adds its input gradients in the
        fixed reverse order of the steps."""
        grads = dict(grads)

        def acc(name, t):
            if name in grads:
                _call("og_add", _p(grads[name]), _p(t), _p(grads[name]), t.numel())
            else:
                grads[name] = t

        def acc_slice(name, src_t, src_ld, src_off, nch, doff):
            if name not in grads:
                grads[name] = torch.empty_like(bufs[name])
                zeros_into(grads[name])
            d = grads[name]
            _call("og_copy_channels", _p(src_t), src_ld, src_off, _p(d), d.shape[-1], doff, nch, d.numel() // d.shape[-1],
                  1)

        for st in reversed(self.steps):
            op = st[0]
            if op == "conv":
                _, layer, s, d, off = st
                if d not in grads:
                    continue
                y, g = bufs[d], grads[d]
                n, oh, ow, cy = y.shape
                gp = torch.empty((n, oh, ow, layer.cout), device=y.device, dtype=torch.float32)
                _call("og_relu_grad_slice", _p(y), cy, off, _p(g), cy, off, _p(gp), layer.cout, 0, layer.cout,
                      n * oh * ow, 1 if layer.act == ACT_LRELU else 0)
                src = bufs[s]
                acc(s, enc_conv_dgrad(layer, gp, src.shape[1], src.shape[2]))
            elif op == "copy":
                _, s, soff, d, doff, nch = st
                if d in grads:
                    acc_slice(s, grads[d], self.chans[d], doff, nch, soff)
            elif op == "maxpool":
                _, s, d, off = st
                if d not in grads:
                    continue
                src = bufs[s]
                n, h, w, c = src.shape
                gx = torch.empty_like(src)
                _call("og_maxpool3s2_bwd", _p(src), _p(grads[d]), self.chans[d], off, n, h, w, c, _p(gx))
                acc(s, gx)
            elif op == "avgpool":
                _, s, d = st
                if d not in grads:
                    continue
                n, h, w, c = bufs[s].shape
                gx = torch.empty_like(bufs[s])
                _call("og_avgpool3s1_bwd", _p(grads[d]), n, h, w, c, _p(gx))
                acc(s, gx)
            elif op == "gap":
                _, s, d = st
                if d not in grads:
                    continue
                n, h, w, c = bufs[s].shape
                gx = torch.empty_like(bufs[s])
                _call("og_global_avg_bwd", _p(grads[d].contiguous()), n, h * w, c, _p(gx))
                acc(s, gx)
            elif op == "interp":
                _, s, d, size = st
                if d not in grads:
                    continue
                n, h, w, c = bufs[s].shape
                gx = torch.empty_like(bufs[s])
                _call("og_bilinear_bwd_gather", _p(grads[d]), n, h, w, c, size, size, _p(gx))
                acc(s, gx)
        return grads.get("x")


class _InceptionTrunk(torch.autograd.Function):
    """(x NHWC (N, H, W, 8)) -> the program's outputs; the backward gives the input gradient only, and the forward
    keeps its buffers only when x requires grad."""

    @staticmethod
    def forward(ctx, x, prog):
        _chk(x)
        bufs = prog.forward(x.contiguous())
        ctx.prog = prog
        ctx.bufs = bufs if ctx.needs_input_grad[0] else None
        return tuple(bufs[o] for o in prog.outputs)

    @staticmethod
    def backward(ctx, *gs):
        bufs, prog = ctx.bufs, ctx.prog
        ctx.bufs = None
        grads = {}
        for name, g in zip(prog.outputs, gs):
            if g is not None:
                grads[name] = g.contiguous()
        if not grads:
            return None, None
        return prog.backward(bufs, grads), None


def inception_trunk(x, prog):
    return _InceptionTrunk.apply(x, prog)


def softmax_rows(x):
    """Row softmax of a (rows, C) fp32 tensor (og_softmax_rows)."""
    _chk(x)
    x = x.contiguous()
    y = torch.empty_like(x)
    _call("og_softmax_rows", _p(x), x.shape[0], x.shape[1], _p(y))
    return y


def moments_f64(x, k, s1, s2, init):
    """Adds the rows of x (n, d) fp32 to the fp64 shifted sums (k, s1, s2) of og_moments_f64."""
    _chk(x, k, s1, s2)
    x = x.detach().float().contiguous()
    _call("og_moments_f64", _p(x), x.shape[0], x.shape[1], 1 if init else 0, _p(k), _p(s1), _p(s2))


def images_to_u8(x):
    """(N, 3, H, W) fp32 images in [-1, 1] -> (N, H, W, 3) uint8 on the device (og_images_to_u8): bitwise the
    reference's x.add(1).div(2).mul(255).clamp(0, 255).byte().permute(1, 2, 0) per image (ref: evaluator.py:235-237),
    with NaN -> 0.  A quarter of the float images' bytes crosses to the host for the JPEG encoder."""
    _chk(x)
    x = x.detach().contiguous()
    n, c, h, w = x.shape
    if c != 3 or x.dtype != torch.float32:
        raise ValueError(f"images_to_u8 takes (N, 3, H, W) float32 images, got {tuple(x.shape)} {x.dtype}")
    out = torch.empty((n, h, w, 3), device=x.device, dtype=torch.uint8)
    _call("og_images_to_u8", _p(x), n, h, w, _p(out))
    return out


def snapshot_canvas(images, maps, *, lr_images=None, lens=None, nvis, vis, words, strip, per_map):
    """The pixels of one attention-map snapshot PNG on the device (og_snapshot_canvas; ref: miscc/utils.py:59-306):
    (nvis (strip + 2 vis), (words + 2) (vis + 2), 3) uint8 with the caption strips' backgrounds but no glyphs.
    ``images`` / ``lr_images`` (B, 3, s, s) fp32 in [-1, 1] (None: ``images``), resized to ``vis`` like nn.Upsample
    bilinear; ``maps`` (B, L, att, att) fp32, expanded with pyramid_expand(sigma=20) when vis // att > 1; ``lens``
    int64 (B,) map counts per image (None: L each).  ``per_map``: the shape snapshots' per-map normalisation instead
    of one min / max per image."""
    _chk(images, maps, lr_images, lens)
    for name, t in (("lr_images", lr_images), ("lens", lens)):
        if t is not None and t.device != maps.device:
            raise ValueError(f"snapshot_canvas: {name} is on {t.device}, the maps on {maps.device}")
    if lens is not None and (lens.dim() != 1 or lens.shape[0] < nvis):
        raise ValueError(f"snapshot_canvas: lens must hold >= {nvis} counts, got {tuple(lens.shape)}")
    images = images.detach().contiguous()
    maps = maps.detach().contiguous()
    lr = None if lr_images is None else lr_images.detach().contiguous()
    for name, t in (("images", images), ("lr_images", lr)):
        if t is not None and (t.dim() != 4 or t.shape[1] != 3 or t.shape[2] != t.shape[3] or t.dtype != torch.float32
                              or t.shape[0] < nvis):
            raise ValueError(f"snapshot_canvas: {name} must be (>= {nvis}, 3, s, s) float32, got {tuple(t.shape)} "
                             f"{t.dtype}")
    if maps.dim() != 4 or maps.shape[2] != maps.shape[3] or maps.dtype != torch.float32 or maps.shape[0] < nvis \
            or maps.shape[1] < 1:
        raise ValueError(f"snapshot_canvas: maps must be (>= {nvis}, L >= 1, att, att) float32, got "
                         f"{tuple(maps.shape)} {maps.dtype}")
    L, att = maps.shape[1], maps.shape[2]
    up = vis // att
    if vis % att or not 0 <= words <= 20 or (up > 1 and (vis % 4 or vis <= 80)):
        raise ValueError(f"snapshot_canvas: vis {vis} with {att}-pixel maps and {words} words is not supported")
    if lens is not None:
        _chk(lens)
        lens = lens.to(torch.int64).contiguous()
    dev, m = maps.device, L + 1
    f64 = dict(device=dev, dtype=torch.float64)
    maxmap = torch.empty((nvis, att, att), device=dev, dtype=torch.float32)
    mm0 = torch.empty((nvis, m, 2), **f64)
    stats = torch.empty((nvis, m, 2), **f64)
    work = torch.empty((nvis, m, vis, vis), **f64) if up > 1 else None
    part = torch.empty((nvis, m, vis // 4, 2), **f64) if up > 1 else None
    out = torch.empty((nvis * (strip + 2 * vis), (words + 2) * (vis + 2), 3), device=dev, dtype=torch.uint8)
    _call("og_snapshot_canvas", _p(images), images.shape[2], _p(lr), 0 if lr is None else lr.shape[2], _p(maps), L,
          att, _p(lens), nvis, vis, words, strip, 1 if per_map else 0, _p(maxmap), _p(mm0), _p(work), _p(part),
          _p(stats), _p(out))
    return out
