#!/usr/bin/env python
"""bench_conv.py -- the hot tensor-core convolutions of Step-A, one at a time, and where a whole step's time goes.

    python bench_conv.py                         # fprop / dgrad / wgrad of each layer below (3xFP16)
    python bench_conv.py --step-profile DIR      # torch.profiler over eager Step-A steps (in a run of its own)
    python bench_conv.py --cta-cost              # the conv1 forward's fixed cost per CTA (two channel counts)

Per convolution and direction: ms per call (CUDA events around back-to-back calls, median of three windows, the
spread beside it), algorithmic TFLOP/s (the layer as the model writes it: real channels, every tap of the kernel on
the output grid -- 9 taps of the 2x-upsampled map for the upBlock) and issued TFLOP/s (3 MMAs per product on the
padded M x N x K that the launched tiles cover; the upBlock's four-phase form issues 4 taps per output pixel, not 9).
The operand split of the input (og_prep_split) is done once, outside the timed calls; the input gradient of a
reflection-padded layer includes its small og_reflect_pad_bwd pass, and the weight gradient its fixed-order partial
sum and unpack passes.  Each call reads one of several input sets, together larger than the 50 MB L2.  For the
column-order 3x3 layers the forward and input gradient also report their operand bytes from L2 per call, computed
from the tile geometry, in the per-tap form of conv_tc_kernel and the row-run form of conv_tc_rows_kernel.

--step-profile: batch 16 (bench.py's configuration), eager launches (kernels inside graph replays are not recorded
separately), 2 warm-up steps and 3 profiled ones; prints the GPU time per kernel name and grid, and the share of the
convolution kernels; the trace is written to DIR.  Results go to stdout as text and one JSON line at the end.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

L2_BYTES = 50 << 20

# name, cin, cout, kernel, stride, mode ("reflect", "zero", "up"), GLU split, N, H, W (input extent)
LAYERS = [
    ("hmap_res.conv1 194->388 @128", 194, 388, 3, 1, "reflect", 194, 16, 128, 128),
    ("hmap_res.conv2 194->194 @128", 194, 194, 3, 1, "reflect", 0, 16, 128, 128),
    ("hmap_res.conv1 194->388 @64", 194, 388, 3, 1, "reflect", 194, 16, 64, 64),
    ("hmap_res.conv2 194->194 @64", 194, 194, 3, 1, "reflect", 0, 16, 64, 64),
    ("g_hmap 80->24 @256", 80, 24, 3, 1, "reflect", 0, 16, 256, 256),
    ("img head 48->3 @256", 48, 3, 3, 1, "zero", 0, 16, 256, 256),
    ("upblock 194->96 @256", 194, 96, 3, 1, "up", 48, 16, 128, 128),
    ("patd256.0 3->96 s2 @256", 3, 96, 4, 2, "zero", 0, 16, 256, 256),
    ("patd256.2 96->192 s2 @128", 96, 192, 4, 2, "zero", 0, 16, 128, 128),
    ("patd256.5 192->384 s2 @64", 192, 384, 4, 2, "zero", 0, 16, 64, 64),
    ("patd256.8 384->768 s2 @32", 384, 768, 4, 2, "zero", 0, 16, 32, 32),
]


def card():
    """Card name and power limit, read-only."""
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": q}


# ---------------------------------------------------------------- tile geometry of conv_tc.cu (issued work)
BN_SET = (32, 48, 64, 96, 104, 112, 128)


def _patch(oh, ow):
    tw = 1
    while tw * 2 <= ow and tw * 2 <= 16:
        tw *= 2
    th = 1
    while th * 2 <= oh and tw * th * 2 <= 128:
        th *= 2
    return 128 // (tw * th), th, tw


def issued_tc(n, oh, ow, c, k, ntaps):
    """Issued MMA flops of one og_conv2d_tc launch: GEMM rows n x oh x ow, c input channels, k output channels."""
    tn, th, tw = _patch(oh, ow)
    m = math.ceil(n / tn) * math.ceil(oh / th) * math.ceil(ow / tw) * 128
    cchunks = math.ceil(c / 64)
    kred = ntaps * ((cchunks - 1) * 64 + math.ceil((c - (cchunks - 1) * 64) / 16) * 16)
    ntile = math.ceil(k / 128)
    bn8 = (math.ceil(k / ntile) + 7) // 8 * 8
    bn = next((b for b in BN_SET if b >= bn8), 128)
    if bn == 32 and k <= 32:                       # stacked [w_hi | w_lo]: two MMAs of twice the width
        return 2 * 2.0 * m * (32 if k <= 16 else 64) * kred
    return 3 * 2.0 * m * math.ceil(k / bn) * bn * kred


def operand_bytes_tc(n, oh, ow, c, k, ntaps, run=1):
    """L2 -> shared-memory operand bytes of one og_conv2d_tc launch, from its tile geometry: per (tap, 64-channel
    chunk) stage every CTA loads an A tile (hi + lo) of its 128 pixels and a B tile (hi + lo) of its output columns.
    run = 3: conv_tc_rows_kernel's form, one A box of TH + 2 rows per run of three taps and chunk.  Real channels and
    output columns only (TMA fills the rest of a partial chunk or tile without reading); pixels outside the source are
    counted as read."""
    tn, th, tw = _patch(oh, ow)
    ptiles = math.ceil(n / tn) * math.ceil(oh / th) * math.ceil(ow / tw)
    ntile = math.ceil(k / 128)
    bn = next((b for b in BN_SET if b >= (math.ceil(k / ntile) + 7) // 8 * 8), 128)
    a_pix = 128 if run == 1 else (th + run - 1) * tw
    a = ptiles * math.ceil(k / bn) * (ntaps // run) * a_pix * c * 2 * 2
    b = ptiles * ntaps * k * c * 2 * 2
    return a + b


def issued_wgrad(n, oh, ow, kp, c, entries):
    """Issued MMA flops of one og_conv2d_wgrad_tc launch over an oh x ow gradient grid of n images."""
    cw = 1
    while cw * 2 <= 64 and ow % (cw * 2) == 0:
        cw *= 2
    chh = 1
    while cw * chh * 2 <= 64 and oh % (chh * 2) == 0:
        chh *= 2
    cn = 64 // (cw * chh)
    pix = (ow // cw) * (oh // chh) * math.ceil(n / cn) * 64
    ntile = math.ceil(c / 128)                     # ci tiles fitted like the forward's N tile
    bnw = next((b for b in BN_SET if b >= (math.ceil(c / ntile) + 7) // 8 * 8), 128)
    rows = math.ceil(kp / 64) * 64                 # a 64-row co slab wholly past kp issues nothing
    return 3 * 2.0 * rows * ntile * bnw * pix * entries


def layer_work(cin, cout, k, stride, mode, split, n, h, w):
    """(algorithmic flops, {direction: issued flops}) of one layer."""
    from objgan_b200 import ops
    c = ops.cpad(cin)
    kp = 2 * ops.cpad(split) if split else ops.cpad(cout)
    if mode == "up":
        oh, ow = 2 * h, 2 * w
        alg = 2.0 * n * oh * ow * cout * cin * 9
        iss = {"fprop": 4 * issued_tc(n, h, w, c, kp, 4),
               "dgrad": issued_tc(n, h, w, kp, c, 16),
               "wgrad": issued_wgrad(n, h, w, kp, c, 16)}
    elif stride == 2:
        oh, ow = h // 2, w // 2
        alg = 2.0 * n * oh * ow * cout * cin * k * k
        iss = {"fprop": issued_tc(n, oh, ow, c, kp, k * k),
               "dgrad": 4 * issued_tc(n, oh, ow, kp, c, (k // 2) ** 2),
               "wgrad": issued_wgrad(n, oh, ow, kp, c, k * k)}
    else:
        oh, ow = h, w
        alg = 2.0 * n * oh * ow * cout * cin * k * k
        halo = 2 if mode == "reflect" else 0           # the reflect dgrad writes the padded extent
        iss = {"fprop": issued_tc(n, oh, ow, c, kp, k * k),
               "dgrad": issued_tc(n, h + halo, w + halo, kp, c, k * k),
               "wgrad": issued_wgrad(n, oh, ow, kp, c, k * k)}
    return alg, iss


# ---------------------------------------------------------------- per-layer timing
def _time(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def bench_layer(spec, window_ms, dirs=("fprop", "dgrad", "wgrad")):
    from objgan_b200 import model, ops
    from objgan_b200.lib import ACT_NONE, PAD_REFLECT, PAD_ZERO, UPSAMPLE2X
    name, cin, cout, k, stride, mode_s, split, n, h, w = spec
    mode = {"reflect": PAD_REFLECT, "zero": PAD_ZERO, "up": UPSAMPLE2X}[mode_s]
    torch.manual_seed(cin * 1000 + cout)
    m = model.Conv2dP(cin, cout, k, stride, 1, mode=mode, split=split).cuda()
    c = ops.cpad(cin)
    splitp = ops.cpad(split) if split else 0
    kp = 2 * splitp if split else ops.cpad(cout)
    path = ops.conv_path(n, h, w, k, k, stride, 1, 1, mode, kp, "f16x3")
    assert path in ("s1", "s2"), f"{name}: not a tensor-core shape"
    oh, ow = ops._out_hw(h, w, k, k, stride, 1, mode)
    geo = ops._conv2d_geo(n, h, w, k, k, stride, 1, mode)
    plan = ops._tc_plan(ops.FPROP, *geo)
    per_set = 2 * 2 * (n * h * w * c + n * oh * ow * kp)          # hi + lo copies of x and of g
    nsets = max(1, math.ceil(2 * L2_BYTES / per_set))
    sets = []
    for _ in range(nsets):
        x = torch.randn(n, h, w, c, device="cuda")
        x[..., cin:] = 0
        xs = ops._split(x, *plan.xsplit)
        x.og_split = (*xs, *plan.xsplit, x._version)  # fprop reuses these copies: no split pass timed
        g = torch.randn(n, oh, ow, kp, device="cuda")
        gs = ops._split(g, *plan.gsplit)
        sets.append((x, xs, gs))
    wt, cache = m.weight, m._cache
    calls = {
        "fprop": lambda i: ops._tc_fprop(sets[i % nsets][0], cache, wt, kp, split, splitp, geo, None, ACT_NONE),
        "dgrad": lambda i: ops._tc_dgrad(sets[i % nsets][2], cache, wt, c, kp, split, splitp, geo),
        "wgrad": lambda i: ops._tc_wgrad(sets[i % nsets][1], sets[i % nsets][2], wt, c, kp, split, splitp, geo),
    }
    alg, iss = layer_work(cin, cout, k, stride, mode_s, split, n, h, w)
    nbytes = {}
    if k == 3 and stride == 1 and mode_s != "up":    # the two forms of a column-order 3x3 tap list
        halo = 2 if mode_s == "reflect" else 0
        for d, geo_d in (("fprop", (n, oh, ow, c, kp)), ("dgrad", (n, h + halo, w + halo, kp, c))):
            nbytes[d] = {"operand_MB_per_tap": round(operand_bytes_tc(*geo_d, 9) / 1e6, 1),
                         "operand_MB_row_runs": round(operand_bytes_tc(*geo_d, 9, 3) / 1e6, 1)}
    out = {}
    with torch.no_grad():
        for d, fn in calls.items():
            if d not in dirs:
                continue
            for i in range(2 * nsets):
                fn(i)
            torch.cuda.synchronize()
            est = _time(fn, nsets)
            reps = max(nsets, min(500, math.ceil(window_ms / max(est, 1e-3))))
            ms = sorted(_time(fn, reps) for _ in range(3))
            out[d] = {"ms": round(ms[1], 4), "ms_min": round(ms[0], 4), "ms_max": round(ms[2], 4),
                      "alg_tflops": round(alg / (ms[1] * 1e-3) / 1e12, 2),
                      "issued_tflops": round(iss[d] / (ms[1] * 1e-3) / 1e12, 1), "reps": reps, **nbytes.get(d, {})}
    return out


# ---------------------------------------------------------------- fixed cost per CTA of the forward
# The res-block conv1 forward with 192 and with 384 input channels: the same CTAs (pixel tiles x 4 N tiles of 104),
# each with 27 resp. 54 stages of 4 k-steps.  With t = F + S (F: per-CTA set-up, fill and epilogue; S: the stages),
# F = 2 t192 - t384.
CTA_COST = [("conv1 fprop 192->388 @128", 192, 388, 3, 1, "reflect", 194, 16, 128, 128),
            ("conv1 fprop 384->388 @128", 384, 388, 3, 1, "reflect", 194, 16, 128, 128)]


def cta_cost(window_ms):
    t1, t2 = (bench_layer(spec, window_ms, ("fprop",))["fprop"]["ms"] for spec in CTA_COST)
    fixed = 2 * t1 - t2
    print(f"conv1 fprop: {t1:.3f} ms at 192 channels, {t2:.3f} ms at 384; fixed per-CTA part {fixed:.3f} ms "
          f"= {fixed / t1:.1%} of the 192-channel time")
    return {"ms_192": t1, "ms_384": t2, "fixed_ms": round(fixed, 4), "fixed_share_192": round(fixed / t1, 4)}


# ---------------------------------------------------------------- step profile
def step_profile(out_dir, steps=3, warmup=2):
    from torch.profiler import ProfilerActivity, profile
    from objgan_b200 import synth, trainer
    os.makedirs(out_dir, exist_ok=True)
    tr = trainer.StepATrainer(device="cuda:0", seed=1234)
    full = synth.make_inputs(16, seed=1234, parity=False)
    full.pop("eps")
    dev = tr.to_device(trainer.pin(synth.compact(full)))
    for _ in range(warmup):
        tr.step(dev)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        for _ in range(steps):
            tr.step(dev)
        e1.record()
        torch.cuda.synchronize()
    wall = e0.elapsed_time(e1) / steps
    trace = os.path.join(out_dir, "step_a.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    rows = {}
    for ev in events:
        if ev.get("cat") != "kernel":
            continue
        key = (ev["name"], str(ev.get("args", {}).get("grid")))
        r = rows.setdefault(key, [0.0, 0])
        r[0] += ev["dur"] / 1e3 / steps
        r[1] += 1
    total = sum(r[0] for r in rows.values())
    conv = sum(r[0] for (nm, _), r in rows.items() if "conv_tc" in nm)
    conv_all = sum(r[0] for (nm, _), r in rows.items() if "conv" in nm)
    top = sorted(rows.items(), key=lambda kv: -kv[1][0])
    print(f"\nStep-A, batch 16, eager: {wall:.2f} ms per step (wall, profiler on); kernel time {total:.2f} ms per step")
    print(f"tensor-core conv kernels (conv_tc*): {conv:.2f} ms = {conv / total:.1%} of kernel time; every kernel "
          f"with 'conv' in its name: {conv_all:.2f} ms = {conv_all / total:.1%}")
    print(f"{'ms/step':>8} {'share':>6} {'calls':>5}  kernel [grid]")
    for (nm, grid), (ms, cnt) in top[:40]:
        short = nm if len(nm) < 110 else nm[:107] + "..."
        print(f"{ms:8.3f} {ms / total:6.1%} {cnt // steps:5d}  {short} {grid}")
    return {"wall_ms_per_step": round(wall, 2), "kernel_ms_per_step": round(total, 2),
            "conv_tc_ms_per_step": round(conv, 2), "conv_tc_share_of_kernel_time": round(conv / total, 4),
            "conv_any_share_of_kernel_time": round(conv_all / total, 4), "trace": trace,
            "top": [{"kernel": nm, "grid": grid, "ms_per_step": round(ms, 4), "calls_per_step": cnt // steps}
                    for (nm, grid), (ms, cnt) in top[:40]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--step-profile", metavar="DIR", help="profile whole Step-A steps instead; trace written to DIR")
    ap.add_argument("--window-ms", type=float, default=200.0, help="GPU time per timing window")
    ap.add_argument("--layers", default="", help="comma-separated substrings selecting layers (default: all)")
    ap.add_argument("--cta-cost", action="store_true", help="split the conv1 forward into per-CTA and per-stage time")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_conv.py needs a CUDA device"
    torch.cuda.set_device(0)
    from objgan_b200 import ops
    assert ops.CONV_ENGINE == "f16x3", "measures the parity engine (OBJGAN_CONV=f16x3)"
    res = {"card": card()}
    if args.step_profile:
        res["step_profile"] = step_profile(args.step_profile)
    elif args.cta_cost:
        res["cta_cost"] = cta_cost(args.window_ms)
    else:
        sel = [s for s in args.layers.split(",") if s]
        res["layers"] = {}
        print(f"{'layer':32s} {'dir':5s} {'ms':>8s} {'(min-max)':>17s} {'alg TF/s':>9s} {'issued TF/s':>11s}")
        for spec in LAYERS:
            if sel and not any(s in spec[0] for s in sel):
                continue
            r = bench_layer(spec, args.window_ms)
            res["layers"][spec[0]] = r
            for d, v in r.items():
                mb = (f"  operand MB per call: {v['operand_MB_per_tap']} per-tap A, {v['operand_MB_row_runs']} row runs"
                      if "operand_MB_per_tap" in v else "")
                print(f"{spec[0]:32s} {d:5s} {v['ms']:8.3f} ({v['ms_min']:7.3f}-{v['ms_max']:7.3f}) "
                      f"{v['alg_tflops']:9.1f} {v['issued_tflops']:11.1f}{mb}")
    print(f"card: {res['card']}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
