"""Box-conditioned sampling throughput (GSampler with a shape generator: box maps -> SHP_G_NET -> generated heat maps ->
G_NET) at batch 1 and 16 with 10 rois per image.  Prints one JSON line.

    python bench_sample_shapes.py [--batches 1,16] [--seconds 3] [--rounds 3]

Reported per batch:
  * images/s of the whole box-conditioned sample, eager against CUDA-graph replay, alternated in rounds (as
    bench_sample.py does; CUDA events around a window of back-to-back calls, device-resident seeded inputs);
  * the shape stage alone (box maps + SHP_G_NET + form_gen_hmaps, eager), ms per batch from CUDA events;
  * SHP_G_NET's algorithmic GMAC (the reference's direct form: every roi slot, the full 480-channel Gates conv at every
    step), computed from the layer shapes below, and the TFLOP/s that the shape stage's time gives it;
  * the largest difference between the replayed and the eager outputs, and whether they are bitwise equal;
  * the card name and power limit.
Needs a GPU; writes nothing."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_sample import _card, _rate  # noqa: E402


def shp_g_net_gmac(net, rmax, size=64):
    """Multiply-accumulates of one SHP_G_NET forward per image with rmax roi slots (ref: model.py:920-985), in GMAC."""
    fm = net.fm_size
    conv = lambda w, hw: w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3] * hw * hw
    per_slot = 2 * conv(net.downsample1[0].weight, size // 2) + 2 * conv(net.downsample2[0].weight, fm)   # fwd + bwd
    per_slot += conv(net.fwd_convlstm.Gates.weight, fm) + conv(net.bwd_convlstm.Gates.weight, fm)
    per_slot += conv(net.jointConv[0].weight, fm)
    for blk in net.residual:
        per_slot += sum(conv(blk.block[i].weight, fm) for i in (0, 3, 6))
    per_slot += conv(net.upsample1[1].weight, 2 * fm) + conv(net.upsample2[1].weight, 4 * fm)
    per_slot += conv(net.img_net.img[0].weight, size)
    return per_slot * rmax / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from objgan_b200 import lib, model, ops, synth
    from objgan_b200.sampler import GSampler
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_shapes.py needs a CUDA device")
    torch.manual_seed(0)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    shp = model.SHP_G_NET(80)
    shp.apply(model.weights_init)
    s = GSampler(g.to("cuda"), shp.to("cuda"))
    res = {"bench": "gsampler_shapes", "gpu": None, "power_limit": None, "conv_engine": ops.CONV_ENGINE, "rois": 10,
           "batches": {}}
    res["gpu"], res["power_limit"] = _card()
    flat = lambda o: [*o[0], *o[1], *o[2], *o[3], o[4], o[5]]
    for b in [int(x) for x in a.batches.split(",")]:
        x = synth.compact(synth.make_inputs(b, seed=100 + b))
        for k in ("bt_masks", "fm_bt_masks"):
            x.pop(k)
        x["noise_shp"] = torch.randn(b, 10, 320, generator=torch.Generator().manual_seed(b))
        dev = {k: (v.cuda() if torch.is_tensor(v) else [t.cuda() for t in v] if isinstance(v, list) else v)
               for k, v in x.items()}
        s.sample(dev)                          # eager warm-up + capture
        s.sample(dev)
        n0 = lib.get().launches
        eager = s.sample_eager(dev)
        calls = lib.get().launches - n0
        replay = s.sample(dev)
        torch.cuda.synchronize()
        diff = max(((p - q).abs().max() / q.abs().max().clamp(min=1e-30)).item()
                   for p, q in zip(flat(replay), flat(eager)) if q.numel())
        exact = all(torch.equal(p, q) for p, q in zip(flat(replay), flat(eager)))
        # the shape stage alone
        with torch.no_grad():
            prep = s._prepare(dev)
            for _ in range(3):
                s._shapes(prep)
            n_iter = 20 if b > 1 else 50
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(n_iter):
                s._shapes(prep)
            end.record()
            end.synchronize()
        shape_ms = start.elapsed_time(end) / n_iter
        gmac = shp_g_net_gmac(s.netShpG, 10) * b
        rates = {"eager": [], "graph": []}
        for _ in range(a.rounds):
            rates["eager"].append(_rate(lambda: s.sample_eager(dev), b, a.seconds))
            rates["graph"].append(_rate(lambda: s.sample(dev), b, a.seconds))
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["batches"][str(b)] = {
            "eager_img_s": round(med["eager"], 2), "graph_img_s": round(med["graph"], 2),
            "speedup": round(med["graph"] / med["eager"], 3),
            "eager_rounds": [round(r, 2) for r in rates["eager"]], "graph_rounds": [round(r, 2) for r in rates["graph"]],
            "shape_stage_ms": round(shape_ms, 3), "shp_g_net_gmac": round(gmac, 2),
            "shape_stage_tflops": round(2 * gmac / (shape_ms * 1e-3) / 1e3, 2),
            "calls_per_sample": calls, "max_rel_diff_replay_vs_eager": diff, "replay_bitwise_equal": exact}
        del dev, eager, replay, prep
    print(json.dumps(res))


if __name__ == "__main__":
    main()
