"""Cost of the attention-map snapshot PNGs at batch 16 (8 images shown), on the device and on the writer's thread.

    python bench_snapshots.py [--iters 20] [--steps 30] [--interval 10] [--rounds 3]

Per PNG kind of a trainer display (G stage 0: 64 -> 128 maps, G stage 1: 128 -> 256, D: 17 -> 272 DAMSM maps) and of
the evaluator's shape PNG (64, no expansion), with CUDA events: the device time of og_snapshot_canvas alone and with
the canvas's copy to pinned host memory; the Gaussian's multiply-adds (2 passes x 161 taps per expanded pixel); and
the host time of one PNG on the writer (read-back wait, caption text, PNG encoding).  For information, the host
oracle's time for the same D PNG.

Then the training loop (condGANTrainer.train_step at batch 16 on bench_train.py's synthetic loader): rounds of
--steps steps with a display every --interval steps, alternated with rounds without displays; host clock to the last
step's device synchronise (the writer is drained after the clock stops).  The cost of one display is the difference
of the two rounds' times over the displays in a round; its share of the loop at DISPLAY_INTERVAL = 500 is that cost
over 500 steps without displays.  A display waits for the writer when the previous one is still queued, so at an
interval of 10 the cost includes that backpressure and bounds the cost at 500 from above.

Prints one JSON line; writes nothing to the tree (PNGs go to a temporary directory)."""
import argparse
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import torch  # noqa: E402
from PIL import Image, ImageFont  # noqa: E402

from objgan_b200 import snapshots  # noqa: E402
from objgan_b200.config import cfg  # noqa: E402

B, WORDS = 16, 18


def kinds():
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.rand(*s, device="cuda", generator=g) * 2 - 1
    maps = lambda L, a: torch.softmax(torch.randn(B, L, a, a, device="cuda", generator=g) * 3, 1)
    lens = torch.randint(1, WORDS + 1, (B,), device="cuda", generator=g)
    return {
        "G_stage0": (lambda i=rnd(B, 3, 128, 128), lr=rnd(B, 3, 64, 64), m=maps(WORDS, 64):
                     snapshots.super_images(i, None, None, m, lr_images=lr), 128, 64, WORDS + 1),
        "G_stage1": (lambda i=rnd(B, 3, 256, 256), lr=rnd(B, 3, 128, 128), m=maps(WORDS, 128):
                     snapshots.super_images(i, None, None, m, lr_images=lr), 256, 128, WORDS + 1),
        "D": (lambda i=rnd(B, 3, 256, 256), m=maps(WORDS, 17): snapshots.super_images(i, None, None, m, lens=lens),
              272, 17, None),
        "shape": (lambda i=rnd(B, 3, 64, 64), m=(rnd(B, 80, 64, 64) + 1) / 2: snapshots.super_shape_images(i, m),
                  64, 64, 81),
    }, lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--interval", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_snapshots.py needs a GPU")
    cfg.TEXT.WORDS_NUM = WORDS
    font = ImageFont.load_default(size=50)
    caps = torch.randint(1, 50, (B, 12))
    words = {i: "word%d" % i for i in range(50)}
    table, lens = kinds()
    res = {"batch": B}
    tmpdir = tempfile.TemporaryDirectory()
    tmp = tmpdir.name
    for name, (fn, vis, att, nmaps) in table.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            c = fn()
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / args.iters
        real_read = snapshots._to_host
        snapshots._to_host = lambda t: (t, None)                 # the kernels alone, without the read-back copy
        try:
            fn()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
        finally:
            snapshots._to_host = real_read
        kernel_ms = e0.elapsed_time(e1) / args.iters
        maps_shown = 8 * nmaps if nmaps is not None else int((lens[:8] + 1).sum())
        macs = 0 if vis == att else maps_shown * vis * vis * 161 * 2
        c = fn()
        c.captions, c.ixtoword, c.font = (None, None, None) if name == "shape" else (caps, words, font)
        t = time.perf_counter()
        Image.fromarray(c.pixels()).save(os.path.join(tmp, name + ".png"))
        host_s = time.perf_counter() - t
        res[name] = {"device_ms": round(dev_ms, 3), "kernel_ms": round(kernel_ms, 3), "blur_gmac": round(macs / 1e9, 3), "host_s": round(host_s, 3),
                     "canvas_mb": round(c.host.numel() / 1e6, 1)}
    for key in ("device_ms", "kernel_ms"):
        res["trainer_display_" + key] = round(2 * res["G_stage0"][key] + 2 * res["G_stage1"][key] + res["D"][key], 3)
    try:
        from oracle import snapshot_oracle as O
        g = torch.Generator().manual_seed(1)
        imgs = torch.rand(B, 3, 256, 256, generator=g) * 2 - 1
        maps = torch.softmax(torch.randn(B, WORDS, 17, 17, generator=g) * 3, 1)
        t = time.perf_counter()
        O.super_images(imgs, caps, words, maps, 17, words=WORDS, font=font)
        res["oracle_host_D_s"] = round(time.perf_counter() - t, 2)
    except ImportError:
        pass
    res["loop"] = loop_rounds(args, font)
    tmpdir.cleanup()
    from bench_sample import _card
    res["gpu"], res["power_limit"] = _card()
    print(json.dumps(res))


def loop_rounds(args, font):
    import random
    import statistics
    from bench_train import NTOKEN, _loader
    from objgan_b200 import model, synth, trainer
    loader = _loader(B, 2)
    with tempfile.TemporaryDirectory() as tmp:
        torch.manual_seed(0)
        fast, model.FAST_INIT = model.FAST_INIT, True
        try:
            cfg.TRAIN.update(NET_E=synth.reference_encoders(tmp, n_words=NTOKEN), NET_G="", BATCH_SIZE=B)
            ds = synth.reference_dataset(n_words=NTOKEN, n_glove=NTOKEN)
            ds.ixtoword = {i: "word%d" % i for i in range(NTOKEN)}
            t = trainer.condGANTrainer(os.path.join(tmp, "out"), loader, ds,
                                       inception_weights=model._Inception3().state_dict(), device="cuda:0", font=font)
            t.setup()
        finally:
            model.FAST_INIT = fast
        random.seed(0)

        def run(display):
            writer = snapshots.PngWriter()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k in range(1, args.steps + 1):
                t.train_step(loader[k % len(loader)])
                if display and k % args.interval == 0:
                    t.save_img_results(0, writer)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            writer.close()
            return dt

        run(True)                                              # warm-up: every shape of both kinds of round
        times = {"display": [], "plain": []}
        for _ in range(args.rounds):
            times["display"].append(run(True))
            times["plain"].append(run(False))
    med = {k: statistics.median(v) for k, v in times.items()}
    n = args.steps // args.interval
    step_s = med["plain"] / args.steps
    per_display = (med["display"] - med["plain"]) / n
    return {"steps": args.steps, "interval": args.interval, "displays_per_round": n,
            "rounds_display_s": [round(v, 3) for v in times["display"]],
            "rounds_plain_s": [round(v, 3) for v in times["plain"]],
            "step_ms": round(step_s * 1e3, 2), "display_cost_s": round(per_display, 3),
            "share_at_interval_500": round(per_display / (500 * step_s), 5)}


if __name__ == "__main__":
    main()
