"""Training-loop throughput: trainer.condGANTrainer's step (batch intake, copies to the device, heat-map rebuild, text
stage, complete step, INCEPTION_V3 on the 256-pixel images) against StepBTrainer.step alone on inputs staged on the
device beforehand.  Prints one JSON line.

    python bench_train.py [--batch 16] [--steps 10] [--warmup 3] [--rounds 3]

The loader is synthetic and in the reference's tuple format (what its DataLoader collates from TrainDataset): batch 16,
18-token captions of mixed lengths, 10 rois per image, float64 heat maps and masks, pinned (all but the heat maps,
which the intake never reads), generated before timing (--distinct different batches, cycled).  The DAMSM encoders and Inception weights are seeded, not pretrained: the
work per step does not depend on the values.  Reported:
  * images/s of the loop step and of the bare Step-B step, alternated in rounds (host clock around --steps steps
    that end in a device synchronise), medians and every round;
  * the intake (prepare_reference_batch) alone: host ms per batch, and its share of the loop's step time;
  * the card name and power limit.
Per-epoch work (the score file and snapshots) is outside the timed steps.  Needs a GPU; writes only to a temporary
directory."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_sample import _card  # noqa: E402

NTOKEN = 30000


def _loader(b, n):
    """n reference-format batches, pinned as DataLoader(pin_memory=True) leaves them, except the float64 heat maps
    (about 880 MB a batch at 16, never read by the intake): one unpinned set is shared by every batch, which keeps the
    host memory of the benchmark near 1.5 GB."""
    import torch
    from objgan_b200 import synth
    pin = lambda t: t.pin_memory() if torch.is_tensor(t) else [pin(x) for x in t] if isinstance(t, list) and \
        t and torch.is_tensor(t[0]) else t
    out = []
    for i in range(n):
        data = synth.reference_batch(b, seed=1000 + i, parity=False, n_words=NTOKEN, n_glove=NTOKEN)
        hmaps = data[4] if i == 0 else out[0][4]
        out.append(tuple(hmaps if k == 4 else pin(x) for k, x in enumerate(data)))
        del data
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=2)
    a = ap.parse_args()
    import random

    import torch
    from objgan_b200 import losses, model, ops, synth, trainer
    from objgan_b200.config import cfg
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py needs a CUDA device")
    torch.cuda.set_device(0)
    b = a.batch
    loader = _loader(b, a.distinct)
    with tempfile.TemporaryDirectory() as tmp:
        torch.manual_seed(0)
        fast, model.FAST_INIT = model.FAST_INIT, True
        try:
            cfg.TRAIN.update(NET_E=synth.reference_encoders(tmp, n_words=NTOKEN), NET_G="", BATCH_SIZE=b)
            inception = model._Inception3().state_dict()
            t = trainer.condGANTrainer(os.path.join(tmp, "out"), loader,
                                       synth.reference_dataset(n_words=NTOKEN, n_glove=NTOKEN),
                                       inception_weights=inception, device="cuda:0")
            t.setup()
        finally:
            model.FAST_INIT = fast
        random.seed(0)
        # the bare step's inputs: everything the loop does before StepBTrainer.step, done once per distinct batch
        staged = []
        for data in loader:
            batch, class_ids, _ = trainer.prepare_reference_batch(data)
            dev = t.net.to_device(dict(batch, clabels_emb=t.clabels_emb))
            with torch.no_grad():
                dev.update(trainer.text_stage(t.text_encoder, t.glove, dev["captions"], dev["cap_lens"],
                                              dev["glove_captions"], batch["max_len"]))
            dev["z"] = torch.randn(b, cfg.GAN.Z_DIM, device="cuda")
            staged.append((dev, class_ids))
        torch.cuda.synchronize()
        score = [None]

        def loop(k):
            t.train_step(loader[k % len(loader)], score[0])

        def bare(k):
            dev, cids = staged[k % len(staged)]
            t.net.step(dev, cids)

        def rate(fn):
            for k in range(a.warmup):
                fn(k)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k in range(a.steps):
                fn(k)
            torch.cuda.synchronize()
            return a.steps * b / (time.perf_counter() - t0)

        rates = {"loop": [], "step_b": []}
        for _ in range(a.rounds):
            score[0] = losses.InceptionScore(min(10, b))
            rates["loop"].append(rate(loop))
            rates["step_b"].append(rate(bare))
        # the intake alone, on the host (no device work in flight)
        for data in loader:
            trainer.prepare_reference_batch(data)
        reps = 5 * len(loader)
        t0 = time.perf_counter()
        for k in range(reps):
            trainer.prepare_reference_batch(loader[k % len(loader)])
        intake_ms = (time.perf_counter() - t0) * 1e3 / reps
    med = {k: statistics.median(v) for k, v in rates.items()}
    loop_ms = b / med["loop"] * 1e3
    gpu, power = _card()
    res = {"bench": "train_loop", "gpu": gpu, "power_limit": power, "conv_engine": ops.CONV_ENGINE, "batch": b,
           "rois": cfg.ROI.BOXES_NUM, "words_num": cfg.TEXT.WORDS_NUM, "steps": a.steps, "warmup": a.warmup,
           "loop_img_s": round(med["loop"], 3), "step_b_img_s": round(med["step_b"], 3),
           "loop_vs_step_b": round(med["loop"] / med["step_b"], 4),
           "loop_ms_per_step": round(loop_ms, 2), "step_b_ms_per_step": round(b / med["step_b"] * 1e3, 2),
           "loop_rounds": [round(v, 3) for v in rates["loop"]], "step_b_rounds": [round(v, 3) for v in rates["step_b"]],
           "intake_host_ms_per_batch": round(intake_ms, 3), "intake_share_of_loop_step": round(intake_ms / loop_ms, 4),
           "batch_bytes_from_loader": int(sum(x.numel() * x.element_size() for v in loader[0] for x in
                                              (v if isinstance(v, list) else [v]) if torch.is_tensor(x)))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
