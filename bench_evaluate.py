"""Evaluation-loop throughput: evaluator.condGANEvaluator's batch (intake, eager sampling with the text stage,
CNN_ENCODER + RPrecision, INCEPTION_V3 + InceptionScore, INCEPTION_V3_FID + FrechetDistance) against the bare loop on
inputs staged on the device beforehand (GSampler.sample_eager, encode_image + RPrecision, score_images +
InceptionScore + FrechetDistance).  Prints one JSON line per mode.

    python bench_evaluate.py [--batch 16] [--steps 10] [--warmup 3] [--rounds 3] [--modes 2,0]

The loader is synthetic and in the reference's test tuple format (what its DataLoader collates from TestDataset):
18-token captions of mixed lengths, 10 rois per image, float64 activations, masks and box tables, pinned.  The box
maps and heat maps, which the intake never reads, are zero-stride views of their shapes, which keeps the host memory
of the benchmark small.  Networks and Inception weights are seeded, not trained: the work per batch does not depend
on the values.  Reported per mode (cfg.TEST.USE_GT_BOX_SEG 2: generated boxes and shapes, the reference's default;
0: ground-truth boxes and masks):
  * images/s of the evaluator's batch and of the bare loop, alternated in rounds (host clock around --steps batches
    that end in a device synchronise), medians and every round;
  * the intake (prepare_reference_test_batch) alone: host ms per batch, and its share of the evaluator's batch time;
  * the card name and power limit.
No image files are written (DISPLAY_INTERVAL larger than the run).  Needs a GPU; writes only to a temporary
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


def _pin(x):
    import torch
    if torch.is_tensor(x):
        return x if x.stride() and 0 in x.stride() else x.pin_memory()
    if isinstance(x, list) and x and torch.is_tensor(x[0]):
        return [_pin(t) for t in x]
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=2)
    ap.add_argument("--modes", default="2,0")
    a = ap.parse_args()
    import torch
    from objgan_b200 import evaluator, losses, model, ops, synth, trainer
    from objgan_b200.config import cfg
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate.py needs a CUDA device")
    torch.cuda.set_device(0)
    b = a.batch
    gpu, power = _card()
    with tempfile.TemporaryDirectory() as tmp:
        torch.manual_seed(0)
        fast, model.FAST_INIT = model.FAST_INIT, True
        try:
            net_e = synth.reference_encoders(tmp, n_words=NTOKEN)
            torch.save(model.G_NET(80).state_dict(), os.path.join(tmp, "netG.pth"))
            torch.save(model.SHP_G_NET(80).state_dict(), os.path.join(tmp, "shape_gen.pth"))
            inception = model._Inception3().state_dict()
        finally:
            model.FAST_INIT = fast
        cfg.TRAIN.update(NET_E=net_e, NET_G=os.path.join(tmp, "netG.pth"), BATCH_SIZE=b, DISPLAY_INTERVAL=10 ** 9)
        cfg.TEST.update(NET_SHP_G=os.path.join(tmp, "shape_gen.pth"), USE_TF=0, SAVE_OPTIONS="IMAGE")
        for mode in [int(m) for m in a.modes.split(",")]:
            cfg.TEST.USE_GT_BOX_SEG = mode
            loader = [tuple(_pin(x) for x in synth.reference_test_batch(
                b, seed=2000 + i, mode=mode, full_maps=False, max_rois=cfg.ROI.BOXES_NUM, n_words=NTOKEN,
                n_glove=NTOKEN, fid_dims=cfg.TEST.FID_DIMS)) for i in range(a.distinct)]
            ds = synth.reference_test_dataset(n_words=NTOKEN, n_glove=NTOKEN)
            e = evaluator.condGANEvaluator(os.path.join(tmp, f"out{mode}"), loader, ds, inception_weights=inception,
                                           device="cuda:0")
            s = e.build_models()
            # the bare loop's inputs: the intake and the copies, done once per distinct batch
            staged = []
            for data in loader:
                batch, acts, class_ids, _, _ = trainer.prepare_reference_test_batch(data, mode)
                dev = {k: ([t.to("cuda") for t in v] if isinstance(v, list) else
                           v.to("cuda") if torch.is_tensor(v) else v) for k, v in batch.items()}
                staged.append((dev, acts.to("cuda"), class_ids))
            torch.cuda.synchronize()
            state = {}

            def fresh():
                state.update(rp=losses.RPrecision(cfg.TEST.RP_POOL_SIZE), is_=losses.InceptionScore(min(10, b)),
                             fid=losses.FrechetDistance(cfg.TEST.FID_DIMS))

            def loop(k):
                e.evaluate_batch(loader[k % len(loader)], state["rp"], state["is_"], state["fid"], gen_iterations=1)

            def bare(k):
                dev, acts, cids = staged[k % len(staged)]
                text = {}
                fake = s.sample_eager(dev, text_out=text)[0]
                region, code = s.encode_image(fake)
                state["rp"].add(region, code, text["words_embs"], text["sent_emb"], dev["cap_lens"], cids)
                pred, fake_acts = s.score_images(fake)
                state["is_"].add(pred)
                state["fid"].add(fake_acts, acts)

            def rate(fn):
                fresh()
                for k in range(a.warmup):
                    fn(k)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for k in range(a.steps):
                    fn(k)
                torch.cuda.synchronize()
                return a.steps * b / (time.perf_counter() - t0)

            rates = {"evaluator": [], "bare": []}
            for _ in range(a.rounds):
                rates["evaluator"].append(rate(loop))
                rates["bare"].append(rate(bare))
            for data in loader:
                trainer.prepare_reference_test_batch(data, mode)
            reps = 5 * len(loader)
            t0 = time.perf_counter()
            for k in range(reps):
                trainer.prepare_reference_test_batch(loader[k % len(loader)], mode)
            intake_ms = (time.perf_counter() - t0) * 1e3 / reps
            med = {k: statistics.median(v) for k, v in rates.items()}
            ms = b / med["evaluator"] * 1e3
            print(json.dumps({
                "bench": "evaluate", "gpu": gpu, "power_limit": power, "conv_engine": ops.CONV_ENGINE,
                "use_gt_box_seg": mode, "batch": b, "rois": cfg.ROI.BOXES_NUM, "fid_dims": cfg.TEST.FID_DIMS,
                "steps": a.steps, "warmup": a.warmup, "evaluator_img_s": round(med["evaluator"], 3),
                "bare_img_s": round(med["bare"], 3), "evaluator_vs_bare": round(med["evaluator"] / med["bare"], 4),
                "evaluator_ms_per_batch": round(ms, 2),
                "evaluator_rounds": [round(v, 3) for v in rates["evaluator"]],
                "bare_rounds": [round(v, 3) for v in rates["bare"]],
                "intake_host_ms_per_batch": round(intake_ms, 3), "intake_share_of_batch": round(intake_ms / ms, 4)}))
            del e, s, staged, loader
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
