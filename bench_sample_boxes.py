"""Caption-to-image sampling throughput (GSampler with a box generator, a shape generator and a text encoder: captions
-> PreEncoderRNN + DecoderRNN + layout -> text encoder -> SHP_G_NET -> G_NET) at batch 1 and 16, with 84 decoder
labels, early_stop_len 10, untruncated box captions of 24 tokens and a 30,000-token vocabulary.  Prints one JSON line.

    python bench_sample_boxes.py [--batches 1,16] [--seconds 3] [--rounds 3]

Reported per batch:
  * images/s of the whole caption -> image sample, eager (every stage, the box stage included, launched without a
    graph) against CUDA-graph replay (the box graph, then the image graph), alternated in rounds (CUDA events
    around a window of back-to-back calls, device-resident seeded inputs and noise, so every call has the same layout);
  * the box stage alone (encoder state, og_box_decode, og_box_layout; eager) and og_box_decode alone, ms per batch
    from CUDA events;
  * the roi counts of the layout, and whether replayed and eager outputs are bitwise equal;
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
from bench_sample_text import _events_ms  # noqa: E402

NTOKEN = 30000
BOX_LEN = 24
CAT_IDS = [*range(1, 12), *range(13, 26), 27, 28, *range(31, 45), *range(46, 66), 67, 70, *range(72, 83),
           *range(84, 91)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from objgan_b200 import boxgen, lib, model, ops, synth
    from objgan_b200.config import cfg
    from objgan_b200.sampler import GSampler
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_boxes.py needs a CUDA device")
    torch.manual_seed(0)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    shp = model.SHP_G_NET(80)
    shp.apply(model.weights_init)
    enc = model.RNN_ENCODER(NTOKEN, nhidden=cfg.TEXT.EMBEDDING_DIM)
    pre = model.PreEncoderRNN(NTOKEN, nhidden=256)
    pre.load_state_dict(enc.state_dict())
    l2i = {**{w: i for i, w in enumerate(["<pad>", "<sos>", "<eos>", "<unk>"])},
           **{str(c): 4 + i for i, c in enumerate(CAT_IDS)}}
    dec = model.DecoderRNN(l2i, 0.5, 0.4, 0.3, 1.1, 1, 150, 256, 5, dropout_p=0.2, bidirectional=True)
    with torch.no_grad():
        for p in dec.parameters():
            p.uniform_(-0.08, 0.08)                  # sample.py:141
    box = boxgen.BoxGenerator(pre.cuda(), dec.cuda(), [[120.0, 60.0], [110.0, 55.0], [70.0, 40.0], [1.0, 0.5]],
                              [[3.0, 1.0]] * 80, [-1] * 4 + list(range(80)))
    glove = 0.5 * torch.randn(NTOKEN, cfg.TEXT.GLOVE_EMBEDDING_DIM)
    s = GSampler(g.cuda(), shp.cuda(), text_encoder=enc.cuda(), glove=glove, box_generator=box)
    res = {"bench": "gsampler_boxes", "gpu": None, "power_limit": None, "conv_engine": ops.CONV_ENGINE,
           "early_stop_len": box.early_stop_len, "box_caption_len": BOX_LEN, "vocabulary": NTOKEN, "batches": {}}
    res["gpu"], res["power_limit"] = _card()
    flat = lambda o: [*o[0], *o[1], *o[2], *o[3], o[4], o[5]]
    L = cfg.TEXT.WORDS_NUM
    for b in [int(x) for x in a.batches.split(",")]:
        gen = torch.Generator().manual_seed(b)
        x = {"captions": torch.randint(1, NTOKEN, (b, L), generator=gen),
             "glove_captions": torch.randint(1, NTOKEN, (b, L), generator=gen),
             "cap_lens": torch.full((b,), L, dtype=torch.int64),
             "box_captions": torch.randint(1, NTOKEN, (b, BOX_LEN), generator=gen),
             "box_cap_lens": torch.full((b,), BOX_LEN, dtype=torch.int64),
             "z": torch.randn(b, cfg.GAN.Z_DIM, generator=gen), "eps": torch.randn(b, cfg.GAN.CONDITION_DIM, generator=gen),
             "noise_shp": torch.randn(b, cfg.ROI.BOXES_NUM, 320, generator=gen),
             "noise_cnt": torch.randn(b, 80, generator=gen),
             "clabels_emb": synth.make_inputs(1, seed=b)["clabels_emb"]}
        nb = torch.randn(b, box.early_stop_len, 6, generator=gen)
        nb[:, :, 0::3] = torch.rand(b, box.early_stop_len, 2, generator=gen)
        x["noise_box"] = nb
        dev = {k: v.cuda() for k, v in x.items()}
        s.sample(dev)                          # eager warm-up + capture of both graphs
        s.sample(dev)
        n0 = lib.get().launches
        eager = s.sample_eager(dev)
        calls = lib.get().launches - n0
        replay = s.sample(dev)
        torch.cuda.synchronize()
        exact = all(torch.equal(p, q) for p, q in zip(flat(replay), flat(eager)))
        n_iter = 50 if b > 1 else 200
        with torch.no_grad():
            box_ms = _events_ms(lambda: box.sample(dev["box_captions"], dev["box_cap_lens"], BOX_LEN, dev["noise_box"],
                                                   dev["noise_cnt"]), n_iter)
            _, h, c = pre.encode_state(dev["box_captions"], dev["box_cap_lens"], BOX_LEN)
            dec_ms = _events_ms(lambda: dec.sample_state(h, c, dev["noise_box"], box.early_stop_len), n_iter)
            lay = s.sample_layout(dev)
        rates = {"eager": [], "graph": []}
        for _ in range(a.rounds):
            rates["eager"].append(_rate(lambda: s.sample_eager(dev), b, a.seconds))
            rates["graph"].append(_rate(lambda: s.sample(dev), b, a.seconds))
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["batches"][str(b)] = {
            "eager_img_s": round(med["eager"], 2), "graph_img_s": round(med["graph"], 2),
            "speedup": round(med["graph"] / med["eager"], 3),
            "eager_rounds": [round(v, 2) for v in rates["eager"]], "graph_rounds": [round(v, 2) for v in rates["graph"]],
            "box_stage_ms": round(box_ms, 4), "box_decode_ms": round(dec_ms, 4),
            "num_rois": lay["num_rois"].tolist(), "calls_per_sample": calls, "replay_bitwise_equal": exact}
        del dev, eager, replay
    print(json.dumps(res))


if __name__ == "__main__":
    main()
