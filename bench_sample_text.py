"""Caption-conditioned sampling throughput (GSampler with a text encoder: token ids -> RNN_ENCODER + GloVe lookups ->
G_NET, ground-truth masks) at batch 1 and 16 with WORDS_NUM = 18, 10 rois per image and a 30,000-token vocabulary.
Prints one JSON line.

    python bench_sample_text.py [--batches 1,16] [--seconds 3] [--rounds 3]

Reported per batch:
  * images/s of the whole caption-conditioned sample, eager against CUDA-graph replay, alternated in rounds (as
    bench_sample.py does; CUDA events around a window of back-to-back calls, device-resident seeded inputs);
  * the text stage alone (token lookup, input projection, og_lstm_bidir, GloVe lookups + mask; eager), ms per batch
    from CUDA events, and og_lstm_bidir alone;
  * for information only: the same encoding through torch's nn.LSTM + pack_padded_sequence (the reference's
    RNN_ENCODER.forward, cuDNN on this card), ms per batch from CUDA events, and the largest difference from ours;
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

NTOKEN = 30000
NGLOVE = 30000


def _events_ms(fn, n_iter):
    import torch
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(n_iter):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / n_iter


def _torch_lstm(enc):
    """nn.LSTM with the encoder's weights, the reference's RNN_ENCODER.forward recipe (model.py:145-179)."""
    import torch
    lstm = torch.nn.LSTM(enc.ninput, enc.nhidden, 1, batch_first=True, bidirectional=True).cuda().eval()
    lstm.load_state_dict({k: v for k, v in enc.rnn.state_dict().items()})

    def run(captions, cap_lens, max_len):
        from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
        emb = torch.nn.functional.embedding(captions, enc.encoder.weight)
        packed = pack_padded_sequence(emb, cap_lens.tolist(), batch_first=True)       # host read of the lengths
        out, (h, _) = lstm(packed)
        out = pad_packed_sequence(out, batch_first=True)[0].transpose(1, 2)
        words = torch.zeros(captions.shape[0], 2 * enc.nhidden, max_len, device=captions.device)
        words[:, :, :out.shape[2]] = out
        return words, h.transpose(0, 1).reshape(-1, 2 * enc.nhidden)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from objgan_b200 import lib, model, ops, synth
    from objgan_b200.config import cfg
    from objgan_b200.sampler import GSampler
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_text.py needs a CUDA device")
    torch.manual_seed(0)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    enc = model.RNN_ENCODER(NTOKEN, nhidden=cfg.TEXT.EMBEDDING_DIM)
    glove = 0.5 * torch.randn(NGLOVE, cfg.TEXT.GLOVE_EMBEDDING_DIM)
    s = GSampler(g.to("cuda"), text_encoder=enc.to("cuda"), glove=glove)
    ref_lstm = _torch_lstm(s.text_encoder)
    res = {"bench": "gsampler_text", "gpu": None, "power_limit": None, "conv_engine": ops.CONV_ENGINE, "rois": 10,
           "words_num": cfg.TEXT.WORDS_NUM, "vocabulary": NTOKEN, "batches": {}}
    res["gpu"], res["power_limit"] = _card()
    flat = lambda o: [*o[0], *o[1], *o[2], *o[3], o[4], o[5]]
    L = cfg.TEXT.WORDS_NUM
    for b in [int(x) for x in a.batches.split(",")]:
        gen = torch.Generator().manual_seed(b)
        x = synth.compact(synth.make_inputs(b, seed=100 + b))
        for k in ("words_embs", "sent_emb", "glove_words_embs", "mask"):
            x.pop(k)
        lens = torch.randint(1, L + 1, (b,), generator=gen)
        lens[0] = L
        lens = torch.sort(lens, descending=True).values       # sorted, so that pack_padded_sequence accepts it
        keep = torch.arange(L).view(1, L) < lens.view(b, 1)
        x["captions"] = torch.randint(1, NTOKEN, (b, L), generator=gen) * keep
        x["glove_captions"] = torch.randint(1, NGLOVE, (b, L), generator=gen) * keep
        x["cap_lens"] = lens
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
        n_iter = 50 if b > 1 else 200
        with torch.no_grad():
            prep = s._prepare(dev)
            text_ms = _events_ms(lambda: s._text(prep), n_iter)
            emb, wih, bias = s.text_encoder.derived_weights()
            xg = ops.gather_rows(emb, prep["captions"][:, :L].reshape(-1))
            gx = ops.linear_rows(xg, wih, bias, s.text_encoder._cache)
            r = s.text_encoder.rnn
            lstm_ms = _events_ms(lambda: ops.lstm_bidir(gx, r.weight_hh_l0, r.weight_hh_l0_reverse, prep["cap_lens"], L),
                                 n_iter)
            ours = s.text_encoder(prep["captions"], prep["cap_lens"], L)
            theirs = ref_lstm(prep["captions"], prep["cap_lens"], L)
            torch_diff = max(((p - q).abs().max() / q.abs().max()).item() for p, q in zip(ours, theirs))
            torch_ms = _events_ms(lambda: ref_lstm(prep["captions"], prep["cap_lens"], L), n_iter)
        rates = {"eager": [], "graph": []}
        for _ in range(a.rounds):
            rates["eager"].append(_rate(lambda: s.sample_eager(dev), b, a.seconds))
            rates["graph"].append(_rate(lambda: s.sample(dev), b, a.seconds))
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["batches"][str(b)] = {
            "eager_img_s": round(med["eager"], 2), "graph_img_s": round(med["graph"], 2),
            "speedup": round(med["graph"] / med["eager"], 3),
            "eager_rounds": [round(v, 2) for v in rates["eager"]], "graph_rounds": [round(v, 2) for v in rates["graph"]],
            "text_stage_ms": round(text_ms, 4), "lstm_bidir_ms": round(lstm_ms, 4),
            "torch_lstm_packed_ms_info": round(torch_ms, 4), "max_rel_diff_vs_torch_lstm": torch_diff,
            "cap_lens": lens.tolist(), "calls_per_sample": calls, "max_rel_diff_replay_vs_eager": diff,
            "replay_bitwise_equal": exact}
        del dev, eager, replay, prep
    print(json.dumps(res))


if __name__ == "__main__":
    main()
