"""Writing the box layout files of a test split (boxgen.Evaluator, output_opt 0) on a synthetic COCO-val2014-sized
split: 40,504 keys x 5 captions of 1 to 40 tokens, 84 decoder labels, early_stop_len 10, a seeded random decoder whose
<eos> bias is chosen from a grid so that samples average close to 4.5 rows (reported as mean_rows).  Prints one JSON line.

    python bench_box_files.py [--keys 40504] [--chunks 64,256,1024,4096] [--oracle 1000]

Reported:
  * the device stage alone (og_box_noise, the encoder state, og_box_decode, og_box_records; device-resident captions),
    captions/s at each chunk size, from CUDA events around a pass over the split;
  * end to end (reading the split's files, every chunk, the last boxes.txt closed) into a temporary directory, in
    captions/s, with the host intake (read and index the split) and the writer's busy time given separately;
  * the reference algorithm's cost: the CPU oracle composition (encoder state, the decoder step by step, the rows and
    the boxes.txt text) at batch 1 over --oracle captions, per caption, with the core count;
  * the card name and power limit.
Needs a GPU; writes only under a temporary directory it removes."""
import argparse
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_sample import _card  # noqa: E402

NTOKEN = 5000
CAT_IDS = [*range(1, 12), *range(13, 26), 27, 28, *range(31, 45), *range(46, 66), 67, 70, *range(72, 83),
           *range(84, 91)]
SPECIAL = ["<pad>", "<sos>", "<eos>", "<unk>"]
MEAN_STD = [[120.0, 60.0], [110.0, 55.0], [70.0, 40.0], [1.0, 0.5]]


def _modules(bias):
    import torch
    from objgan_b200 import model
    g = torch.Generator().manual_seed(0)
    l2i = {**{w: i for i, w in enumerate(SPECIAL)}, **{str(c): 4 + i for i, c in enumerate(CAT_IDS)}}
    enc = model.PreEncoderRNN(NTOKEN, nhidden=256)
    dec = model.DecoderRNN(l2i, 0.5, 0.4, 0.3, 1.1, 1, 150, 256, 5, dropout_p=0.2, bidirectional=True)
    with torch.no_grad():
        for p in list(enc.parameters()) + list(dec.parameters()):
            p.copy_(torch.rand(p.shape, generator=g) * 0.16 - 0.08)          # sample.py:141
        dec.l_out.bias[l2i["<eos>"]] += bias
    return enc, dec, l2i


def _split(n_keys, tmp):
    """The synthetic split's files (the reference's dev file and key file) and their vocabulary."""
    import numpy as np
    rng = np.random.default_rng(1)
    words = [f"w{i}" for i in range(1, NTOKEN)]
    dev, keys = os.path.join(tmp, "dev.txt"), os.path.join(tmp, "keys.txt")
    with open(dev, "w") as fd, open(keys, "w") as fk:
        for k in range(n_keys):
            for _ in range(5):
                n = int(rng.integers(1, 41))
                cap = " ".join(words[j] for j in rng.integers(0, len(words), n))
                fd.write(f"{cap}\t1 2\t3 4\t5 6\t1 1\t1 3\n")
                fk.write(f"COCO_val2014_{k:012d}\n")
    return dev, keys, {w: i + 1 for i, w in enumerate(words)}


def _evaluator(root, l2i, w2i, chunk):
    import types
    from objgan_b200 import boxgen
    gd = {c: (2.0 + i / 37.0, 0.3 + i / 101.0) for i, c in enumerate(CAT_IDS)}
    return boxgen.Evaluator(1, 10, root, types.SimpleNamespace(word2index=w2i, index2word={i: w for w, i in w2i.items()}),
                            types.SimpleNamespace(word2index=l2i, index2word={i: w for w, i in l2i.items()}),
                            *[tuple(r) for r in MEAN_STD], gd, root + "/gen_masks/", 0, chunk=chunk, seed=0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=40504)
    ap.add_argument("--chunks", default="64,256,1024,4096")
    ap.add_argument("--oracle", type=int, default=1000)
    a = ap.parse_args()
    import torch
    from objgan_b200 import boxgen, ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_files.py needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import box_files_oracle as F
    from oracle import box_oracle as O
    gpu, power = _card()
    out = {"bench": "box_files", "gpu": gpu, "power_limit": power, "keys": a.keys, "captions": 5 * a.keys}
    tmp = tempfile.mkdtemp(prefix="objgan_box_files_")
    try:
        dev_path, keys_path, w2i = _split(a.keys, tmp)
        t0 = time.perf_counter()
        data, keys = boxgen.read_test_tuples(dev_path), boxgen.read_keys(keys_path)
        seqs = boxgen.caption_sequences(data, keys, w2i)
        out["intake_s"] = time.perf_counter() - t0
        n = len(seqs)

        # the <eos> bias: the label is the argmax of nearly uniform logits, so a small bias moves the stop a lot; the
        # bias of this grid whose samples average closest to 4.5 rows
        best = None
        for b in [0.025 * k for k in range(13)]:
            enc, dec, l2i = _modules(b)
            ev = _evaluator(tmp, l2i, w2i, 4096)
            ev.generator = boxgen.BoxGenerator(enc.cuda(), dec.cuda(), ev.mean_std, ev.count_stats, ev.label_to_class)
            with torch.no_grad():
                packed = ev._device_records(0, seqs[:4096])
            r = float(ops.unpack_box_records(packed, 4096, 10)[2].double().mean())
            if best is None or abs(r - 4.5) < abs(best[1] - 4.5):
                best = (b, r, ev)
        bias, rows, ev = best
        out["eos_bias"], out["mean_rows"] = bias, rows

        # the device stage alone, captions on the device
        caps = torch.zeros(n, 40, dtype=torch.int64)
        lens = torch.tensor([len(q) for q in seqs])
        for i, q in enumerate(seqs):
            caps[i, :len(q)] = torch.tensor(q)
        caps, lens = caps.cuda(), lens.cuda()
        bg = ev.generator
        widths = {}

        def device_pass(chunk):
            for lo in range(0, n, chunk):
                hi = min(lo + chunk, n)
                if (lo, chunk) not in widths:
                    widths[(lo, chunk)] = int(max(len(q) for q in seqs[lo:hi]))
                w = widths[(lo, chunk)]
                nb, nc = ops.box_noise(0, lo, hi - lo, 10, bg.num_classes, "cuda")
                _, h, c = bg.encoder.encode_state(caps[lo:hi, :w].contiguous(), lens[lo:hi], w)
                lab, smp, st, _ = bg.decoder.sample_state(h, c, nb, 10)
                ops.box_records_packed(lab, smp, st, bg.mean_std, bg.label_to_class, bg.count_stats, nc)

        device = {}
        with torch.no_grad():
            for chunk in (int(c) for c in a.chunks.split(",")):
                device_pass(chunk)                                  # warm-up: every shape of the timed pass
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                device_pass(chunk)
                e.record()
                e.synchronize()
                device[str(chunk)] = round(n / (s.elapsed_time(e) / 1e3))
        out["device_captions_per_s"] = device

        # end to end: intake, every chunk, the last file closed
        for chunk in (1024,):
            root = os.path.join(tmp, f"run{chunk}")
            os.makedirs(root)
            enc, dec, _ = _modules(bias)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            data, keys = boxgen.read_test_tuples(dev_path), boxgen.read_keys(keys_path)
            ev = _evaluator(root, l2i, w2i, chunk)
            with contextlib.redirect_stdout(io.StringIO()):         # the reference's progress lines
                ev.evaluate(enc, dec, data, keys)
            dt = time.perf_counter() - t0
            files = sum(len(f) for _, _, f in os.walk(root))
            assert files == n, (files, n)
            out["end_to_end"] = {"chunk": chunk, "captions_per_s": round(n / dt), "seconds": round(dt, 2),
                                 "writer_busy_s": round(ev.write_seconds, 2)}
            shutil.rmtree(root)

        # the reference algorithm: the CPU oracle composition at batch 1
        enc, dec, _ = _modules(bias)
        esd = {k: v.detach() for k, v in enc.state_dict().items()}
        dsd = {k: v.detach() for k, v in dec.state_dict().items()}
        l2c = torch.tensor([-1] * 4 + list(range(80)))
        cs = torch.tensor(ev.count_stats, dtype=torch.float64)
        m = min(a.oracle, n)
        nb, nc = ops.box_noise(0, 0, m, 10, 80, "cuda")
        nb, nc = nb.cpu(), nc.cpu()
        t0 = time.perf_counter()
        with torch.no_grad():
            for i in range(m):
                q = torch.tensor([seqs[i]])
                h, c = O.encoder_state(esd, q, torch.tensor([len(seqs[i])]))
                r = O.decode(dsd, h[0], c[0], nb[i], 10, dec.l_sos_id, dec.l_eos_id, (0.5, 0.4, 0.3, 1.1))
                rows, cls, nv, _ = F.records(r["labels"], torch.stack(r["samples"]), MEAN_STD, l2c, cs, nc[i])
                F.files_text(rows, cls, [str(c) for c in CAT_IDS], keys[i], [], nv)
        per = (time.perf_counter() - t0) / m
        out["oracle_cpu"] = {"captions": m, "ms_per_caption": round(per * 1e3, 2), "cpu_count": os.cpu_count(),
                             "torch_threads": torch.get_num_threads(), "captions_per_s": round(1.0 / per, 1)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
