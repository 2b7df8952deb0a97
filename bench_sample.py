"""Sampling throughput of the eval-mode generator (objgan_b200.sampler.GSampler): images/s at batch 1 and 16, eager
launches against CUDA-graph replay, alternated in the same run.  Prints one JSON line.

    python bench_sample.py [--batches 1,16] [--seconds 3] [--rounds 3]

Each (batch, mode) is timed with CUDA events around a window of back-to-back sample calls (device-resident seeded
inputs, z / eps included, outputs returned as fresh tensors in both modes) after warm-up; the rounds alternate eager and
replay so both see the same machine state, and every round's rate is reported (the spread).  Also reported: library
calls per forward, and the largest difference between the eager and the replayed outputs relative to max|eager|.
Needs a GPU; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 else ("unknown", "", "")
    return name.strip(), power.strip()


def _rate(fn, batch, seconds):
    """images/s of fn over a window of about `seconds`, from CUDA events around the whole window."""
    import torch
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    start.record()
    while True:
        fn()
        n += 1
        if n % 4 == 0:
            torch.cuda.synchronize()
            if time.perf_counter() - t0 >= seconds:
                break
    end.record()
    end.synchronize()
    return n * batch / (start.elapsed_time(end) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from objgan_b200 import lib, model, synth
    from objgan_b200.sampler import GSampler
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py needs a CUDA device")
    torch.manual_seed(0)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    s = GSampler(g.to("cuda"))
    res = {"bench": "gsampler", "gpu": None, "power_limit": None, "conv_engine": None, "batches": {}}
    res["gpu"], res["power_limit"] = _card()
    from objgan_b200 import ops
    res["conv_engine"] = ops.CONV_ENGINE
    for b in [int(x) for x in a.batches.split(",")]:
        x = synth.make_inputs(b, seed=100 + b)
        dev = {k: (v.cuda() if torch.is_tensor(v) else [t.cuda() for t in v] if isinstance(v, list) else v)
               for k, v in x.items()}
        s.sample(dev)                          # eager warm-up + capture
        s.sample(dev)
        n0 = lib.get().launches
        eager = s.sample_eager(dev)
        calls = lib.get().launches - n0
        replay = s.sample(dev)
        torch.cuda.synchronize()
        flat = lambda o: [*o[0], *o[1], *o[2], *o[3], o[4], o[5]]
        diff = max(((p - q).abs().max() / q.abs().max().clamp(min=1e-30)).item()
                   for p, q in zip(flat(replay), flat(eager)) if q.numel())
        exact = all(torch.equal(p, q) for p, q in zip(flat(replay), flat(eager)))
        rates = {"eager": [], "graph": []}
        for _ in range(a.rounds):
            rates["eager"].append(_rate(lambda: s.sample_eager(dev), b, a.seconds))
            rates["graph"].append(_rate(lambda: s.sample(dev), b, a.seconds))
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["batches"][str(b)] = {
            "eager_img_s": round(med["eager"], 2), "graph_img_s": round(med["graph"], 2),
            "speedup": round(med["graph"] / med["eager"], 3),
            "eager_rounds": [round(r, 2) for r in rates["eager"]], "graph_rounds": [round(r, 2) for r in rates["graph"]],
            "calls_per_forward": calls, "max_rel_diff_replay_vs_eager": diff, "replay_bitwise_equal": exact}
        del dev, eager, replay
    print(json.dumps(res))


if __name__ == "__main__":
    main()
