"""Times the DAMSM image encoder (CNN_ENCODER, Inception-v3 trunk) on one GPU: forward at B = 1 and 16 and forward +
input gradient at B = 16, in ms and algorithmic TFLOP/s (2 x the multiply-adds counted from the layer table below).
For information, the same computation through cuDNN (the oracle's torch.nn.functional restatement on the GPU, with
TF32 allowed and disallowed) is timed too, and each result's distance from the float64 oracle is printed.  Then
StepBTrainer.step at batch 16, with and without the DAMSM terms, in images/s.  Prints the card name and power limit
first and one JSON line last.

    python bench_image_encoder.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0)
    return out


def encoder_macs(net, size=256):
    """Multiply-adds of one image: every convolution from the program's layer table (299 x 299 trunk input)."""
    prog = net.program()
    hw = {"x299": (299, 299)}
    total = 0
    for st in prog.steps:
        if st[0] == "conv":
            _, layer, s, d, _ = st
            h, w = hw[s]
            total += layer.macs(h, w)
            hw[d] = layer.out_hw(h, w)
        elif st[0] in ("copy",):
            hw[st[3]] = hw[st[1]]
        elif st[0] == "maxpool":
            h, w = hw[st[1]]
            hw[st[2]] = ((h - 3) // 2 + 1, (w - 3) // 2 + 1)
        elif st[0] == "avgpool":
            hw[st[2]] = hw[st[1]]
    return total + 2048 * net.nef


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def step_b_images_per_s(image_encoder, steps=6):
    """StepBTrainer.step at batch 16 on bench.py's Step-B inputs (synth.make_inputs -> compact -> pinned -> device),
    with the DAMSM terms when ``image_encoder`` is given; images/s from CUDA events over ``steps`` eager steps."""
    import random
    from objgan_b200 import synth, trainer
    random.seed(1234)
    tr = trainer.StepBTrainer(device="cuda", seed=1234, image_encoder=image_encoder)
    full = synth.make_inputs(16, seed=1234, parity=False)
    full.pop("eps")
    dev = tr.to_device(trainer.pin(synth.compact(full)))
    ms = timed(lambda: tr.step(dev), steps)
    return 16 / (ms * 1e-3), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_image_encoder.py needs a GPU"
    from objgan_b200 import model
    from oracle import image_encoder_oracle as E
    print("card:", card())
    net = model.CNN_ENCODER(256)
    net.load_state_dict(E.test_state_dict(net.state_dict(), seed=0))
    net = net.to("cuda")
    sd = {k: v.cuda() for k, v in net.state_dict().items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    macs = encoder_macs(net)
    print(f"forward: {macs / 1e9:.2f} G multiply-adds per image")
    res = {"macs_per_image": macs}
    g = torch.Generator().manual_seed(0)
    for b in (1, 16):
        x = (torch.rand(b, 3, 256, 256, generator=g) * 2 - 1).cuda()
        with torch.no_grad():
            ms = timed(lambda: net(x), args.iters)
        res[f"fwd_B{b}_ms"] = ms
        res[f"fwd_B{b}_tflops"] = 2 * macs * b / ms / 1e9
        print(f"ours fwd B={b}: {ms:.3f} ms, {2 * macs * b / ms / 1e9:.1f} TFLOP/s")
    b = 16
    x = (torch.rand(b, 3, 256, 256, generator=g) * 2 - 1).cuda()
    a, c = torch.randn(b, 256, 17, 17, generator=g).cuda(), torch.randn(b, 256, generator=g).cuda()

    def ours_fb():
        xg = x.clone().requires_grad_(True)
        f, code = net(xg)
        ((f * a).sum() + (code * c).sum()).backward()
        return f, code, xg.grad

    ms = timed(ours_fb, args.iters)
    res["fwd_bwd_B16_ms"] = ms
    print(f"ours fwd+dgrad B=16: {ms:.3f} ms, {4 * macs * b / ms / 1e9:.1f} TFLOP/s (2 x forward MACs counted)")

    def cudnn_fb(dtype=torch.float32, s=sd):
        xg = x.to(dtype).clone().requires_grad_(True)
        f, code = E.cnn_encoder_forward(s, xg)
        ((f * a.to(dtype)).sum() + (code * c.to(dtype)).sum()).backward()
        return f, code, xg.grad

    rf, rc, rg = cudnn_fb(torch.float64, sd64)
    dev = lambda t, r: ((t.double() - r).norm() / r.norm()).item()
    of, oc, og = ours_fb()
    res["ours_dev"] = [dev(of, rf), dev(oc, rc), dev(og, rg)]
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        ms = timed(cudnn_fb, args.iters)
        with torch.no_grad():
            msf = timed(lambda: E.cnn_encoder_forward(sd, x), args.iters)
        f, code, gx = cudnn_fb()
        key = "cudnn_tf32" if tf32 else "cudnn_fp32"
        res[key] = {"fwd_B16_ms": msf, "fwd_bwd_B16_ms": ms, "dev": [dev(f, rf), dev(code, rc), dev(gx, rg)]}
        print(f"{key}: fwd B=16 {msf:.3f} ms, fwd+dgrad B=16 {ms:.3f} ms, rel-L2 vs float64 (features, code, dgrad) "
              + ", ".join(f"{v:.2e}" for v in res[key]["dev"]))
    print("ours rel-L2 vs float64 (features, code, dgrad): " + ", ".join(f"{v:.2e}" for v in res["ours_dev"]))
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    for rnd in range(2):                  # alternated, so that both see the same clock and neighbours
        for name, e in (("step_b_no_damsm", None), ("step_b_damsm", net)):
            ips, ms = step_b_images_per_s(e)
            res.setdefault(name, []).append(round(ips, 2))
            print(f"{name} round {rnd}: {ips:.1f} images/s ({ms:.1f} ms/step, batch 16)")
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
