"""Times the scoring networks on one GPU: INCEPTION_V3 (probabilities) and INCEPTION_V3_FID (2048-d activations)
forward at B = 1, 16 and 32, against the same computation through cuDNN (tests/inception_oracle.py's
torch.nn.functional restatement on the GPU) with TF32 allowed and disallowed, each with its distance from the float64
oracle at B = 16.  Then the evaluator's loop at batch 16 in images/s: GSampler.sample, encode_image + RPrecision,
score_images + InceptionScore + FrechetDistance.  Prints the card name and power limit first and one JSON line last.

    python bench_inception.py [--iters 20]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from bench_image_encoder import card, timed  # noqa: E402


def evaluator_images_per_s(inc, fid, steps=8):
    """One evaluator iteration per batch of 16 (ref: evaluator.py:268-436): sample, the image encoder and the
    R-precision pool, both scoring networks and both accumulators; the real activations are precomputed, as the
    reference's dump_fid_acts does."""
    from objgan_b200 import losses, model, synth
    from objgan_b200.sampler import GSampler, _new_g
    from oracle import image_encoder_oracle as E
    enc = model.CNN_ENCODER(256)
    enc.load_state_dict(E.test_state_dict(enc.state_dict(), seed=0))
    s = GSampler(_new_g(80, "cuda"), image_encoder=enc, inception=inc, inception_fid=fid)
    batch = synth.make_inputs(16, seed=77, parity=True)
    words, sent = batch["words_embs"].cuda(), batch["sent_emb"].cuda()
    g = torch.Generator().manual_seed(5)
    real = fid.activations((torch.rand(16, 3, 256, 256, generator=g) * 2 - 1).cuda())
    rp, sc, fd = losses.RPrecision(100), losses.InceptionScore(10), losses.FrechetDistance(2048)

    def one():
        fake_imgs = s.sample(batch)[0]
        region, code = s.encode_image(fake_imgs)
        rp.add(region, code, words, sent, batch["cap_lens"])
        pred, acts = s.score_images(fake_imgs)
        sc.add(pred)
        fd.add(acts, real)

    ms = timed(one, steps)
    return 16 / (ms * 1e-3), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_inception.py needs a GPU"
    import inception_oracle as I
    from objgan_b200 import model
    print("card:", card())
    sd = I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0)
    inc = model.INCEPTION_V3()
    inc.load_state_dict({"model." + k: v for k, v in sd.items()})
    fid = model.INCEPTION_V3_FID([3])
    fid.load_state_dict(fid.from_torchvision(sd))
    inc, fid = inc.cuda(), fid.cuda()
    sd = {k: v.cuda() for k, v in sd.items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    nets = {"is": (inc, lambda s, x: I.inception_v3_forward(s, x)),
            "fid": (fid.activations, lambda s, x: I.fid_activations(s, x, 2048))}
    res = {}
    g = torch.Generator().manual_seed(0)
    xs = {b: (torch.rand(b, 3, 256, 256, generator=g) * 2 - 1).cuda() for b in (1, 16, 32)}
    dev = lambda t, r: ((t.double() - r).norm() / r.norm()).item()
    for name, (ours, ref) in nets.items():
        with torch.no_grad():
            r64 = ref(sd64, xs[16].double())
        for b, x in xs.items():
            res[f"{name}_B{b}_ms"] = timed(lambda: ours(x), args.iters)
        res[f"{name}_dev"] = dev(ours(xs[16]), r64)
        print(f"ours {name}: " + ", ".join(f"B={b} {res[f'{name}_B{b}_ms']:.3f} ms" for b in xs)
              + f"; rel-L2 vs float64 at B=16 {res[f'{name}_dev']:.2e}")
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            key = f"{name}_cudnn_{'tf32' if tf32 else 'fp32'}"
            with torch.no_grad():
                res[key] = {f"B{b}_ms": timed(lambda: ref(sd, x), args.iters) for b, x in xs.items()}
                res[key]["dev"] = dev(ref(sd, xs[16]), r64)
            print(f"{key}: " + ", ".join(f"B={b} {res[key][f'B{b}_ms']:.3f} ms" for b in xs)
                  + f"; rel-L2 vs float64 at B=16 {res[key]['dev']:.2e}")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    ips, ms = evaluator_images_per_s(inc, fid)
    res["evaluator_images_per_s"], res["evaluator_ms_per_batch16"] = ips, ms
    print(f"evaluator loop: {ips:.1f} images/s ({ms:.1f} ms per batch of 16)")
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
