"""The snapshot canvases (og_snapshot_canvas) against the host oracle (oracle/snapshot_oracle.py) at every shape the
networks issue: G maps 64 -> 128 and 128 -> 256, DAMSM 17 -> 272 with ragged caption lengths, and shape maps at 64
(no expansion), at B = 1, 3, 8, 16, plus map counts below, at and above WORDS_NUM and constant maps.  Shape canvases
and unresized image tiles are bitwise; expanded maps and resized image tiles are within one byte, with at most 1e-3
of the bytes differing.  Then a condGANTrainer display step: its PNGs against the oracle composed from the images and
maps it used; every network's weights, Adam moments and EMA unchanged; the generator's BatchNorm buffers equal to
those of a train-mode forward with the EMA weights; the next step's images bitwise equal to the same step's without
the display, and the generator's state after it within the spread of two identical steps.  Last, the kernels against canvases made by the reference's own functions
(tests/golden/reference/snapshot_*.npz)."""
import os
import random

import numpy as np
import pytest
import torch
from PIL import Image, ImageFont

from objgan_b200 import ops, snapshots, synth, trainer
from objgan_b200.config import cfg
from oracle import snapshot_oracle as O
import snapshot_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORDS = 18


def _maps(b, L, att, seed, const=None):
    g = torch.Generator().manual_seed(seed)
    m = torch.softmax(torch.randn(b, L, att, att, generator=g) * 3, 1)
    if const is not None:
        m.fill_(const)
    return m


def _imgs(b, s, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 3, s, s, generator=g) * 2 - 1


def _near(got, want, what):
    d = np.abs(got.astype(np.int16) - want.astype(np.int16))
    frac = float((d > 0).mean())
    print(f"{what}: max |diff| {d.max()}, fraction of bytes differing {frac:.2e}")
    assert d.max() <= 1 and frac <= 1e-3, (what, d.max(), frac)


CASES = [  # (B, image side, lr side, map side, L, ragged lengths, constant)
    *[(b, 128, 64, 64, 6, False, None) for b in (1, 3, 8, 16)],
    *[(b, 256, 128, 128, 6, False, None) for b in (1, 3, 8, 16)],
    *[(b, 256, None, 17, 12, True, None) for b in (1, 3, 8, 16)],
    (8, 128, 64, 64, WORDS, False, None),
    (8, 128, 64, 64, WORDS + 3, False, None),
    (3, 256, None, 17, WORDS + 2, True, None),
    (8, 128, 64, 64, 4, False, 0.5),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_%d_att%d_L%d%s%s" % (
    c[0], c[1], c[3], c[4], "_ragged" if c[5] else "", "_const" if c[6] is not None else ""))
def test_super_images_vs_oracle(case, monkeypatch):
    monkeypatch.setitem(cfg.TEXT, "WORDS_NUM", WORDS)
    b, s, ls, att, L, ragged, const = case
    imgs, maps = _imgs(b, s, 1), _maps(b, L, att, 2, const)
    lr = _imgs(b, ls, 3) if ls else None
    lens = torch.randint(1, L + 1, (b,), generator=torch.Generator().manual_seed(4)) if ragged else None
    per_image = [maps[i, :int(lens[i])] for i in range(b)] if ragged else maps
    want = O.super_images(imgs, None, None, per_image, att, lr_imgs=lr, words=WORDS, batch_rows=min(8, b))
    c = snapshots.super_images(imgs.to(DEV), None, None, maps.to(DEV), lr_images=None if lr is None else lr.to(DEV),
                               lens=None if lens is None else lens.to(DEV))
    got = c.pixels()
    assert got.shape == want.shape
    _near(got, want, "B%d %d<-%d" % (b, s, att))
    if s == (att * 16 if att == 17 else s) and att != 17:          # unresized image tiles of the merged row
        vis, per = s, 50 + 2 * s
        for i in range(min(8, b)):
            r0 = i * per + 50 + vis
            assert np.array_equal(got[r0:r0 + vis, :vis], want[r0:r0 + vis, :vis])
    again = snapshots.super_images(imgs.to(DEV), None, None, maps.to(DEV),
                                   lr_images=None if lr is None else lr.to(DEV),
                                   lens=None if lens is None else lens.to(DEV)).pixels()
    assert np.array_equal(got, again)


@pytest.mark.parametrize("b,r", [(1, 3), (3, 10), (8, 7), (16, 80), (16, 10)])
def test_super_shape_images_bitwise(b, r):
    imgs = _imgs(b, 64, 5)
    maps = torch.rand(b, r, 64, 64, generator=torch.Generator().manual_seed(6))
    maps[:, 0] = 0                                   # an empty class channel: max == min
    want = O.super_shape_images(imgs, maps, cfg.ROI.BOXES_NUM)
    got = snapshots.super_shape_images(imgs.to(DEV), maps.to(DEV)).pixels()
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------- the training loop
N_WORDS = 150


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """NET_E (text and image encoder) and Inception weights, as the training-loop tests make them."""
    import inception_oracle as I
    from objgan_b200 import model
    from oracle import image_encoder_oracle as E
    d = tmp_path_factory.mktemp("pretrained")
    torch.manual_seed(0)
    text_sd = model.RNN_ENCODER(N_WORDS, nhidden=256).state_dict()
    torch.save(text_sd, d / "text_encoder100.pth")
    torch.save(E.test_state_dict(model.CNN_ENCODER(256).state_dict(), seed=0), d / "image_encoder100.pth")
    return (str(d / "text_encoder100.pth"), I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0),
            text_sd)


def _bn_buffers(net):
    return [t.clone() for t in net.buffers()]


def test_trainer_display_step(files, tmp_path, monkeypatch):
    for k, v in dict(MAX_EPOCH=1, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=100, BATCH_SIZE=3, FLAG=True, NET_E=files[0],
                     NET_G="", DISPLAY_INTERVAL=1).items():
        monkeypatch.setitem(cfg.TRAIN, k, v)
    monkeypatch.setitem(cfg.TEXT, "WORDS_NUM", WORDS)
    ds = synth.reference_dataset(n_words=N_WORDS)
    ds.ixtoword = {i: "w%dgjy" % i for i in range(N_WORDS)}
    font = ImageFont.load_default(size=50)
    t = trainer.condGANTrainer(str(tmp_path), [], ds, inception_weights=files[1], device=DEV, font=font)
    torch.manual_seed(3)
    t.setup()
    data = [synth.reference_batch(3, seed=70 + i, n_words=N_WORDS) for i in range(2)]
    g = torch.Generator(device=DEV).manual_seed(9)
    z = [torch.randn(3, cfg.GAN.Z_DIM, device=DEV, generator=g) for _ in range(2)]
    eps = [torch.randn(3, cfg.GAN.CONDITION_DIM, device=DEV, generator=g) for _ in range(2)]
    t.train_step(data[0], z=z[0], eps=eps[0])
    net = t.net
    # EMA weights far from the live ones: a display that left the EMA weights (or their fp16 operand copies) in the
    # generator would change the next step's images well beyond its rounding
    net.bG.avg.add_(torch.randn(net.bG.avg.shape, device=DEV, generator=g) * 0.05)
    buckets = [net.bG, *net._d_buckets()]
    nets = [net.netG, *net.netsPatD, *net.netsShpD, net.netObjSSD, net.netObjLSD]
    state = [(bk.flat.clone(), bk.m.clone(), bk.v.clone(), None if bk.avg is None else bk.avg.clone(), bk.step,
              bk.step_dev.clone()) for bk in buckets]
    bufs = [_bn_buffers(n) for n in nets]
    # the host shuffles of the step draw from these generators; the display draws from none of them except the CUDA
    # one (CA_NET's noise): both runs of the next step start from the states a run without the display would have
    rng = (random.getstate(), np.random.get_state(), torch.get_rng_state(), torch.cuda.get_rng_state())

    def restore_rng():
        random.setstate(rng[0]); np.random.set_state(rng[1]); torch.set_rng_state(rng[2])
        torch.cuda.set_rng_state(rng[3])

    used = []
    real = snapshots.super_images

    def spy(images, captions, ixtoword, maps, **kw):
        used.append((images.detach().cpu(), captions, maps.detach().cpu(),
                     None if kw.get("lr_images") is None else kw["lr_images"].detach().cpu(),
                     None if kw.get("lens") is None else kw["lens"].cpu()))
        return real(images, captions, ixtoword, maps, **kw)

    monkeypatch.setattr(snapshots, "super_images", spy)
    w = snapshots.PngWriter()
    t.save_img_results(0, w)
    w.close()
    names = sorted(os.listdir(tmp_path / "Image"))
    assert names == sorted(["G_average_0_0.png", "G_average_0_1.png", "bt_G_average_0_0.png",
                            "bt_G_average_0_1.png", "D_average_0.png"])
    # the display leaves every network's weights, Adam moments and EMA as they were
    for bk, (flat, m, v, avg, step, _) in zip(buckets, state):
        assert torch.equal(bk.flat, flat) and torch.equal(bk.m, m) and torch.equal(bk.v, v) and bk.step == step
        assert avg is None or torch.equal(bk.avg, avg)
    # its train-mode forward updated the generator's BatchNorm buffers exactly as a train-mode forward with the EMA
    # weights does: the same forward run again from the buffers before the display, the EMA weights and the same
    # random state (CA_NET's noise) gives the same buffers, bit for bit.  (The forward itself is checked against the
    # oracle in test_gpu_zz_train_loop.py.)
    post = _bn_buffers(net.netG)
    changed = sum(not torch.equal(x, y) for x, y in zip(post, bufs[0]))
    assert changed > 0
    for x, s0 in zip(net.netG.buffers(), bufs[0]):
        x.copy_(s0)
    t._load_g(net.bG.avg)
    torch.cuda.set_rng_state(rng[3])
    dev, _ = t._display
    with torch.no_grad():
        net.generate(dict({k: v for k, v in dev.items() if k != "eps"}, z=t.fixed_noise[:3]))
    for x, y in zip(net.netG.buffers(), post):
        assert torch.equal(x, y)
    t._load_g(state[0][0])
    order = ["G_average_0_0.png", "bt_G_average_0_0.png", "G_average_0_1.png", "bt_G_average_0_1.png",
             "D_average_0.png"]
    for name, (images, captions, maps, lr, lens) in zip(order, used):
        png = np.asarray(Image.open(tmp_path / "Image" / name))
        att = maps.shape[-1]
        per_image = [maps[i, :int(lens[i])] for i in range(maps.shape[0])] if lens is not None else maps
        want = O.super_images(images, captions, ds.ixtoword, per_image, att, lr_imgs=lr, words=WORDS, font=font)
        _near(png, want, name)

    restore_rng()
    out_a = t.train_step(data[1], z=z[1], eps=eps[1])
    g = net.bG
    a = [g.flat.clone(), g.m.clone(), g.v.clone(), g.avg.clone()]
    def without_display():
        for bk, (flat, m, v, avg, step, step_dev) in zip(buckets, state):
            bk.flat.copy_(flat); bk.m.copy_(m); bk.v.copy_(v); bk.step = step; bk.step_dev.copy_(step_dev)
            if avg is not None:
                bk.avg.copy_(avg)
            bk.epoch[0] += 1
            bk.plan.run()
        for n, saved in zip(nets, bufs):
            for x, s0 in zip(n.buffers(), saved):
                x.copy_(s0)
        restore_rng()
        out = t.train_step(data[1], z=z[1], eps=eps[1])
        return out, [g.flat.clone(), g.m.clone(), g.v.clone(), g.avg.clone()]

    out_b, b1 = without_display()
    _, b2 = without_display()
    # The next step's images (the generator's forward, which reads the weights and operand copies the display swapped
    # and restored) are bitwise those of the step without the display.  The generator's update after it is not
    # bit-repeatable even between two identical steps: it goes through the discriminators just updated, some of which
    # accumulate their weight gradients with atomics.  So the generator's weights, Adam moments and EMA after the step
    # are held to four times the spread of two identical steps without the display (with a floor of 1e-6 when those
    # two agree bit for bit).  On the H100 the display's difference and that spread were 3.63e-4 and 3.69e-4.
    for x, y in zip(out_a["fake_imgs"], out_b["fake_imgs"]):
        assert torch.equal(x, y)
    for x, y, y2, what in zip(a, b1, b2, ["weights", "m", "v", "EMA"]):
        d, spread = (x - y).abs().max().item(), (y2 - y).abs().max().item()
        print("generator %s after the next step: max |diff| %.3g, two steps without the display %.3g" % (what, d,
                                                                                                           spread))
        assert d <= max(4 * spread, 1e-6), what


# ---------------------------------------------------------------------------------- stored reference canvases
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_canvas_vs_stored_reference(name, monkeypatch):
    """The kernels against the canvases made by the reference's own functions (tests/golden/reference/
    snapshot_*.npz).  The caption strips' rows are left out: their glyphs are drawn by the host's Pillow."""
    c = C.CASES[name]
    f = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference", "snapshot_%s.npz" % name))
    assert abs(C.checksum(name) - float(f["checksum"])) <= 1e-9 * abs(float(f["checksum"]))
    imgs, lr, maps, lens, _ = (None if t is None else t.to(DEV) for t in C.inputs(name))
    if c.get("shape"):
        monkeypatch.setitem(cfg.ROI, "BOXES_NUM", c["words"])
        got = snapshots.super_shape_images(imgs, maps).pixels()
        strip = 20
    else:
        got = snapshots.super_images(imgs, None, None, maps, lr_images=lr, lens=lens, words=c["words"]).pixels()
        strip = 50
    want = f["canvas"]
    got = got[:want.shape[0]]
    vis = 272 if c["att"] == 17 else c["s"]
    keep = np.ones(want.shape[0], dtype=bool)
    for i in range(c["keep"]):
        keep[i * (strip + 2 * vis):i * (strip + 2 * vis) + strip] = False
    if c.get("shape"):
        assert np.array_equal(got[keep], want[keep])
    else:
        _near(got[keep], want[keep], name)
