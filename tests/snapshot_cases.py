"""The inputs of the snapshot fixtures (tests/golden/reference/snapshot_*.npz, written by
tests/golden/make_snapshot_golden.py from the reference's own build_super_images / build_super_shape_images /
drawCaption): rebuilt from seeds with torch's CPU generator on every machine, checked against the stored checksum.
Images and shape maps are smooth (bilinear from 8 x 8) so the stored canvases compress; only the first ``keep``
images' rows of each canvas are stored."""
import torch
import torch.nn.functional as F

CASES = {
    "g64": dict(b=8, s=128, lr=64, att=64, L=3, words=2, keep=1, seed=11),
    "g128": dict(b=8, s=256, lr=128, att=128, L=2, words=1, keep=1, seed=12),
    "d17": dict(b=8, s=256, lr=None, att=17, L=5, lens=[5, 2, 4, 1, 5, 3, 2, 4], words=1, keep=1, seed=13),
    "const": dict(b=8, s=128, lr=64, att=64, L=2, words=2, keep=1, seed=14, const=0.5),
    "shape_r4": dict(b=3, s=64, att=64, L=4, words=10, keep=2, seed=15, shape=True),
    "shape_r80": dict(b=8, s=64, att=64, L=80, words=10, keep=1, seed=16, shape=True),
}
IXTOWORD = {i: "w%dqyjg" % i for i in range(1, 60)}


def _smooth(g, b, c, s):
    return F.interpolate(torch.rand(b, c, 8, 8, generator=g), size=(s, s), mode="bilinear", align_corners=False)


def inputs(name):
    """(images, lr_images or None, maps (B, L, att, att), lens or None, captions (B, 14)) on the CPU."""
    c = CASES[name]
    g = torch.Generator().manual_seed(c["seed"])
    imgs = _smooth(g, c["b"], 3, c["s"]) * 2 - 1
    lr = _smooth(g, c["b"], 3, c["lr"]) * 2 - 1 if c.get("lr") else None
    if c.get("shape"):
        maps = _smooth(g, c["b"], c["L"], c["att"]) * 2
        maps[:, 0] = 0                                 # an empty class channel: max == min
    else:
        maps = torch.softmax(torch.randn(c["b"], c["L"], c["att"], c["att"], generator=g) * 3, 1)
    if c.get("const") is not None:
        maps.fill_(c["const"])
    lens = torch.tensor(c["lens"]) if "lens" in c else None
    caps = torch.randint(1, 60, (c["b"], 14), generator=g)
    caps[1, 5:] = 0
    return imgs, lr, maps, lens, caps


def checksum(name):
    imgs, lr, maps, _, caps = inputs(name)
    return float(sum(t.double().sum() for t in (imgs, maps, caps) + ((lr,) if lr is not None else ())))


def rows(name):
    """Rows of the stored part of the canvas: the first ``keep`` images."""
    c = CASES[name]
    vis = 272 if c["att"] == 17 else c["s"]
    strip = 20 if c.get("shape") else 50
    return c["keep"] * (strip + 2 * vis)
