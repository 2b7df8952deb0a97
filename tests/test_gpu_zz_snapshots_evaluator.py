"""The evaluator's snapshot PNGs on the GPU (condGANEvaluator with SAVE_OPTIONS = 'SNAPSHOT', modes 0, 1 and 2, one
display batch): the expected file set; each PNG's pixels against the oracle composed from the images and maps the
library passed (attention-map PNGs within one byte, at most 1e-3 of the bytes differing; shape PNGs bitwise); the
real 64-pixel images of the shape PNGs equal to the loader's, in the batch's caption-length order; and in mode 1 the
ground-truth heat maps rebuilt on the device equal to the loader's.  (File name sorts last: it builds every network
of the evaluation.)"""
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFont

from objgan_b200 import evaluator, losses, snapshots, synth
from objgan_b200.config import cfg
from oracle import snapshot_oracle as O
from test_gpu_snapshots import _near
from test_gpu_zz_evaluator import B, DIMS, N_WORDS, POOL, _batch, _cfg, _noise, files  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
FONT = ImageFont.load_default(size=50)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_evaluator_snapshots_vs_oracle(mode, files, tmp_path, monkeypatch):  # noqa: F811
    _cfg(monkeypatch, files, mode)
    monkeypatch.setitem(cfg.TEST, "SAVE_OPTIONS", "SNAPSHOT")
    monkeypatch.setitem(cfg.TRAIN, "DISPLAY_INTERVAL", 1)
    monkeypatch.setitem(cfg.TEXT, "WORDS_NUM", 18)
    ds = synth.reference_test_dataset(n_words=N_WORDS)
    ds.ixtoword = {i: "w%dgjy" % i for i in range(N_WORDS)}
    e = evaluator.condGANEvaluator(str(tmp_path), [None], ds, inception_weights=files["inc"], device=DEV, font=FONT)
    e.build_models()
    used = []
    real_si, real_ssi = snapshots.super_images, snapshots.super_shape_images

    def si(images, captions, ixtoword, maps, **kw):
        lr = kw.get("lr_images")
        used.append(("G", images.cpu(), captions, maps.cpu(), None if lr is None else lr.cpu()))
        return real_si(images, captions, ixtoword, maps, **kw)

    def ssi(images, maps):
        used.append(("S", images.cpu(), None, maps.cpu(), None))
        return real_ssi(images, maps)
    monkeypatch.setattr(snapshots, "super_images", si)
    monkeypatch.setattr(snapshots, "super_shape_images", ssi)
    data = _batch(mode, 0)
    z, eps, noise_shp = (t.to(DEV) for t in _noise(0))
    rp, is_, fid = losses.RPrecision(POOL), losses.InceptionScore(min(10, B)), losses.FrechetDistance(DIMS)
    out = e.evaluate_batch(data, rp, is_, fid, z=z, eps=eps, noise_shp=noise_shp, gen_iterations=0)
    e.close_writer()
    names = ["G_0_0.png", "bt_G_0_0.png", "G_0_1.png", "bt_G_0_1.png"]
    names += ["ShapeG_0.png"] if mode > 0 else []
    names += ["ShapeD_0.png"] if mode == 1 else []
    assert sorted(os.listdir(tmp_path / "Snapshot")) == sorted(names)
    assert len(used) == len(names)
    for name, (kind, images, captions, maps, lr) in zip(names, used):
        png = np.asarray(Image.open(tmp_path / "Snapshot" / name))
        if kind == "S":
            assert np.array_equal(png, O.super_shape_images(images, maps, cfg.ROI.BOXES_NUM)), name
        else:
            want = O.super_images(images, captions, ds.ixtoword, maps, maps.shape[-1], lr_imgs=lr, words=18,
                                  font=FONT)
            _near(png, want, name)
    if mode > 0:
        keys = list(data[15] if mode == 1 else data[12])
        perm = [keys.index(k) for k in out["keys"]]
        imgs0 = torch.as_tensor(data[0][0])[perm].float()
        assert torch.equal(used[4][1], imgs0)                               # ShapeG: the loader's images, sorted
        assert used[4][3].shape[:2] == (B, int(torch.as_tensor(data[11 if mode == 1 else 10]).max()))   # SHP_G_NET's (B, R) masks
    if mode == 1:
        assert torch.equal(used[5][1], imgs0)
        hm = torch.as_tensor(data[5][0])[perm].float()
        assert used[5][3].shape == hm.shape
        torch.testing.assert_close(used[5][3], hm, rtol=0, atol=1e-6)       # ShapeD: the ground-truth heat maps
