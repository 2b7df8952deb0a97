"""CPU tests of the snapshot PNGs: the host oracle (oracle/snapshot_oracle.py) bitwise against the reference's own
build_super_images / build_super_shape_images / drawCaption (with the oracle's pyramid_expand in place of skimage's
and Pillow's built-in font at size 50 in place of FreeMono), pyramid_expand worked by hand, and the host side of
snapshots.py without a GPU: one og_snapshot_canvas call per PNG, the canvas geometry, the caption strips, the font
fallback and the background writer."""
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image, ImageFont

import refimport
import snapshot_cases as C
from objgan_b200 import lib, snapshots
from objgan_b200.config import cfg
from oracle import snapshot_oracle as O

FONT = ImageFont.load_default(size=50)
IXTOWORD = {i: "w%dqyjg" % i for i in range(1, 60)}


@pytest.fixture(scope="module")
def ref():
    if not refimport.available():
        pytest.skip("the reference is not available")
    r = refimport.load(18)
    sys.modules["skimage.transform"].pyramid_expand = O.pyramid_expand
    return r


@pytest.fixture()
def default_font(monkeypatch):
    monkeypatch.setattr(ImageFont, "truetype", lambda *a, **k: FONT)


def _case(b, s, att, L, lr, const=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(b, 3, s, s, generator=g) * 2 - 1
    lri = torch.rand(b, 3, s // 2, s // 2, generator=g) * 2 - 1 if lr else None
    maps = torch.softmax(torch.randn(b, L, att, att, generator=g) * 3, 1)
    if const is not None:
        maps.fill_(const)
    caps = torch.randint(1, 60, (b, 14), generator=g)
    caps[min(1, b - 1), 5:] = 0
    return imgs, lri, maps, caps


@pytest.mark.parametrize("b,s,att,L,lr,const", [
    (8, 128, 64, 5, True, None), (16, 128, 64, 18, True, None), (8, 256, 128, 3, True, None),
    (8, 256, 17, 4, False, None), (16, 256, 17, 20, False, None), (8, 64, 64, 22, False, None),
    (8, 128, 64, 3, True, 0.5)])
def test_super_images_vs_reference(ref, default_font, b, s, att, L, lr, const):
    imgs, lri, maps, caps = _case(b, s, att, L, lr, const)
    with np.errstate(all="ignore"):
        want, _ = ref.utils.build_super_images(imgs, caps, IXTOWORD, maps, att, lr_imgs=lri)
    got = O.super_images(imgs, caps, IXTOWORD, maps, att, lr_imgs=lri, words=18, font=FONT)
    assert np.array_equal(got, want)


def test_super_images_ragged_vs_reference(ref, default_font):
    """DAMSM maps: caption i has its own count of 17-pixel maps."""
    imgs, _, maps, caps = _case(8, 256, 17, 9, False, seed=1)
    lens = [9, 3, 7, 1, 9, 2, 5, 4]
    per = [maps[i:i + 1, :n] for i, n in enumerate(lens)]
    want, _ = ref.utils.build_super_images(imgs, caps, IXTOWORD, per, 17)
    assert np.array_equal(O.super_images(imgs, caps, IXTOWORD, per, 17, words=18, font=FONT), want)


@pytest.mark.parametrize("b,r", [(3, 4), (8, 10), (16, 80)])
def test_super_shape_images_vs_reference(ref, default_font, b, r):
    g = torch.Generator().manual_seed(b)
    imgs = torch.rand(b, 3, 64, 64, generator=g) * 2 - 1
    hm = torch.rand(b, r, 64, 64, generator=g)
    hm[:, 1] = 0
    caps = torch.randint(1, 60, (b, 10), generator=g)            # drawn beyond the canvas by the reference
    want, _ = ref.utils.build_super_shape_images(imgs, caps, IXTOWORD, hm, 64, font_max=20, font_size=12,
                                                 max_word_num=10, batch_size=b)
    assert np.array_equal(O.super_shape_images(imgs, hm, 10), want)


def test_draw_captions_vs_reference(ref, default_font):
    _, _, _, caps = _case(4, 64, 64, 1, False, seed=3)
    strip = O.strip_background(4 * 50, 18, 128)
    want, _ = ref.utils.drawCaption(strip.copy(), caps, IXTOWORD, 128)
    assert np.array_equal(O.draw_captions(strip, caps, IXTOWORD, 128, FONT), np.asarray(want))


def test_library_captions_match_oracle():
    """snapshots.draw_captions on a canvas of strips and tiles gives the oracle's strips, descenders included."""
    nvis, vis, words = 3, 64, 18
    _, _, _, caps = _case(nvis, vis, vis, 1, False, seed=4)
    width = (words + 2) * (vis + 2)
    per = 50 + 2 * vis
    canvas = np.zeros((nvis * per, width, 3), dtype=np.uint8)
    bg = O.strip_background(nvis * 50, words, vis)
    for i in range(nvis):
        canvas[i * per:i * per + 50] = bg[i * 50:(i + 1) * 50]
    snapshots.draw_captions(canvas, caps, IXTOWORD, vis, nvis, 50, FONT)
    want = O.draw_captions(bg, caps, IXTOWORD, vis, FONT)
    for i in range(nvis):
        assert np.array_equal(canvas[i * per:i * per + 50], want[i * 50:(i + 1) * 50])
        assert not canvas[i * per + 50:(i + 1) * per].any()


# ----------------------------------------------------------------------------- pyramid_expand worked by hand
def test_pyramid_expand_constant():
    out = O.pyramid_expand(np.full((17, 17, 3), 0.25, np.float32), upscale=16, sigma=20)
    assert out.shape == (272, 272, 3) and out.dtype == np.float64
    np.testing.assert_allclose(out, 0.25, rtol=0, atol=1e-15)


def test_pyramid_expand_centred_impulse_is_symmetric():
    a = np.zeros((9, 9))
    a[4, 4] = 1.0
    out = O.pyramid_expand(a, upscale=16, sigma=20)
    np.testing.assert_allclose(out, out[::-1], atol=1e-15)
    np.testing.assert_allclose(out, out.T, atol=1e-15)
    assert np.unravel_index(out.argmax(), out.shape) in {(71, 71), (71, 72), (72, 71), (72, 72)}


def test_pyramid_expand_boundary_rules():
    """Resize: numpy reflect (-1 -> 1); blur: half-sample symmetric (-1 -> 0), here with sigma small enough to
    follow by hand."""
    a = np.array([[0.0, 1.0, 4.0]])
    a = np.repeat(a, 3, 0)
    r = O.expand_plane(a, 2, sigma=1e-9)                 # a blur of width ~0: the resize alone
    # output column 0: src = -0.25 -> 0.75 * a[0] + 0.25 * a[reflect(-1) = 1]
    np.testing.assert_allclose(r[0], [0.25, 0.25, 0.75, 1.75, 3.25, 3.25], atol=1e-12)
    # the clip of step 3 keeps the values inside [0, 4]; the Gaussian with a half-sample mirror keeps a constant row
    line = np.tile(np.arange(6.0), (6, 1))
    b = O.ndimage.gaussian_filter(line, 1.0, mode="reflect")
    mirrored = np.concatenate([line[:, ::-1], line, line[:, ::-1]], 1)
    want = O.ndimage.gaussian_filter(mirrored, 1.0, mode="nearest")[:, 6:12]
    np.testing.assert_allclose(b, want, atol=1e-12)


# ----------------------------------------------------------------------------- host logic without a GPU
@pytest.fixture()
def dry():
    lib.DRY_RUN = True
    yield
    lib.DRY_RUN = False


def test_one_call_per_png_and_geometry(dry, monkeypatch):
    monkeypatch.setitem(cfg.TEXT, "WORDS_NUM", 18)
    n0 = lib.get().launches
    c = snapshots.super_images(torch.zeros(16, 3, 256, 256), None, None, torch.zeros(16, 12, 17, 17),
                               lens=torch.full((16,), 5, dtype=torch.int64))
    assert lib.get().launches - n0 == 1
    assert c.host.shape == (8 * (50 + 2 * 272), 20 * 274, 3)
    s = snapshots.super_shape_images(torch.zeros(3, 3, 64, 64), torch.zeros(3, 80, 64, 64))
    assert lib.get().launches - n0 == 2
    assert s.host.shape == (3 * (20 + 128), 12 * 66, 3)
    g = snapshots.super_images(torch.zeros(2, 3, 128, 128), None, None, torch.zeros(2, 7, 64 * 64),
                               lr_images=torch.zeros(2, 3, 64, 64))
    assert g.host.shape == (2 * (50 + 256), 20 * 130, 3)


def test_unsupported_geometry_is_refused(dry):
    with pytest.raises(ValueError):
        snapshots.super_images(torch.zeros(2, 3, 100, 100), None, None, torch.zeros(2, 3, 30, 30))
    with pytest.raises(ValueError):
        snapshots.super_images(torch.zeros(2, 3, 128, 128), None, None, torch.zeros(2, 3, 64, 64), words=21)
    with pytest.raises(ValueError, match="lens"):                   # fewer counts than images shown
        snapshots.super_images(torch.zeros(4, 3, 256, 256), None, None, torch.zeros(4, 3, 17, 17),
                               lens=torch.ones(2, dtype=torch.int64))


def test_font_fallback(monkeypatch, tmp_path):
    monkeypatch.setitem(cfg, "DATA_DIR", str(tmp_path))
    assert snapshots.load_font() is None
    assert snapshots.load_font(FONT) is FONT
    assert snapshots.load_font(str(tmp_path / "missing.ttf")) is None


class _Pixels:
    def __init__(self, arr=None, fail=False):
        self.arr, self.fail = arr, fail

    def pixels(self):
        if self.fail:
            raise OSError("disk full")
        return self.arr


def test_writer_drains_and_surfaces_errors(tmp_path):
    w = snapshots.PngWriter()
    arr = np.arange(4 * 5 * 3, dtype=np.uint8).reshape(4, 5, 3)
    w.submit([(str(tmp_path / f"a{i}.png"), _Pixels(arr)) for i in range(3)])
    w.submit([(str(tmp_path / "b.png"), _Pixels(arr))])
    w.close()
    for name in ("a0.png", "a1.png", "a2.png", "b.png"):
        assert np.array_equal(np.asarray(Image.open(tmp_path / name)), arr)
    w = snapshots.PngWriter()
    w.submit([(str(tmp_path / "c.png"), _Pixels(fail=True))])
    with pytest.raises(RuntimeError, match="snapshot PNG"):
        w.close()
    w = snapshots.PngWriter()
    w.submit([(str(tmp_path / "d.png"), _Pixels(fail=True))])
    w._q.join()
    with pytest.raises(RuntimeError):
        w.submit([(str(tmp_path / "e.png"), _Pixels(arr))])
    w.close()


# ----------------------------------------------------------------------------- stored reference canvases
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_oracle_vs_stored_reference(name):
    """The oracle against the canvases the reference's own functions made (tests/golden/make_snapshot_golden.py),
    text included, where the reference itself is absent."""
    import os
    c = C.CASES[name]
    f = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference", "snapshot_%s.npz" % name))
    assert abs(C.checksum(name) - float(f["checksum"])) <= 1e-9 * abs(float(f["checksum"]))
    imgs, lr, maps, lens, caps = C.inputs(name)
    if c.get("shape"):
        got = O.super_shape_images(imgs, maps, c["words"])
    else:
        per = [maps[i, :int(lens[i])] for i in range(c["b"])] if lens is not None else maps
        with np.errstate(all="ignore"):
            got = O.super_images(imgs, caps, C.IXTOWORD, per, c["att"], lr_imgs=lr, words=c["words"], font=FONT)
    assert np.array_equal(got[:C.rows(name)], f["canvas"])
