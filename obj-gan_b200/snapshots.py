"""The attention-map snapshot PNGs of the training and evaluation loops (ref: miscc/utils.py:36-306, drawCaption /
build_super_images / build_super_shape_images).  The pixels of each PNG are composed on the device in one
og_snapshot_canvas call (ops.snapshot_canvas: image tiles, maps expanded with skimage's pyramid_expand(sigma=20),
normalisation, the 210/255 blend, pads and strip backgrounds) and read back once; the host draws only the caption
text, and a background thread PNG-encodes, so the loop's thread does not wait for either.

Differences from the reference where it breaks: nvis = min(8, B) (its build_super_images raises IndexError for B < 8),
the column count is cfg.TEXT.WORDS_NUM at call time, and 0 / 0 in the normalisation gives 0."""
from __future__ import annotations

import contextlib
import os
import queue
import threading

import numpy as np
import torch

from . import ops
from .config import cfg

FONT_MAX = 50          # caption-strip rows of build_super_images
SHAPE_STRIP = 20       # caption-strip rows of build_super_shape_images (its text lands beyond the canvas)
FONT_PATH = "/share/Pillow/Tests/fonts/FreeMono.ttf"


def load_font(font=None):
    """The caption font: ``font`` as a TrueType path or a PIL font; None: the reference's
    cfg.DATA_DIR + '/share/Pillow/Tests/fonts/FreeMono.ttf' at size 50.  None when it cannot be loaded."""
    from PIL import ImageFont
    if font is not None and not isinstance(font, (str, os.PathLike)):
        return font
    try:
        return ImageFont.truetype(str(font) if font is not None else cfg.DATA_DIR + FONT_PATH, FONT_MAX)
    except OSError:
        return None


def _to_host(t):
    """The one device -> host read of a canvas: an asynchronous copy into pinned memory on the current stream, and
    the event that marks it complete (None without CUDA)."""
    if not t.is_cuda:
        return t, None
    host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    host.copy_(t, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    return host, ev


def _square(maps, b):
    maps = maps.detach()
    if maps.dim() == 3:
        side = int(round(maps.shape[2] ** 0.5))
        maps = maps.reshape(b, maps.shape[1], side, side)
    return maps


class Canvas:
    """One PNG in flight: the host copy of the device canvas and what the text needs.  ``pixels()`` waits for the
    copy, draws the captions and returns the (H, W, 3) uint8 array."""

    def __init__(self, dev, captions, ixtoword, vis, nvis, strip, font):
        self.host, self.event = _to_host(dev)
        self.captions, self.ixtoword, self.vis, self.nvis, self.strip, self.font = \
            captions, ixtoword, vis, nvis, strip, font

    def pixels(self):
        if self.event is not None:
            self.event.synchronize()
        arr = self.host.numpy()
        if self.font is not None and self.captions is not None:
            draw_captions(arr, self.captions, self.ixtoword, self.vis, self.nvis, self.strip, self.font)
        return arr


def draw_captions(canvas, captions, ixtoword, vis, nvis, strip, font):
    """drawCaption on the strips of ``canvas`` in place: '%d:%s' % (j, word[:6]) in white at ((j + 2)(vis + 2),
    i * strip) for image i's tokens up to the first 0.  The strips are drawn as one contiguous canvas, as in the
    reference, so a caption's descenders reach into the next image's strip."""
    from PIL import Image, ImageDraw
    per = strip + 2 * vis
    rows = canvas.reshape(nvis, per, canvas.shape[1], 3)
    text = np.ascontiguousarray(rows[:, :strip]).reshape(nvis * strip, canvas.shape[1], 3)
    im = Image.fromarray(text)
    d = ImageDraw.Draw(im)
    caps = np.asarray(torch.as_tensor(captions).cpu())
    for i in range(min(nvis, caps.shape[0])):
        for j, ix in enumerate(caps[i]):
            if ix == 0:
                break
            word = ixtoword[int(ix)].encode("ascii", "ignore").decode("ascii")
            d.text(((j + 2) * (vis + 2), i * strip), "%d:%s" % (j, word[:6]), font=font, fill=(255, 255, 255, 255))
    rows[:, :strip] = np.asarray(im).reshape(nvis, strip, canvas.shape[1], 3)
    return canvas


def super_images(images, captions, ixtoword, maps, *, lr_images=None, lens=None, font=None, words=None) -> Canvas:
    """build_super_images(images, captions, ixtoword, maps, maps' side, lr_imgs=lr_images): the canvas of one PNG.
    ``maps`` (B, L, h, w) or (B, L, h * w) on the device; ``lens`` (B,) int64 per-image map counts (the DAMSM maps
    of caption i are its first cap_lens[i]); the tile side is 272 for 17-pixel maps, else the images' side."""
    b = images.shape[0]
    nvis = min(8, b)
    maps = _square(maps, b)
    att = maps.shape[2]
    vis = att * 16 if att == 17 else images.shape[2]
    words = cfg.TEXT.WORDS_NUM if words is None else words
    dev = ops.snapshot_canvas(images, maps, lr_images=lr_images, lens=lens, nvis=nvis, vis=vis, words=words,
                              strip=FONT_MAX, per_map=False)
    return Canvas(dev, captions, ixtoword, vis, nvis, FONT_MAX, font)


def super_shape_images(images, maps) -> Canvas:
    """build_super_shape_images' PNG (ref: evaluator.py:207-229): the real 64-pixel images and (B, R, 64, 64) shape
    maps, cfg.ROI.BOXES_NUM columns, per-map normalisation, no caption text."""
    b = images.shape[0]
    maps = _square(maps, b)
    dev = ops.snapshot_canvas(images, maps, nvis=min(8, b), vis=images.shape[2], words=cfg.ROI.BOXES_NUM,
                              strip=SHAPE_STRIP, per_map=True)
    return Canvas(dev, None, None, images.shape[2], min(8, b), SHAPE_STRIP, None)


class PngWriter:
    """PNG-encodes snapshot canvases on one background thread.  ``submit`` takes one display's [(path, Canvas)] and
    blocks while an earlier display is still queued, so a slow disk holds the loop back instead of growing memory; an
    error of the writer is raised by the next ``submit`` or by ``close``."""

    def __init__(self):
        self._q = queue.Queue(maxsize=1)
        self._thread = None
        self._error = None

    def _raise(self):
        if self._error is not None:
            err, self._error = self._error, None
            raise RuntimeError("writing a snapshot PNG failed") from err

    def _run(self):
        from PIL import Image
        while True:
            jobs = self._q.get()
            try:
                if jobs is None:
                    return
                for path, canvas in jobs:
                    Image.fromarray(canvas.pixels()).save(path)
            except BaseException as e:      # surfaced on the loop's thread
                self._error = e
            finally:
                self._q.task_done()

    def submit(self, jobs):
        self._raise()
        if self._thread is None:
            self._thread = threading.Thread(target=self._run, name="snapshot-png", daemon=True)
            self._thread.start()
        self._q.put(list(jobs))

    def close(self, raise_error=True):
        """Waits until every submitted PNG is written and stops the thread; raises a writer error unless
        ``raise_error`` is False (an exception already on its way out of the loop is not replaced)."""
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None
        if raise_error:
            self._raise()
        else:
            self._error = None


@contextlib.contextmanager
def writing(writer):
    """Closes ``writer`` (None: nothing) when the block ends: raising its error after a clean exit, quietly when the
    block raised."""
    try:
        yield writer
    except BaseException:
        if writer is not None:
            writer.close(raise_error=False)
        raise
    if writer is not None:
        writer.close()
