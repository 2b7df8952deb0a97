"""Host restatement of the attention-map snapshot PNGs (ref: image_generation/miscc/utils.py:36-306: drawCaption,
build_super_images, build_super_shape_images) and of skimage 0.14's ``skimage.transform.pyramid_expand``, which the
reference calls with ``sigma=20``.  numpy / scipy / PIL / torch on the CPU; float64 where the reference is float64
(every expanded map), float32 where it is float32 (image tiles, maps at unchanged size).

pyramid_expand(image, upscale, sigma) as skimage 0.14 computes it (restated from its documented behaviour; checked
against no installed skimage, so the rules are listed here for anyone who has one):
  1. bilinear ``resize`` to upscale * side with half-pixel centres: src = (dst + 0.5) / upscale - 0.5, the value
     (1 - dr) ((1 - dc) a[r0, c0] + dc a[r0, c1]) + dr ((1 - dc) a[r1, c0] + dc a[r1, c1]) with r0 = floor(src),
     r1 = ceil(src);
  2. neighbours outside the map come from numpy 'reflect' (mirror, the edge not repeated: -1 -> 1, n -> n - 2);
  3. the result is clipped to the input's min / max (``clip=True``);
  4. ``scipy.ndimage.gaussian_filter(sigma)`` on each channel (truncate 4: radius int(4 sigma + 0.5) = 80 for
     sigma 20), boundary scipy 'reflect' (half-sample symmetric: -1 -> 0);
  5. all in float64.  The snapshot maps carry three identical channels; one is computed and repeated.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image, ImageDraw
from scipy import ndimage

FONT_MAX = 50          # caption-strip rows of build_super_images
SHAPE_STRIP = 20       # caption-strip rows of build_super_shape_images
COLORS = [(128, 64, 128), (244, 35, 232), (70, 70, 70), (102, 102, 156), (190, 153, 153), (153, 153, 153),
          (250, 170, 30), (220, 220, 0), (107, 142, 35), (152, 251, 152), (70, 130, 180), (220, 20, 60),
          (255, 0, 0), (0, 0, 142), (119, 11, 32), (0, 60, 100), (0, 80, 100), (0, 0, 230), (0, 0, 70), (0, 0, 0)]


def _reflect_np(k, n):
    if n == 1:
        return np.zeros_like(k)
    return np.where(k < 0, -k, np.where(k > n - 1, 2 * (n - 1) - k, k))


def expand_plane(plane, upscale, sigma=20.0):
    """Steps 1-5 of the module docstring on one 2-D map."""
    a = np.asarray(plane, dtype=np.float64)
    h, w = a.shape

    def axis(n):
        s = (np.arange(n * upscale, dtype=np.float64) + 0.5) / upscale - 0.5
        lo, hi = np.floor(s).astype(np.int64), np.ceil(s).astype(np.int64)
        return _reflect_np(lo, n), _reflect_np(hi, n), s - lo

    r0, r1, dr = axis(h)
    c0, c1, dc = axis(w)
    dc = dc[None, :]
    top = (1 - dc) * a[r0][:, c0] + dc * a[r0][:, c1]
    bot = (1 - dc) * a[r1][:, c0] + dc * a[r1][:, c1]
    v = (1 - dr)[:, None] * top + dr[:, None] * bot
    v = np.clip(v, a.min(), a.max())
    return ndimage.gaussian_filter(v, sigma, mode="reflect", truncate=4.0)


def pyramid_expand(image, upscale=2, sigma=None, order=1, mode="reflect", cval=0, multichannel=None):
    """skimage.transform.pyramid_expand (0.14) for the arguments the reference passes: (h, w) or (h, w, C)."""
    a = np.asarray(image, dtype=np.float64)
    sigma = 2 * upscale / 6.0 if sigma is None else sigma
    if a.ndim == 2:
        return expand_plane(a, int(upscale), sigma)
    first = expand_plane(a[..., 0], int(upscale), sigma)
    chans = [first if np.array_equal(a[..., c], a[..., 0]) else expand_plane(a[..., c], int(upscale), sigma)
             for c in range(a.shape[2])]
    return np.stack(chans, axis=2)


def image_tiles(images, vis):
    """nn.Upsample(vis, bilinear, align_corners=False), then (x + 1) / 2 * 255 in float32: (n, vis, vis, 3)."""
    x = torch.as_tensor(images).detach().float().cpu()
    x = F.interpolate(x, size=(vis, vis), mode="bilinear", align_corners=False)
    x = x.add(1).div(2).mul(255)
    return x.permute(0, 2, 3, 1).numpy()


def to_u8(v):
    """np.uint8 truncation; NaN (0 / 0) gives 0, out-of-range values saturate."""
    v = np.asarray(v)
    return np.clip(np.where(np.isnan(v), 0, v), 0, 255).astype(np.uint8)


def blend210(img_u8, att_u8):
    """PIL paste(att, mask=L 210) over img: DIV255(img * 45 + att * 210) per byte."""
    v = img_u8.astype(np.int64) * 45 + att_u8.astype(np.int64) * 210 + 128
    return (((v >> 8) + v) >> 8).astype(np.uint8)


def strip_background(rows, words, vis):
    """The caption canvas before the text: ones, and column k + 2 in COLORS[k] for k < words."""
    s = np.ones((rows, (words + 2) * (vis + 2), 3), dtype=np.uint8)
    for k in range(words):
        s[:, (k + 2) * (vis + 2):(k + 3) * (vis + 2)] = COLORS[k]
    return s


def draw_captions(strip, captions, ixtoword, vis, font, row_step=FONT_MAX):
    """drawCaption: '%d:%s' % (j, word[:6]) in white at ((j + 2)(vis + 2), i * row_step) until the first 0 token."""
    im = Image.fromarray(strip)
    d = ImageDraw.Draw(im)
    caps = np.asarray(torch.as_tensor(captions).cpu())
    for i in range(caps.shape[0]):
        for j, ix in enumerate(caps[i]):
            if ix == 0:
                break
            word = ixtoword[int(ix)].encode("ascii", "ignore").decode("ascii")
            d.text(((j + 2) * (vis + 2), i * row_step), "%d:%s" % (j, word[:6]), font=font, fill=(255, 255, 255, 255))
    return np.asarray(im).astype(np.uint8)


def _maps_of(maps_i, att):
    m = torch.as_tensor(maps_i).detach().cpu().float().reshape(-1, att, att).numpy()
    return [m.max(axis=0)] + list(m)


def super_images(real_imgs, captions, ixtoword, attn_maps, att_sze, lr_imgs=None, words=18, font=None,
                 batch_rows=None):
    """build_super_images with nvis = min(8, B); ``attn_maps[i]`` holds image i's maps (any shape with att^2 per
    map).  The caption strip is one canvas of ``batch_rows`` (default B) x 50 rows, text drawn when ``font``."""
    b = real_imgs.shape[0]
    nvis = min(8, b)
    vis = att_sze * 16 if att_sze == 17 else real_imgs.shape[2]
    up = vis // att_sze
    imgs = image_tiles(real_imgs[:nvis], vis)
    lrs = imgs if lr_imgs is None else image_tiles(lr_imgs[:nvis], vis)
    text = strip_background((batch_rows or b) * FONT_MAX, words, vis)
    if font is not None:
        text = draw_captions(text, captions, ixtoword, vis, font)
    rows = []
    pad = np.zeros((vis, 2, 3), dtype=np.uint8)
    zero = np.zeros((vis, vis, 3), dtype=np.uint8)
    for i in range(nvis):
        maps = _maps_of(attn_maps[i], att_sze)
        if up > 1:
            maps = [expand_plane(m, up) for m in maps]
        mn, mx = 1, 0
        for m in maps:
            if mn > m.min():
                mn = m.min()
            if mx < m.max():
                mx = m.max()
        img_u8 = to_u8(imgs[i])
        top, bot = [to_u8(lrs[i]), pad], [img_u8, pad]
        with np.errstate(invalid="ignore", divide="ignore"):
            for j in range(words + 1):
                if j < len(maps):
                    q = (maps[j] - mn) / (mx - mn)
                    q = q * (np.float32(255) if q.dtype == np.float32 else 255.0)
                    a = np.repeat(to_u8(q)[..., None], 3, 2)
                    top += [a, pad]
                    bot += [blend210(img_u8, a), pad]
                else:
                    top += [zero, pad]
                    bot += [zero, pad]
        rows += [text[i * FONT_MAX:(i + 1) * FONT_MAX], np.concatenate(top, 1), np.concatenate(bot, 1)]
    return np.concatenate(rows, 0)


def super_shape_images(real_imgs, attn_maps, boxes_num=10):
    """build_super_shape_images's PNG: nvis = min(8, B), 20-row strips without text (the reference's caption offsets
    put it beyond the canvas), per-map min / max guarded by max != min, no expansion (maps at the image's side),
    float32 arithmetic."""
    b = real_imgs.shape[0]
    nvis = min(8, b)
    vis = real_imgs.shape[2]
    att = vis
    imgs = image_tiles(real_imgs[:nvis], vis)
    text = strip_background(b * SHAPE_STRIP, boxes_num, vis)
    rows = []
    pad = np.zeros((vis, 2, 3), dtype=np.uint8)
    zero = np.zeros((vis, vis, 3), dtype=np.uint8)
    for i in range(nvis):
        maps = _maps_of(attn_maps[i], att)
        img_u8 = to_u8(imgs[i])
        top, bot = [img_u8, pad], [img_u8, pad]
        for j in range(boxes_num + 1):
            if j < len(maps):
                m = maps[j]
                mn, mx = m.min(), m.max()
                if mx != mn:
                    m = (m - mn) / (mx - mn)
                a = np.repeat(to_u8(m * np.float32(255))[..., None], 3, 2)
                top += [a, pad]
                bot += [blend210(img_u8, a), pad]
            else:
                top += [zero, pad]
                bot += [zero, pad]
        rows += [text[i * SHAPE_STRIP:(i + 1) * SHAPE_STRIP], np.concatenate(top, 1), np.concatenate(bot, 1)]
    return np.concatenate(rows, 0)
