"""Seeded synthetic COCO-shaped inputs for the image_generation training step.

Shapes follow what the reference's data pipeline hands to ``condGANTrainer.train``
(reference: image_generation/trainDataset.py:79-128 ``prepare_data``,
image_generation/trainer.py:357-393) with the dataset replaced by random draws, as
SURVEY.md section 8(d) specifies.  Everything is generated on the CPU with an explicit
``torch.Generator`` so the same call gives the same tensors here and on the GPU box.
"""
from __future__ import annotations

import numpy as np
import torch

from .config import cfg

IMG_SIZES = (64, 128, 256)


def _ellipse_masks(boxes: torch.Tensor, num_rois: torch.Tensor, size: int, scale: float) -> torch.Tensor:
    """Filled axis-aligned ellipse inside each box, 1.0 inside with a one-pixel soft edge.

    boxes: (B, R, 4) float64 [x, y, w, h] at 64-pixel scale; returns (B, R, size, size) float32.
    """
    B, R, _ = boxes.shape
    ys = torch.arange(size, dtype=torch.float64).view(1, 1, size, 1) + 0.5
    xs = torch.arange(size, dtype=torch.float64).view(1, 1, 1, size) + 0.5
    x = (boxes[..., 0] * scale).view(B, R, 1, 1)
    y = (boxes[..., 1] * scale).view(B, R, 1, 1)
    w = (boxes[..., 2] * scale).clamp(min=1.0).view(B, R, 1, 1)
    h = (boxes[..., 3] * scale).clamp(min=1.0).view(B, R, 1, 1)
    cx, cy, rx, ry = x + w / 2, y + h / 2, w / 2, h / 2
    # signed "distance" in pixels along the ellipse normal (approximate), soft edge of 1 px
    d = (((xs - cx) / rx) ** 2 + ((ys - cy) / ry) ** 2).sqrt()
    edge = (1.0 - d) * torch.minimum(rx, ry)
    m = edge.clamp(0.0, 1.0)
    valid = (torch.arange(R).view(1, R) < num_rois.view(B, 1)).view(B, R, 1, 1)
    return (m * valid).float()


def make_inputs(batch: int, seed: int = 1234, *, words: int | None = None, max_rois: int | None = None,
                parity: bool = False, num_classes: int = 80) -> dict:
    """Build one batch of step inputs (all CPU tensors).

    parity=False: throughput workload -- every caption has ``words`` tokens (mask all False) and
    every image has ``max_rois`` boxes.  parity=True: ragged caption lengths (sorted descending,
    as ``prepare_data`` does) and 1..max_rois boxes per image, so the mask quirk and the padded
    roi slots are exercised.
    """
    L = int(words if words is not None else cfg.TEXT.WORDS_NUM)
    RB = cfg.ROI.BOXES_NUM
    Rm = int(max_rois if max_rois is not None else RB)
    g = torch.Generator().manual_seed(seed)
    B = batch

    def randn(*s):
        return torch.randn(*s, generator=g)

    def rand(*s):
        return torch.rand(*s, generator=g)

    z = randn(B, cfg.GAN.Z_DIM)
    eps = randn(B, cfg.GAN.CONDITION_DIM)  # CA_NET reparametrisation noise, injected for parity
    sent_emb = rand(B, cfg.TEXT.EMBEDDING_DIM) * 2 - 1
    words_embs = rand(B, cfg.TEXT.EMBEDDING_DIM, L) * 2 - 1
    glove_words_embs = 0.5 * randn(B, cfg.TEXT.GLOVE_EMBEDDING_DIM, L)
    clabels_emb = 0.5 * randn(num_classes, cfg.TEXT.GLOVE_EMBEDDING_DIM)

    if parity:
        cap_lens = torch.randint(5, L + 1, (B,), generator=g)
        cap_lens[0] = L  # the text encoder emits max(cap_lens) words; keep that equal to L
        cap_lens = torch.sort(cap_lens, descending=True).values
        num_rois = torch.randint(1, Rm + 1, (B,), generator=g)
        num_rois[B // 2] = Rm
    else:
        cap_lens = torch.full((B,), L, dtype=torch.long)
        num_rois = torch.full((B,), Rm, dtype=torch.long)
    mask = torch.arange(L).view(1, L) >= cap_lens.view(B, 1)  # (B, L) bool, True = padding

    xy = rand(B, RB, 2).double() * 40.0
    wh = 6.0 + rand(B, RB, 2).double() * 18.0
    wh = torch.minimum(wh, 64.0 - xy)
    cls = torch.randint(0, num_classes, (B, RB), generator=g).double()
    rois0 = torch.cat([xy, wh, cls.unsqueeze(-1), torch.zeros(B, RB, 1, dtype=torch.float64)], dim=2)
    valid = (torch.arange(RB).view(1, RB) < num_rois.view(B, 1)).unsqueeze(-1)
    rois0 = rois0 * valid
    rois = []
    for i in range(3):
        r = rois0.clone()
        r[..., :4] *= 2.0 ** i
        rois.append(r)
    fm_rois = rois0.clone()
    fm_rois[..., :4] /= 2.0

    boxes = rois0[..., :4]
    bt_masks = [_ellipse_masks(boxes, num_rois, s, s / 64.0) for s in IMG_SIZES]
    fm_bt_masks = _ellipse_masks(boxes, num_rois, 32, 0.5)
    hmaps = []
    cls_idx = cls.long()
    for i, s in enumerate(IMG_SIZES):
        hm = torch.zeros(B, num_classes, s, s)
        hm.scatter_add_(1, cls_idx.view(B, RB, 1, 1).expand(B, RB, s, s), bt_masks[i])
        hmaps.append(hm.clamp_(max=1.0))

    # slabels_feat: class-label GloVe vectors per roi, (B, 50, Rmax, 1) -- reference
    # image_generation/miscc/utils.py:502-522 (form_clabels_feat)
    rmax = int(num_rois.max())
    slabels = torch.zeros(B, rmax, clabels_emb.shape[1])
    for b in range(B):
        n = int(num_rois[b])
        slabels[b, :n] = clabels_emb[cls_idx[b, :n]]
    slabels_feat = slabels.transpose(1, 2).unsqueeze(3).contiguous()

    imgs = [rand(B, 3, s, s) * 2 - 1 for s in IMG_SIZES]

    return dict(z=z, eps=eps, sent_emb=sent_emb, words_embs=words_embs, glove_words_embs=glove_words_embs,
                clabels_emb=clabels_emb, slabels_feat=slabels_feat, cap_lens=cap_lens, mask=mask,
                num_rois=num_rois, rois=rois, fm_rois=fm_rois, bt_masks=bt_masks, fm_bt_masks=fm_bt_masks,
                hmaps=hmaps, imgs=imgs, glb_max_num_roi=rmax)


HMAP_CLAMP = 1.0     # make_inputs clamps its synthetic class heat maps at 1 (the reference's loader does not clamp)


def compact(inp: dict) -> dict:
    """The batch as it needs to cross PCIe: without the two tensors the device rebuilds from the rest
    (``hmaps`` = per-class sums of ``bt_masks``, 86 % of the bytes; ``slabels_feat`` = label embeddings of the roi
    classes), plus the roi class ids as an int64 table (column 4 of ``rois[0]``)."""
    out = {k: v for k, v in inp.items() if k not in ("hmaps", "slabels_feat")}
    out["roi_cls"] = inp["rois"][0][..., 4].to(torch.int64).contiguous()
    return out


def input_bytes(inp: dict) -> int:
    """Bytes a step copies host->device (every tensor in the batch)."""
    n = 0
    for v in inp.values():
        if torch.is_tensor(v):
            n += v.numel() * v.element_size()
        elif isinstance(v, (list, tuple)):
            n += sum(t.numel() * t.element_size() for t in v if torch.is_tensor(t))
    return n


def shard(inp: dict, rank: int, world: int) -> dict:
    """Data-parallel shard: samples [rank*B/world, (rank+1)*B/world) of every per-sample tensor
    (what ``nn.DataParallel``'s scatter does on dim 0; reference trainer.py:136-152)."""
    B = inp["z"].shape[0]
    assert B % world == 0
    lo, hi = rank * B // world, (rank + 1) * B // world
    out = {}
    for k, v in inp.items():
        if k == "clabels_emb" or k == "glb_max_num_roi":
            out[k] = v
        elif torch.is_tensor(v):
            out[k] = v[lo:hi].contiguous()
        else:
            out[k] = [t[lo:hi].contiguous() for t in v]
    rmax = int(out["num_rois"].max())
    out["glb_max_num_roi"] = rmax
    out["slabels_feat"] = out["slabels_feat"][:, :, :rmax].contiguous()
    return out


def reference_batch(batch: int, seed: int = 1234, *, lens=None, parity: bool = True, max_rois: int | None = None,
                    n_words: int = 200, n_glove: int = 200, num_classes: int = 80):
    """One batch in the format the reference's DataLoader collates from ``TrainDataset.__getitem__`` (ref:
    trainDataset.py:56-74, miscc/load.py:112-191): (imgs, captions (B, 18, 1) int64, glove_captions (B, 18, 1),
    cap_lens (B,) UNSORTED, hmaps (float64 per-class sums of the masks, unclamped), rois, fm_rois, num_rois, bt_masks
    and fm_bt_masks (float64), class_ids (B,), keys (B strings)).  The boxes, masks and images are ``make_inputs``'s
    (``parity``: ragged roi counts); ``lens``: the caption lengths (default: seeded draws in [5, 18]); token ids are
    drawn in [1, n_words) / [1, n_glove) on the first cap_lens[b] positions and 0 after."""
    inp = make_inputs(batch, seed, parity=parity, max_rois=max_rois, num_classes=num_classes)
    g = torch.Generator().manual_seed(seed + 1)
    L = cfg.TEXT.WORDS_NUM
    lens = torch.randint(5, L + 1, (batch,), generator=g) if lens is None else torch.as_tensor(lens, dtype=torch.int64)
    pos = torch.arange(L).view(1, L) < lens.view(-1, 1)
    caps = (torch.randint(1, n_words, (batch, L), generator=g) * pos).view(batch, L, 1)
    gcaps = (torch.randint(1, n_glove, (batch, L), generator=g) * pos).view(batch, L, 1)
    cls = inp["rois"][0][..., 4].long()
    hmaps = []
    for m in inp["bt_masks"]:
        s = m.shape[-1]
        hm = torch.zeros(batch, num_classes, s, s, dtype=torch.float64)
        hmaps.append(hm.scatter_add_(1, cls.view(batch, -1, 1, 1).expand(-1, -1, s, s), m.double()))
    class_ids = torch.randint(0, 100000, (batch,), generator=g)
    keys = [f"COCO_train2014_{seed:06d}{i:06d}" for i in range(batch)]
    return (inp["imgs"], caps, gcaps, lens, hmaps, inp["rois"], inp["fm_rois"], inp["num_rois"],
            [m.double() for m in inp["bt_masks"]], inp["fm_bt_masks"].double(), class_ids, keys)


def reference_dataset(n_words: int = 200, n_glove: int = 200, num_classes: int = 80, seed: int = 0):
    """An object with the attributes the reference's condGANTrainer reads from its ``TrainDataset`` (n_words,
    cats_index_dict, cat_labels, cat_label_lens, sorted_cat_label_indices, glove_embed), seeded: labels of one or
    two GloVe tokens, sorted by length as load_cat_label does (ref: miscc/load.py:305-355)."""
    import types
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, 3, (num_classes,), generator=g)
    order = torch.sort(lens, stable=True).indices
    labels = torch.randint(1, n_glove, (num_classes, 2), generator=g) * (torch.arange(2).view(1, 2) < lens.view(-1, 1))
    glove = torch.nn.Embedding(n_glove, cfg.TEXT.GLOVE_EMBEDDING_DIM)
    with torch.no_grad():
        glove.weight.copy_(0.5 * torch.randn(n_glove, cfg.TEXT.GLOVE_EMBEDDING_DIM, generator=g))
    return types.SimpleNamespace(n_words=n_words, cats_index_dict={i: i for i in range(num_classes)},
                                 cat_labels=labels[order], cat_label_lens=lens[order],
                                 sorted_cat_label_indices=torch.argsort(order), glove_embed=glove)


def reference_encoders(directory: str, n_words: int = 200, seed: int = 0) -> str:
    """Writes seeded DAMSM encoder snapshots in the reference's layout, ``text_encoder100.pth`` and
    ``image_encoder100.pth``, to ``directory``; returns the text encoder's path (what cfg.TRAIN.NET_E names)."""
    import os
    from . import model
    torch.manual_seed(seed)
    torch.save(model.RNN_ENCODER(n_words, nhidden=cfg.TEXT.EMBEDDING_DIM).state_dict(),
               os.path.join(directory, "text_encoder100.pth"))
    torch.save(model.CNN_ENCODER(cfg.TEXT.EMBEDDING_DIM).state_dict(), os.path.join(directory, "image_encoder100.pth"))
    return os.path.join(directory, "text_encoder100.pth")


def loader_box_maps(rois0, fm_rois, num_rois, num_classes: int = 80):
    """The box maps of the reference's test loader, float64 (ref: miscc/load.py:621-645 rasterises, 178-212 places
    them per slot): bbox_maps_fwd (B, BOXES_NUM, num_classes, 64, 64) with box r of its class in slot r,
    bbox_maps_bwd the slots reversed, and bbox_fmaps (B, BOXES_NUM, 16, 16) from fm_rois / 2.  A box covers
    [round(y), round(y + h)) x [round(x), round(x + w)), each edge min(round-half-even(v), size - 1)."""
    boxes, s, fs = cfg.ROI.BOXES_NUM, IMG_SIZES[0], cfg.ROI.FM_SIZE
    edge = lambda v, size: min(int(round(float(v))), size - 1)
    r0, fm = np.asarray(rois0, dtype=np.float64), np.asarray(fm_rois, dtype=np.float64)
    b = r0.shape[0]
    fwd = np.zeros((b, boxes, num_classes, s, s))
    fmaps = np.zeros((b, boxes, fs, fs))
    for i in range(b):
        for r in range(int(num_rois[i])):
            x, y, w, h = r0[i, r, :4]
            fwd[i, r, int(r0[i, r, 4]), edge(y, s):edge(y + h, s), edge(x, s):edge(x + w, s)] = 1
            x, y, w, h = fm[i, r, :4] / 2.0
            fmaps[i, r, edge(y, fs):edge(y + h, fs), edge(x, fs):edge(x + w, fs)] = 1
    fwd = torch.from_numpy(fwd)
    return fwd, fwd.flip(1).contiguous(), torch.from_numpy(fmaps)


def reference_test_batch(batch: int, seed: int = 1234, mode: int = 2, *, lens=None, full_maps: bool = True,
                         max_rois: int | None = None, n_words: int = 200, n_glove: int = 200, num_classes: int = 80,
                         fid_dims: int = 2048):
    """One batch in the format the reference's DataLoader collates from ``TestDataset.__getitem__`` (ref:
    testDataset.py:67-103): for ``mode`` (cfg.TEST.USE_GT_BOX_SEG) 0 / 1 the 17 fields (imgs, acts, captions
    (B, 18, 1), glove_captions, cap_lens UNSORTED, hmaps, bbox_maps_fwd, bbox_maps_bwd, bbox_fmaps, rois, fm_rois,
    num_rois, bt_masks, fm_bt_masks, class_ids, keys, sent_ids), for mode 2 the 14 without hmaps and masks.  Captions,
    layout, masks and images are ``reference_batch``'s; ``acts`` are float64 (B, fid_dims) activations (float32
    values, non-negative like pooled ReLU features); ``sent_ids`` index * 5 + a seeded caption index.

    The box maps are float64 (B, BOXES_NUM, num_classes, 64, 64) / (B, BOXES_NUM, 16, 16), rasterised from the box
    tables like the reference's loader (``loader_box_maps``).  ``full_maps`` False: the box maps and heat maps are
    zero-stride float64 views of their shapes instead (no memory; an intake that never reads them cannot tell)."""
    data = reference_batch(batch, seed, lens=lens, max_rois=max_rois, n_words=n_words, n_glove=n_glove,
                           num_classes=num_classes)
    imgs, caps, gcaps, lens, hmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks, class_ids, keys = data
    g = torch.Generator().manual_seed(seed + 2)
    acts = torch.randn(batch, fid_dims, generator=g).abs().double()
    sent_ids = torch.arange(batch) * cfg.TEXT.CAPTIONS_PER_IMAGE + torch.randint(0, cfg.TEXT.CAPTIONS_PER_IMAGE,
                                                                                  (batch,), generator=g)
    boxes, s, fs = cfg.ROI.BOXES_NUM, IMG_SIZES[0], cfg.ROI.FM_SIZE
    if full_maps:
        fwd, bwd, fmaps = loader_box_maps(rois[0], fm_rois, num_rois, num_classes)
    else:
        zero = torch.zeros((), dtype=torch.float64)
        fwd = bwd = zero.expand(batch, boxes, num_classes, s, s)
        fmaps = zero.expand(batch, boxes, fs, fs)
        hmaps = [zero.expand(h.shape) for h in hmaps]
    keys = [k.replace("train", "val") for k in keys]
    if mode == 2:
        return (imgs, acts, caps, gcaps, lens, fwd, bwd, fmaps, rois, fm_rois, num_rois, class_ids, keys, sent_ids)
    return (imgs, acts, caps, gcaps, lens, hmaps, fwd, bwd, fmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks,
            class_ids, keys, sent_ids)


def reference_test_dataset(n_words: int = 200, n_glove: int = 200, num_classes: int = 80, seed: int = 0):
    """An object with the attributes the reference's condGANEvaluator reads from its ``TestDataset``: those of
    ``reference_dataset``, and ``acts_dict`` None (no activation file read yet)."""
    ds = reference_dataset(n_words, n_glove, num_classes, seed)
    ds.acts_dict = None
    return ds


def reference_acts_batches(batch: int, n: int, seed: int = 1234):
    """``n`` batches as the reference's DataLoader collates them from ``TestDataset.__getitem__`` before the
    activation file exists (ref: testDataset.py:76-77): (imgs, keys), the images of ``make_inputs``."""
    out = []
    for i in range(n):
        inp = make_inputs(batch, seed + i, parity=True)
        out.append((inp["imgs"], [f"COCO_val2014_{seed + i:06d}{j:06d}" for j in range(batch)]))
    return out
