"""Loss functions of the hot path with the reference's names and argument order
(reference: image_generation/miscc/losses.py:163-211 ``patD_loss``, 364-399 patch-D part of ``G_loss``,
533-537 ``KL_loss``).  BCE / KL values and their gradients come from the fused kernels ``og_bce`` / ``og_kl``.
"""
from __future__ import annotations

import torch

from . import ops
from .config import cfg


def _heads(net):
    net = net.module if hasattr(net, "module") else net
    return net.COND_DNET, net.UNCOND_DNET


def patD_loss(netPatD, real_imgs, fake_imgs, conditions):
    """ref: miscc/losses.py:163-211 -- two body forwards (separate BatchNorm statistics), COND head on
    (real, fake, wrong = real[:B-1] x cond[1:]), UNCOND head on (real, fake)."""
    real_features = netPatD(real_imgs)
    fake_features = netPatD(fake_imgs.detach())
    cond, uncond = _heads(netPatD)
    ul, tl = cfg.TRAIN.SMOOTH.UNCOND_LAMBDA, cfg.TRAIN.SMOOTH.TXT_LAMBDA
    batch_size = real_features.size(0)
    cond_real = cond(real_features, conditions)
    cond_fake = cond(fake_features, conditions)
    cond_wrong = cond(real_features[:(batch_size - 1)], conditions[1:batch_size])
    if uncond is not None:
        real_logits = uncond(real_features)
        fake_logits = uncond(fake_features)
        # errD = (u_real*UL + c_real*TL)/2 + (u_fake*UL + (c_fake + c_wrong)*TL)/3, folded into the weights
        return (ops.bce(real_logits, 1.0, ul / 2.0) + ops.bce(cond_real, 1.0, tl / 2.0)
                + ops.bce(fake_logits, 0.0, ul / 3.0) + ops.bce(cond_fake, 0.0, tl / 3.0)
                + ops.bce(cond_wrong, 0.0, tl / 3.0))
    return ops.bce(cond_real, 1.0, tl) + ops.bce(cond_fake, 0.0, tl / 2.0) + ops.bce(cond_wrong, 0.0, tl / 2.0)


def G_loss_pat(netsPatD, fake_imgs, sent_emb, streams=None):
    """Patch-discriminator terms of ``G_loss`` (ref: miscc/losses.py:372-399).  ``streams``: optional CUDA streams, one
    per discriminator: the three branches are independent until their losses are summed, so they may run
    concurrently (autograd replays each branch's backward on the stream of its forward)."""
    import contextlib
    ul, tl = cfg.TRAIN.SMOOTH.UNCOND_LAMBDA, cfg.TRAIN.SMOOTH.TXT_LAMBDA
    per = []
    main = torch.cuda.current_stream() if streams else None
    for i in range(len(netsPatD)):
        if streams:
            streams[i].wait_stream(main)
        with (torch.cuda.stream(streams[i]) if streams else contextlib.nullcontext()):
            features = netsPatD[i](fake_imgs[i])
            cond, uncond = _heads(netsPatD[i])
            cond_err = ops.bce(cond(features, sent_emb), 1.0, tl if uncond is not None else 1.0)
            loss = cond_err
            if uncond is not None:
                loss = loss + ops.bce(uncond(features), 1.0, ul)
            per.append(loss)
    total = None
    for i, loss in enumerate(per):
        if streams:
            main.wait_stream(streams[i])
        total = loss if total is None else total + loss
    return total, per


def KL_loss(mu, logvar):
    """ref: miscc/losses.py:533-537.  ``mu`` / ``logvar`` are the column views G_NET returns; the fused
    kernel runs on their shared row buffer."""
    base = mu._base if mu._base is not None else None
    if base is not None and logvar._base is base and base.dim() == 2:
        return ops.kl_rows(base, mu.shape[1], 1.0)
    d = mu.shape[1]
    rows = torch.zeros(mu.shape[0], ops.cpad(2 * d), device=mu.device)
    rows = torch.cat((mu, logvar, rows[:, 2 * d:]), 1)
    return ops.kl_rows(rows, d, 1.0)


def permute_seg(seg_conditions, rois, num_rois):
    """ref: miscc/utils.py:445-462 -- per sample, shuffle the segmentation channels of the classes present (host
    `random.shuffle`, drawn in the reference's order); returns the permuted maps and the indices of the samples that
    changed.  The shuffles become one (B, C) channel-permutation table, applied by ONE kernel pass
    (``og_permute_channels``) instead of a clone plus two indexed copies per sample."""
    import random
    from copy import deepcopy

    import numpy as np
    rois_np = rois.detach().cpu().numpy() if torch.is_tensor(rois) else np.asarray(rois)
    nums = num_rois.detach().cpu().numpy().tolist() if torch.is_tensor(num_rois) else list(num_rois)
    bsz, nch = seg_conditions.size(0), seg_conditions.size(1)
    perm = np.tile(np.arange(nch, dtype=np.int64), (bsz, 1))
    valid = []
    for b in range(bsz):
        if nums[b] == 0:
            continue
        classes = list(np.unique(rois_np[b, :nums[b], 4]).astype(int))
        shuffled = deepcopy(classes)
        random.shuffle(shuffled)
        if classes != shuffled:
            valid.append(b)
            perm[b, classes] = shuffled                 # new_seg[b, classes] = seg[b, shuffled]
    if not valid:
        return seg_conditions, valid                    # nothing changed (the reference returns an equal clone)
    return ops.permute_channels(seg_conditions, ops.h2d(perm, seg_conditions.device)), valid


def shpD_loss(netShpD, real_imgs, fake_imgs, seg_conditions, rois, num_rois):
    """ref: miscc/losses.py:213-251."""
    real_features = netShpD(real_imgs, seg_conditions)
    fake_features = netShpD(fake_imgs.detach(), seg_conditions)
    fake_seg, valid = permute_seg(seg_conditions, rois, num_rois)
    net = netShpD.module if hasattr(netShpD, "module") else netShpD
    err = ops.bce(net.UNCOND_DNET(real_features), 1.0, 1.0)
    fake_err = ops.bce(net.UNCOND_DNET(fake_features), 0.0, 1.0)
    if len(valid) > 0:
        idx = ops.h2d(valid, real_imgs.device, torch.int64)
        wrong = netShpD(real_imgs[idx], fake_seg[idx])
        return err + (fake_err + ops.bce(net.UNCOND_DNET(wrong), 0.0, 1.0)) / 2.0
    return err + fake_err


def feat_select(pooled_feat, raw_bt_c_codes, fm_rois, num_rois, is_large_scale=False):
    """ref: miscc/utils.py:465-499 -- keep the rois of the requested scale class.  The box filter runs on the host
    copy of ``fm_rois`` like the reference; the kept rows are compacted on the device by ONE gather per tensor
    (the reference concatenates per-sample slices).  Returns (features (R', C, h, w), classes (host int array),
    bt_c_codes (R', D)); three empty lists when nothing is kept."""
    import numpy as np
    fm = fm_rois.detach().cpu().numpy() if torch.is_tensor(fm_rois) else np.asarray(fm_rois)
    nums = num_rois.detach().cpu().numpy().tolist() if torch.is_tensor(num_rois) else list(num_rois)
    boxes, code_slots = pooled_feat.shape[1], raw_bt_c_codes.shape[1]
    flat, flat_c, classes = [], [], []
    for b in range(len(nums)):
        for r in range(int(nums[b])):
            _, _, width, height = fm[b, r, :4]
            if width < 1.25 and height < 1.25:
                continue
            big = max(width, height) >= cfg.ROI.ROI_SIZE_THRS
            if big != bool(is_large_scale):
                continue
            flat.append(b * boxes + r)
            flat_c.append(b * code_slots + r)      # the generator's bt_c_code has max(num_rois) slots, not BOXES_NUM
            classes.append(int(fm[b, r, 4]))
    if not flat:
        return [], [], []
    idx = ops.h2d(flat, pooled_feat.device, torch.int64)
    idx_c = ops.h2d(flat_c, pooled_feat.device, torch.int64)
    feats = ops.gather_rows(pooled_feat.reshape((-1,) + tuple(pooled_feat.shape[2:])), idx)
    codes = ops.gather_rows(raw_bt_c_codes.reshape(-1, raw_bt_c_codes.shape[-1]), idx_c)
    return feats, np.asarray(classes, dtype=np.int64), codes


def objD_loss(netObjD, real_imgs, fake_imgs, seg_conditions, raw_conditions, raw_bt_c_codes, fm_rois, num_rois,
              is_large_scale=False):
    """ref: miscc/losses.py:254-361 -- object discriminator loss: real / fake / mismatched-condition / permuted-shape
    terms over the rois of one scale class.  Reproduces the reference's use of ``classes`` (not ``classes2``) for the
    permuted-shape conditions (losses.py:307-311)."""
    net = netObjD.module if hasattr(netObjD, "module") else netObjD
    dev = real_imgs.device

    def lookup(cls_idx, codes):
        idx = ops.h2d([int(c) for c in cls_idx], dev, torch.int64)
        return ops.cat_rows_const(ops.gather_rows(raw_conditions.detach(), idx), codes)

    # the shape branch of the net sees the same segmentation map in the real and the fake pass: evaluate it once
    shared = {"shape_features": net.shape_features(seg_conditions)} if hasattr(net, "shape_features") else {}
    real_pooled = netObjD(real_imgs, seg_conditions, fm_rois, num_rois, **shared)
    real_features, classes, bt_c_codes = feat_select(real_pooled, raw_bt_c_codes, fm_rois, num_rois, is_large_scale)
    fake_pooled = netObjD(fake_imgs.detach(), seg_conditions, fm_rois, num_rois, **shared)
    fake_features, _, _ = feat_select(fake_pooled, raw_bt_c_codes, fm_rois, num_rois, is_large_scale)
    fake_seg, valid = permute_seg(seg_conditions, fm_rois, num_rois)
    classes2 = []
    if len(valid) > 0:
        vi = ops.h2d(valid, dev, torch.int64)
        fm_t = fm_rois if torch.is_tensor(fm_rois) else torch.as_tensor(fm_rois)
        nr_t = num_rois if torch.is_tensor(num_rois) else torch.as_tensor(num_rois)
        # index the (host or device) box tables with an index on THEIR device: no device -> host read of `valid`
        sel = lambda t: t[ops.h2d(valid, t.device, torch.int64)]
        pooled2 = netObjD(real_imgs[vi], fake_seg[vi], sel(fm_t), sel(nr_t))
        fake_features2, classes2, bt_c_codes2 = feat_select(pooled2, raw_bt_c_codes, sel(fm_t), sel(nr_t),
                                                            is_large_scale)
    n = len(classes)
    if n == 0:
        return 0
    conditions = lookup(classes, bt_c_codes)
    cond_real = ops.bce(net.COND_DNET(real_features, conditions), 1.0, 1.0)
    cond_fake = ops.bce(net.COND_DNET(fake_features, conditions), 0.0, 1.0)
    cond_wrong = None
    if n > 1:
        cond_wrong = ops.bce(net.COND_DNET(real_features[:n - 1], conditions[1:n]), 0.0, 1.0)
    cond_wrong2 = None
    if len(valid) > 0 and len(classes2) > 0:
        conditions2 = lookup(classes[:len(classes2)], bt_c_codes2)
        cond_wrong2 = ops.bce(net.COND_DNET(fake_features2, conditions2), 0.0, 1.0)
    if net.UNCOND_DNET is not None:
        err = (ops.bce(net.UNCOND_DNET(real_features), 1.0, 1.0) + cond_real) / 2.0
        tmp = ops.bce(net.UNCOND_DNET(fake_features), 0.0, 1.0) + cond_fake
        denorm = 3.0
    else:
        err = cond_real
        tmp = cond_fake
        denorm = 2.0
    if cond_wrong is not None:
        tmp = tmp + cond_wrong
    if cond_wrong2 is not None:
        tmp = tmp + cond_wrong2
        denorm += 1.0
    return err + tmp / denorm


def _class_masks(class_ids, batch_size, device):
    """ref: miscc/losses.py:27-38 -- mask[i, j] = 1 where caption j comes from the same class as sample i (j != i)."""
    if class_ids is None:
        return None
    import numpy as np
    ids = np.asarray(class_ids)
    m = (ids.reshape(-1, 1) == ids.reshape(1, -1)).astype(np.uint8)
    np.fill_diagonal(m, 0)
    return ops.h2d(m[:batch_size, :batch_size].copy(), device)


def sent_loss(cnn_code, rnn_code, labels, class_ids, batch_size, eps=1e-8, top1=True, is_training=True):
    """ref: miscc/losses.py:22-71 (DAMSM sentence matching): scaled cosine matrix between the image codes and the
    sentence codes, two cross-entropy directions.  ``rnn_code`` is a constant here (trainer.py:369 detaches it).
    Returns (loss0, loss1, accuracy) with the accuracy a device scalar (percent)."""
    if cnn_code.dim() == 3:
        cnn_code, rnn_code = cnn_code[0], rnn_code[0]
    sim = ops.cosine_matrix(cnn_code, rnn_code, eps)
    mask = _class_masks(class_ids, batch_size, cnn_code.device)
    loss0, loss1, correct = ops.ce_pair(sim, mask, labels, cfg.TRAIN.SMOOTH.GAMMA3)
    accuracy = correct * (100.0 / (batch_size * 2.0)) if top1 else sim.detach() * cfg.TRAIN.SMOOTH.GAMMA3
    return loss0, loss1, accuracy


def words_loss(img_features, words_emb, labels, cap_lens, class_ids, batch_size, top1=True, is_training=True,
               need_att_maps=True):
    """ref: miscc/losses.py:74-159 (DAMSM word-region matching).  img_features (B, nef, 17, 17) carries the gradient;
    words_emb (B, nef, T) is a constant.  All B x B (image, caption) pairs run in ONE launch (``ops.words_pairs``:
    func_attention of caption i's words against image b, cosine similarity word / attended context, Eq. (10) pooling)
    instead of the reference's per-caption Python loop; then the two cross-entropy directions over the B x B
    similarity matrix.  ``cap_lens``: int64 tensor on the device (no host synchronisation), or a host list / tensor.
    Returns (loss0, loss1, att_maps, accuracy); att_maps[i] = (1, n_i, 17, 17) like the reference when
    ``need_att_maps`` (slicing by n_i needs the lengths on the host), else the padded (B, T, 17, 17) tensor."""
    dev = img_features.device
    if torch.is_tensor(cap_lens) and cap_lens.device == dev:
        lens_dev = cap_lens.to(torch.int64).contiguous()
    else:
        lens_dev = ops.h2d([int(v) for v in cap_lens], dev, torch.int64)
    sim, attn = ops.words_pairs(img_features, words_emb.detach(), lens_dev[:batch_size], cfg.TRAIN.SMOOTH.GAMMA1,
                                cfg.TRAIN.SMOOTH.GAMMA2)                     # sim[image, caption]
    diag = attn[torch.arange(batch_size, device=dev), torch.arange(batch_size, device=dev)] if need_att_maps else None
    if need_att_maps:
        lens = cap_lens.detach().cpu().tolist() if torch.is_tensor(cap_lens) else list(cap_lens)
        att_maps = [diag[i:i + 1, :int(lens[i])].contiguous() for i in range(batch_size)]
    else:
        att_maps = None
    mask = _class_masks(class_ids, batch_size, dev)
    loss0, loss1, correct = ops.ce_pair(sim, mask, labels, cfg.TRAIN.SMOOTH.GAMMA3)
    accuracy = correct * (100.0 / (batch_size * 2.0)) if top1 else None
    return loss0, loss1, att_maps, accuracy


def _obj_g_term(netObjD, fake_img, seg, slabels_emb, raw_bt_c_codes, rois, num_rois, is_large_scale):
    """One object-discriminator term of G_loss (ref: miscc/losses.py:436-478 / 481-523); None when no roi of that
    scale class exists.  The generator's bt_c_code rows keep their gradient through the conditioning code."""
    net = netObjD.module if hasattr(netObjD, "module") else netObjD
    pooled = netObjD(fake_img, seg, rois, num_rois)
    feats, classes, codes = feat_select(pooled, raw_bt_c_codes, rois, num_rois, is_large_scale)
    if len(classes) == 0:
        return None
    idx = ops.h2d([int(c) for c in classes], fake_img.device, torch.int64)
    conditions = ops.cat_rows(ops.gather_rows(slabels_emb.detach(), idx), codes)
    err = ops.bce(net.COND_DNET(feats, conditions), 1.0, 1.0)
    if net.UNCOND_DNET is not None:
        err = err + ops.bce(net.UNCOND_DNET(feats), 1.0, 1.0)
    return err * cfg.TRAIN.SMOOTH.OBJ_LAMBDA


def G_loss(netsPatD, netsShpD, netObjSSD, netObjLSD, image_encoder, fake_imgs, seg_conditions, words_embs, sent_emb,
           slabels_emb, raw_bt_c_codes, match_labels, cap_lens, class_ids, rois, fm_rois, num_rois):
    """ref: miscc/losses.py:364-531 -- the generator's full adversarial + matching loss: per scale the patch-D terms
    (COND * TXT_LAMBDA + UNCOND * UNCOND_LAMBDA) and the shape-D term (SHP_LAMBDA); at the last scale the DAMSM
    word / sentence matching terms through ``image_encoder`` (the pretrained Inception CNN_ENCODER: a stock PyTorch
    module returning (region_features (B, nef, 17, 17), cnn_code (B, nef)); None skips the two terms); the small- and
    large-scale object-D terms (OBJ_LAMBDA).  Returns (errG_total, logs) with ``logs`` a dict of device scalars instead
    of the reference's formatted string (no per-step host synchronisation)."""
    batch_size = fake_imgs[0].size(0)
    ul, tl = cfg.TRAIN.SMOOTH.UNCOND_LAMBDA, cfg.TRAIN.SMOOTH.TXT_LAMBDA
    logs = {}
    total = None

    def add(x):
        nonlocal total
        total = x if total is None else total + x

    n_d = len(netsPatD)
    for i in range(n_d):
        features = netsPatD[i](fake_imgs[i])
        cond, uncond = _heads(netsPatD[i])
        pat = ops.bce(cond(features, sent_emb), 1.0, tl if uncond is not None else 1.0)
        if uncond is not None:
            pat = pat + ops.bce(uncond(features), 1.0, ul)
        add(pat)
        logs[f"pat_g_loss{i}"] = pat.detach()
        shp_net = netsShpD[i].module if hasattr(netsShpD[i], "module") else netsShpD[i]
        shp = ops.bce(shp_net.UNCOND_DNET(netsShpD[i](fake_imgs[i], seg_conditions[i])), 1.0, cfg.TRAIN.SMOOTH.SHP_LAMBDA)
        add(shp)
        logs[f"shp_g_loss{i}"] = shp.detach()
        if i == n_d - 1 and image_encoder is not None:
            region_features, cnn_code = image_encoder(fake_imgs[i])
            w0, w1, _, _ = words_loss(region_features, words_embs, match_labels, cap_lens, class_ids, batch_size,
                                      need_att_maps=False)
            s0, s1, _ = sent_loss(cnn_code, sent_emb, match_labels, class_ids, batch_size)
            w_loss = (w0 + w1) * cfg.TRAIN.SMOOTH.DAMSM_LAMBDA
            s_loss = (s0 + s1) * cfg.TRAIN.SMOOTH.DAMSM_LAMBDA
            add(w_loss + s_loss)
            logs["w_loss"], logs["s_loss"] = w_loss.detach(), s_loss.detach()
    ss = _obj_g_term(netObjSSD, fake_imgs[-1], seg_conditions[-1], slabels_emb, raw_bt_c_codes, rois, num_rois, False)
    if ss is not None:
        add(ss)
        logs["objss_g_loss"] = ss.detach()
    ls = _obj_g_term(netObjLSD, fake_imgs[-1], seg_conditions[-1], slabels_emb, raw_bt_c_codes, fm_rois, num_rois, True)
    if ls is not None:
        add(ls)
        logs["objls_g_loss"] = ls.detach()
    return total, logs


class RPrecision:
    """R-precision of generated images (ref: evaluator.py:370-411, cfg.TEST.RP_POOL_SIZE = 100), restated with the
    reference's pooling:

      * batches of (region_features, cnn_code, words_embs, sent_emb, cap_lens) are appended until the pooled count
        reaches ``pool_size``;
      * the batch that arrives when the pool is full scores the pool and is itself NOT added (the reference drops it;
        reproduced on purpose, so that the numbers compare);
      * the pool's sets are cut to ``pool_size`` and its words_embs zero-padded to the longest of its captions;
      * words_loss / sent_loss run with labels 0..pool_size-1 and the pool's class ids, like the reference: its losses
        mask same-class pairs whatever ``is_training`` is (miscc/losses.py:27-54, 88-140); on COCO the class ids are
        distinct (load.py:429-435), so the mask is empty there;
      * ``result()`` gives (mean, std) of the word and of the sentence accuracy (percent) over the scored pools."""

    def __init__(self, pool_size=100):
        self.pool_size = pool_size
        self.w_accuracy, self.s_accuracy = [], []
        self._reset()

    def _reset(self):
        self.count = 0
        self.sets = {"region_features": [], "cnn_code": [], "words_embs": [], "sent_emb": [], "cap_lens": []}
        self.class_ids = []

    def add(self, region_features, cnn_code, words_embs, sent_emb, cap_lens, class_ids=None):
        """One batch; ``class_ids``: its class ids (a host sequence; None: every sample its own class)."""
        if self.count >= self.pool_size:
            self._score()
            self._reset()
            return
        dev = cnn_code.device
        lens = cap_lens.to(dev, torch.int64) if torch.is_tensor(cap_lens) else ops.h2d([int(v) for v in cap_lens], dev,
                                                                                      torch.int64)
        for k, v in (("region_features", region_features), ("cnn_code", cnn_code), ("words_embs", words_embs),
                     ("sent_emb", sent_emb), ("cap_lens", lens)):
            self.sets[k].append(v.detach())
        import numpy as np
        b = cnn_code.shape[0]
        self.class_ids.append(np.asarray(class_ids).reshape(-1) if class_ids is not None
                              else -1 - np.arange(self.count, self.count + b))     # distinct: no pair masked
        self.count += b

    def _pool(self):
        """The pooled sets, cut to pool_size, words_embs padded to the pool's longest caption."""
        p = self.pool_size
        cat = {k: torch.cat(v, 0)[:p] for k, v in self.sets.items() if k != "words_embs"}
        max_len = int(cat["cap_lens"].max())
        we = self.sets["words_embs"]
        words = torch.zeros((self.count, we[0].shape[1], max(max_len, *[w.shape[2] for w in we])),
                            device=we[0].device, dtype=torch.float32)
        acc = 0
        for w in we:
            words[acc:acc + w.shape[0], :, :w.shape[2]] = w
            acc += w.shape[0]
        cat["words_embs"] = words[:p, :, :max_len].contiguous()
        import numpy as np
        cat["class_ids"] = np.concatenate(self.class_ids, 0)[:p]
        return cat

    def _score(self):
        s = self._pool()
        p = self.pool_size
        labels = torch.arange(p, device=s["cnn_code"].device)
        _, _, _, w_acc = words_loss(s["region_features"], s["words_embs"], labels, s["cap_lens"], s["class_ids"], p,
                                    is_training=False, need_att_maps=False)
        _, _, s_acc = sent_loss(s["cnn_code"], s["sent_emb"], labels, s["class_ids"], p, is_training=False)
        self.w_accuracy.append(float(w_acc))
        self.s_accuracy.append(float(s_acc))

    def result(self):
        import numpy as np
        w, s = np.asarray(self.w_accuracy), np.asarray(self.s_accuracy)
        return float(w.mean()), float(w.std()), float(s.mean()), float(s.std())


def _split_parts(p, num_splits):
    n = p.shape[0]
    return [p[i * n // num_splits:(i + 1) * n // num_splits] for i in range(num_splits)]


def inception_score(p, num_splits):
    """(mean, std) over ``num_splits`` contiguous splits of exp(E_x KL(p(y|x) || p(y))) on the float32 predictions p
    (N, 1000), in numpy with the reference's arithmetic (utils.py:417-428).  A probability of exactly 0 gives nan,
    as it does there."""
    import numpy as np
    scores = []
    for part in _split_parts(p, num_splits):
        kl = part * (np.log(part) - np.log(np.expand_dims(np.mean(part, 0), 0)))
        scores.append(np.exp(np.mean(np.sum(kl, 1))))
    return np.mean(scores), np.std(scores)


def negative_log_posterior(p, num_splits):
    """(mean, std) over the splits of the mean of -log max_y p(y|x) (utils.py:431-441)."""
    import numpy as np
    scores = [np.mean(-1. * np.log(np.max(part, 1))) for part in _split_parts(p, num_splits)]
    return np.mean(scores), np.std(scores)


class InceptionScore:
    """The evaluator's Inception score and confidence (ref: evaluator.py:421-450) over the INCEPTION_V3 predictions
    of every added batch.  ``add`` keeps the predictions on the device; ``result()`` reads them once and returns
    (mean, std, mean_conf, std_conf).  The evaluator uses min(10, batch_size) splits.  Each data-parallel rank
    scores the predictions it was given."""

    def __init__(self, num_splits=10):
        self.num_splits = num_splits
        self.predictions = []

    def add(self, predictions):
        self.predictions.append(predictions.detach())

    def result(self):
        p = torch.cat(self.predictions, 0).float().cpu().numpy()
        mean, std = inception_score(p, self.num_splits)
        mean_conf, std_conf = negative_log_posterior(p, self.num_splits)
        return float(mean), float(std), float(mean_conf), float(std_conf)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """d^2 = |mu1 - mu2|^2 + Tr(sigma1 + sigma2 - 2 sqrt(sigma1 sigma2)) in float64 with scipy's sqrtm (utils.py:
    660-714): when the square root is not finite it is retried with eps added to both diagonals, and an imaginary
    part larger than 1e-3 on its diagonal raises ValueError.  (sqrtm is called without ``disp``, which scipy 1.18
    removed; the value is the same.)"""
    import numpy as np
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    if mu1.shape != mu2.shape or sigma1.shape != sigma2.shape:
        raise ValueError("the two sets of statistics have different dimensions")
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean)


class _Moments:
    """Streaming fp64 mean and covariance of (n, d) fp32 rows on the device (og_moments_f64): O(d^2) memory however
    many rows are added."""

    def __init__(self, dims):
        self.dims, self.n, self.k = dims, 0, None

    def add(self, x):
        if x.dim() != 2 or x.shape[1] != self.dims:
            raise ValueError(f"activations must be (N, {self.dims}), got {tuple(x.shape)}")
        if self.k is None:
            d = self.dims
            self.k, self.s1 = (torch.empty(d, device=x.device, dtype=torch.float64) for _ in range(2))
            self.s2 = torch.empty((d, d), device=x.device, dtype=torch.float64)
        ops.moments_f64(x, self.k, self.s1, self.s2, self.n == 0)
        self.n += x.shape[0]

    def symmetric_s2(self):
        """s2 with both triangles filled (og_moments_f64 writes the 32-wide tiles on or above the diagonal)."""
        t = torch.arange(self.dims, device=self.s2.device) // 32
        return torch.where(t[:, None] <= t[None, :], self.s2, self.s2.T)

    @classmethod
    def from_sums(cls, n, k, s1, s2):
        """Moments of ``n`` rows from their float64 shifted sums (s2 symmetric or upper-tiled)."""
        m = cls(k.shape[0])
        m.n = int(n)
        if m.n > 0:
            m.k, m.s1, m.s2 = k, s1, s2
        return m

    def merge(self, others):
        """These moments combined with ``others`` (_Moments of other row sets, e.g. the other data-parallel ranks'),
        in float64 torch ops: every s2 is symmetrised, every set of sums is re-centred on this one's shift k with
        delta = k_j - k (S1 += n_j delta, S2 += S1_j delta^T + delta S1_j^T + n_j delta delta^T), and the re-centred
        sums are added.  Sets without rows are skipped.  Returns a new _Moments."""
        parts = [m for m in (self, *others) if m.n > 0]
        if not parts:
            return _Moments(self.dims)
        k = parts[0].k
        s1 = torch.zeros_like(parts[0].s1)
        s2 = torch.zeros_like(parts[0].s2)
        n = 0
        for m in parts:
            d = m.k.to(k.device) - k
            m1, m2 = m.s1.to(k.device), m.symmetric_s2().to(k.device)
            s1 += m1 + m.n * d
            s2 += m2 + torch.outer(m1, d) + torch.outer(d, m1) + m.n * torch.outer(d, d)
            n += m.n
        return _Moments.from_sums(n, k, s1, s2)

    def statistics(self):
        """(mu (d,), sigma (d, d)) float64; sigma as np.cov(rowvar=False), with n - 1."""
        import numpy as np
        if self.n < 2:
            raise ValueError("the covariance needs at least two samples")
        k, s1, s2 = (t.cpu().numpy() for t in (self.k, self.s1, self.s2))
        t = np.arange(self.dims) // 32                 # og_moments_f64 writes the tiles on or above the diagonal
        s2 = np.where(t[:, None] <= t[None, :], s2, s2.T)
        m = s1 / self.n
        return k + m, (s2 - np.outer(s1, m)) / (self.n - 1)


class FrechetDistance:
    """The evaluator's FID (ref: evaluator.py:429-457) from streamed activation moments.  ``add(fake_acts,
    real_acts)`` takes (B, dims) activations of generated and of real images (INCEPTION_V3_FID.activations, or the
    reference's dump_fid_acts arrays as tensors); either may be None.  ``statistics()`` returns ((mu, sigma) of the
    real set, (mu, sigma) of the generated set) in float64; ``result()`` the distance between them."""

    def __init__(self, dims=2048):
        self.dims = dims
        self.fake, self.real = _Moments(dims), _Moments(dims)

    def add(self, fake_acts, real_acts=None):
        if fake_acts is not None:
            self.fake.add(fake_acts)
        if real_acts is not None:
            if not torch.is_tensor(real_acts):
                import numpy as np
                real_acts = torch.from_numpy(np.asarray(real_acts, dtype=np.float32))
            self.real.add(real_acts.to(self.fake.k.device if self.fake.k is not None else "cuda"))

    def statistics(self):
        return self.real.statistics(), self.fake.statistics()

    def result(self):
        (mu1, sigma1), (mu2, sigma2) = self.statistics()
        return float(frechet_distance(mu1, sigma1, mu2, sigma2))
