"""CPU restatement of the rows the reference's box Evaluator writes (box_generation/seq2seq/evaluator/evaluator.py:74-149)
and of the box stage's counter-based noise, composed from oracle/box_oracle.py's step order:

  records(...)     one trajectory -> the boxes.txt rows before the text round trip, their class rows, the valid-step
                   count and the number of boxes dropped for a special label
  layout_of(...)   those rows through the boxes.txt round trip, ROI_MIN_SIZE and the scales: box_oracle.layout's result
  files_text(...)  the boxes.txt text and the dev_bbox_test.txt line (None when the reference writes none)
  noise(...)       og_box_noise's Philox4x32-10 draws of one caption, in numpy (float64 normals)
"""
import numpy as np
import torch


def records(labels, samples, mean_std, label_to_class, count_stats, noise_cnt):
    """Returns (rows [(x, y, w, h)] float64, classes [row], n_valid, n_special).  coord_converter rounds the product and
    the sum separately; a box with a special label (class -1) is dropped and counted where the reference raises."""
    ms = [[float(v) for v in row] for row in mean_std]
    boxes = []
    for l, s in zip(labels, samples):
        x = float(np.float32(s[0])) * ms[0][1] + ms[0][0]                   # coord_converter
        y = float(np.float32(s[1])) * ms[1][1] + ms[1][0]
        w = float(np.float32(s[2])) * ms[2][1] + ms[2][0]
        h = w * (float(np.float32(s[3])) * ms[3][1] + ms[3][0])
        if x > 0 and y > 0 and w > 0 and h > 0:                             # validity_indices
            boxes.append((int(l), x, y, w, h))
    n_valid = len(boxes)
    boxes = boxes[:-1] if len(boxes) > 1 else []                            # drop the last kept step
    classed = [(int(label_to_class[l]), x, y, w, h) for l, x, y, w, h in boxes if int(label_to_class[l]) >= 0]
    n_special = len(boxes) - len(classed)
    rows, cls, seen = [], [], {}
    for c, x, y, w, h in classed:                                           # filter redundant labels
        if c not in seen:
            mu, sigma = float(count_stats[c][0]), float(count_stats[c][1])
            seen[c] = [max(int(mu + sigma * float(np.float32(noise_cnt[c]))), 2), 0]
        if seen[c][1] >= seen[c][0]:
            continue
        seen[c][1] += 1
        x = float(np.clip(x - w / 2.0, 1, 255))
        y = float(np.clip(y - h / 2.0, 1, 255))
        rows.append((x, y, min(w, 256.0 - x), min(h, 256.0 - y)))
        cls.append(c)
    return rows, cls, n_valid, n_special


def layout_of(rows, cls, boxes_num=10, min_size=10, imsizes=(64, 128, 256)):
    """The rows as load_gen_insanns reads them back (image_generation/miscc/load.py:653-776): rois (3, boxes_num, 6),
    fm_rois (boxes_num, 6), roi_cls (boxes_num,), num_rois -- box_oracle.layout's result."""
    rois = np.zeros((3, boxes_num, 6))
    fm = np.zeros((boxes_num, 6))
    out_cls = np.zeros(boxes_num, dtype=np.int64)
    n = 0
    for (x, y, w, h), c in zip(rows, cls):
        v = [int(float("%.2f" % q)) for q in (x, y, w, h)]                  # written '%.2f', read .astype(int)
        if v[2] < min_size and v[3] < min_size:
            continue
        if n >= boxes_num:
            break
        for k, s in enumerate(imsizes):
            rois[k, n, :4] = np.array(v, dtype=np.float64) * (s / float(imsizes[-1]))
            rois[k, n, 4] = c
        fm[n, :4] = rois[0, n, :4] / 2.0
        fm[n, 4] = c
        out_cls[n] = c
        n += 1
    return torch.from_numpy(rois), torch.from_numpy(fm), torch.from_numpy(out_cls), n


def files_text(rows, cls, class_names, key, cap_words, n_valid):
    """(boxes.txt text, dev_bbox_test.txt line or None) of one tuple, as evaluator.py:137-149 write them; class_names
    maps a class row to its category id string."""
    txt = "".join("%.2f,%.2f,%.2f,%.2f,%s,0\n" % (x, y, w, h, class_names[c]) for (x, y, w, h), c in zip(rows, cls))
    if n_valid <= 1:
        return txt, None
    line = "%s - %s - " % (key, list(cap_words))
    for (x, y, w, h), c in zip(rows, cls):
        line += "%.2f,%.2f,%.2f,%.2f,%s - " % (x, y, w, h, class_names[c])
    return txt, line + "\n"


_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))
_MASK = np.uint64(0xFFFFFFFF)


def philox(counters, key):
    """Philox4x32-10 of uint32 counters (N, 4) under key (k0, k1): (N, 4) uint32."""
    c = [np.asarray(counters, dtype=np.uint64)[:, q] for q in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W[0]) & _MASK, (k1 + _W[1]) & _MASK
        p0, p1 = _M[0] * c[0], _M[1] * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & _MASK, p1 & _MASK, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & _MASK,
             p0 & _MASK]
    return np.stack(c, 1).astype(np.uint32)


def noise(seed, i, steps, num_classes):
    """og_box_noise of caption i: noise_box (steps, 6) and noise_cnt (num_classes,), float64 (the device rounds to
    float32; the uniforms are exact)."""
    key = (seed & 0xFFFFFFFF, seed >> 32)
    hi, lo = i >> 32, i & 0xFFFFFFFF

    def draw(n, stream):
        return philox([[j, stream, lo, hi] for j in range(n)], key)
    wb, wc = draw(steps * 6, 0), draw(num_classes, 1)

    def normal(w):
        u1 = (w[:, 0].astype(np.float64) + 1.0) * 2.0 ** -32
        u2 = w[:, 1].astype(np.float64) * 2.0 ** -32
        return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
    nb = normal(wb)
    uni = (wb[:, 0] >> 8).astype(np.float64) * 2.0 ** -24
    j = np.arange(steps * 6)
    nb[j % 3 == 0] = uni[j % 3 == 0]
    return nb.reshape(steps, 6), normal(wc)
