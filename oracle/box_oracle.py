"""CPU restatement (plain torch / Python on the CPU) of the box generator's inference path and of the evaluator's
post-processing of its samples: the PreEncoderRNN final state, the DecoderRNN step with explicit noise (free-running)
and teacher-forced on a given trajectory, and the samples -> boxes.txt -> load_gen_insanns layout.  Paths are under
box_generation/ of the original project unless they name image_generation/.  The tests pin it to the reference's own
modules (tests/golden/reference/box_*.npz) and the CUDA path to it.
"""
import math

import numpy as np
import torch

from oracle import text_oracle as T

SQRT_TEMP = np.float32(math.sqrt(0.4))      # sigma *= np.sqrt(temperature) on a float32 tensor (DecoderRNN.py:404-405)


def encoder_state(sd, captions, cap_lens):
    """PreEncoderRNN.forward (PreEncoderRNN.py:59-99) in eval mode, then _cat_directions (DecoderRNN.py:311-317):
    h, c (B, 256) = [forward state after the last token, backward state after token 0]; each caption runs its own
    cap_lens[b] tokens from a zero state."""
    emb = sd["encoder.weight"][captions]
    hid = sd["rnn.weight_hh_l0"].shape[1]
    b = captions.shape[0]
    hs, cs = torch.zeros(b, 2 * hid), torch.zeros(b, 2 * hid)
    for d, sfx in enumerate(("", "_reverse")):
        w = [sd[f"rnn.{n}_l0{sfx}"] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        for i in range(b):
            n = int(cap_lens[i])
            h, c = torch.zeros(hid), torch.zeros(hid)
            for t in (range(n - 1, -1, -1) if d else range(n)):
                h, c = T.lstm_step(emb[i, t], h, c, *w)
            hs[i, d * hid:(d + 1) * hid], cs[i, d * hid:(d + 1) * hid] = h, c
    return hs, cs


def gmm_params(raw):
    """get_gmm_params (DecoderRNN.py:373-384): raw (30,) -> (30,) = pi (softmax), mu_x, mu_y, sigma_x (exp), sigma_y
    (exp), rho (tanh), 5 each."""
    pi, mx, my, sx, sy, rho = raw.split(5)
    return torch.cat([torch.softmax(pi, 0), mx, my, torch.exp(sx), torch.exp(sy), torch.tanh(rho)])


def component(pi, u):
    """sample_next_state's component (DecoderRNN.py:352-362): adjust_temp in float32, then np.random.choice's rule
    for the uniform u -- searchsorted(cumsum(p) / sum, u, side='right'), clamped to K - 1.  Returns (component, the
    distance of u from the nearest cdf boundary)."""
    q = np.log(pi.numpy().astype(np.float32)) / np.float32(0.4)
    q -= q.max()
    q = np.exp(q)
    q /= q.sum()
    cdf = q.astype(np.float64).cumsum()
    cdf /= cdf[-1]
    k = min(int(np.searchsorted(cdf, u, side="right")), len(cdf) - 1)
    return k, float(np.min(np.abs(cdf[:-1] - u))) if len(cdf) > 1 else 1.0


def bivariate(par, k, n1, n2):
    """The temperature-scaled bivariate normal of component k from standard normals n1, n2 (a Cholesky factor):
    x = mu_x + s_x n1, y = mu_y + s_y (rho n1 + sqrt(1 - rho^2) n2), s = sigma sqrt(0.4), in float32."""
    f = np.float32
    mx, my, sx, sy, rho = (f(par[i * 5 + k]) for i in range(1, 6))
    sx, sy = sx * SQRT_TEMP, sy * SQRT_TEMP
    return f(mx + sx * f(n1)), f(my + sy * (rho * f(n1) + np.sqrt(f(1) - rho * rho) * f(n2)))


def step(sd, label, inp, h, c):
    """One forward_step up to the label distribution (DecoderRNN.py:88-129): the LSTM input cat(xy_embedding([x, y]),
    wh_embedding([w, r]), l_embedding[label]), one LSTM step, p = softmax(l_out(h)).clamp(1e-5, 1)."""
    x = torch.cat([sd["xy_embedding.weight"] @ inp[:2] + sd["xy_embedding.bias"],
                   sd["wh_embedding.weight"] @ inp[2:] + sd["wh_embedding.bias"], sd["l_embedding.weight"][label]])
    h, c = T.lstm_step(x, h, c, sd["rnn.weight_ih_l0"], sd["rnn.weight_hh_l0"], sd["rnn.bias_ih_l0"],
                       sd["rnn.bias_hh_l0"])
    p = torch.softmax(sd["l_out.weight"] @ h + sd["l_out.bias"], 0).clamp(1e-5, 1)
    return p, h, c


def xy_head(sd, h, p):
    return gmm_params(sd["xy_out.weight"] @ torch.cat([h, p]) + sd["xy_out.bias"])


def wh_head(sd, h, p, x_new, y_in):
    """The wh head over cat(h, p, next_xy_embedding([x_new, y_in])): the newly sampled x with this step's input y
    (DecoderRNN.py:166-171)."""
    nxy = sd["next_xy_embedding.weight"] @ torch.stack([x_new, y_in]) + sd["next_xy_embedding.bias"]
    return gmm_params(sd["wh_out.weight"] @ torch.cat([h, p, nxy]) + sd["wh_out.bias"])


def _start(means):
    return torch.tensor([float(m) for m in means], dtype=torch.float32)   # the raw means (DecoderRNN.py:261-265)


def decode(sd, h0, c0, noise, steps, sos, eos, means):
    """The inference loop (DecoderRNN.py:260-292) for one sample with explicit noise (steps, 6).  Returns labels,
    samples (n, 4) float32, and per step p, the xy / wh parameters, and the label / component margins: the gap between
    the two largest p, and each uniform's distance to the nearest cdf boundary."""
    h, c, lab, inp = h0.clone(), c0.clone(), sos, _start(means)
    out = dict(labels=[], samples=[], p=[], xy=[], wh=[], margin=[])
    for t in range(steps):
        p, h, c = step(sd, lab, inp, h, c)
        top = torch.topk(p, 2).values
        lab = int(torch.argmax(p))                                          # the first index of the max
        xy = xy_head(sd, h, p)
        kx, mx = component(xy[:5], float(noise[t, 0]))
        x, y = bivariate(xy, kx, noise[t, 1], noise[t, 2])
        wh = wh_head(sd, h, p, torch.tensor(x), inp[1])
        kw, mw = component(wh[:5], float(noise[t, 3]))
        w, r = bivariate(wh, kw, noise[t, 4], noise[t, 5])
        inp = torch.tensor([x, y, w, r], dtype=torch.float32)
        for k, v in (("labels", lab), ("samples", inp), ("p", p), ("xy", xy), ("wh", wh),
                     ("margin", (float(top[0] - top[1]), mx, mw))):
            out[k].append(v)
        if lab == eos:
            break
    return out


def teacher_forced(sd, h0, c0, labels, samples, sos, means):
    """Every step's p and xy / wh parameters when the decoder is fed the given trajectory (labels (n,), samples (n, 4)):
    step t reads label t-1 and sample t-1 (the start token and the raw means at t = 0)."""
    h, c, lab, inp = h0.clone(), c0.clone(), sos, _start(means)
    ps, xys, whs = [], [], []
    for t in range(len(labels)):
        p, h, c = step(sd, lab, inp, h, c)
        s = torch.as_tensor(samples[t], dtype=torch.float32)
        ps.append(p)
        xys.append(xy_head(sd, h, p))
        whs.append(wh_head(sd, h, p, s[0], inp[1]))
        lab, inp = int(labels[t]), s
    return torch.stack(ps), torch.stack(xys), torch.stack(whs)


def layout(labels, samples, mean_std, label_to_class, count_stats, noise_cnt, boxes_num=10, min_size=10,
           imsizes=(64, 128, 256)):
    """One sample's trajectory (labels (n,), samples (n, 4)) to the loader's layout: Evaluator.evaluate
    (evaluator.py:74-139), the boxes.txt round trip and load_gen_insanns (image_generation/miscc/load.py:653-776).  A
    box with a special label (class -1) is dropped where the reference raises.  noise_cnt (C,) standard normals give the
    per-class thresholds.  Returns rois (3, boxes_num, 6), fm_rois (boxes_num, 6), roi_cls (boxes_num,), num_rois."""
    ms = [[float(v) for v in row] for row in mean_std]
    boxes = []
    for l, s in zip(labels, samples):
        x = float(np.float32(s[0])) * ms[0][1] + ms[0][0]                   # coord_converter
        y = float(np.float32(s[1])) * ms[1][1] + ms[1][0]
        w = float(np.float32(s[2])) * ms[2][1] + ms[2][0]
        h = w * (float(np.float32(s[3])) * ms[3][1] + ms[3][0])
        if x > 0 and y > 0 and w > 0 and h > 0:                             # validity_indices
            boxes.append((int(l), x, y, w, h))
    boxes = boxes[:-1] if len(boxes) > 1 else []                            # drop the last kept step
    boxes = [(int(label_to_class[l]), x, y, w, h) for l, x, y, w, h in boxes if int(label_to_class[l]) >= 0]
    kept, seen = [], {}
    for c, x, y, w, h in boxes:                                             # filter redundant labels
        if c not in seen:
            mu, sigma = float(count_stats[c][0]), float(count_stats[c][1])
            seen[c] = [max(int(mu + sigma * float(np.float32(noise_cnt[c]))), 2), 0]
        if seen[c][1] < seen[c][0]:
            seen[c][1] += 1
            kept.append((c, x, y, w, h))
    rois = np.zeros((3, boxes_num, 6))
    fm = np.zeros((boxes_num, 6))
    cls = np.zeros(boxes_num, dtype=np.int64)
    n = 0
    for c, x, y, w, h in kept:
        x = float(np.clip(x - w / 2.0, 1, 255))
        y = float(np.clip(y - h / 2.0, 1, 255))
        w, h = min(w, 256.0 - x), min(h, 256.0 - y)
        v = [int(float("%.2f" % q)) for q in (x, y, w, h)]                  # written '%.2f', read .astype(int)
        if v[2] < min_size and v[3] < min_size:
            continue
        for k, s in enumerate(imsizes):
            rois[k, n, :4] = np.array(v, dtype=np.float64) * (s / float(imsizes[-1]))
            rois[k, n, 4] = c
        fm[n, :4] = rois[0, n, :4] / 2.0
        fm[n, 4] = c
        cls[n] = c
        n += 1
    return torch.from_numpy(rois), torch.from_numpy(fm), torch.from_numpy(cls), n
