"""GPU tests of writing the box layout files: og_box_records against the rows of the restatement
(tests/box_files_oracle.py) bit for bit, og_box_noise against its numpy restatement, the written files read back by
load_gen_insanns' rules against og_box_layout, boxgen.Evaluator end to end against the oracle composition, its
independence of the chunk size, and a 5,000-caption run."""
import os
import types

import numpy as np
import pytest
import torch

import box_files_oracle as F
from objgan_b200 import boxgen, ops
from oracle import box_oracle as O
from test_box_gen import (CAT_IDS, COUNT_STATS, EDGE_TRAJ, EOS, L2I, LABEL_TO_CLASS, LAYOUT_TRAJ, MEAN_STD,
                          MEAN_STD_EDGE, MEAN_STD_FULL, MEAN_STD_ID, SOS, dec_sd, hand_cases, layout_noise_cnt)
from test_gpu_box import _check_decode, _dec, _pad, _pre
from test_text_encoder import NTOK, captions_for, enc_sd

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = [str(c) for c in CAT_IDS]
I2W = {i: w for w, i in L2I.items()}
W2I = {f"w{i}": i for i in range(1, NTOK)}
BIAS = 0.0                 # added to l_out.bias[<eos>] (the label is the argmax: a bias of 0.3 ends every sample at once)


def _records_vs_oracle(trajs, mean_std, cs, ncnt):
    labels, samples, steps = _pad(trajs)
    S = labels.shape[1]
    rows, cls, n_rows, n_valid, n_special = ops.box_records(
        labels.to(DEV), samples.to(DEV), steps.to(DEV), torch.tensor(mean_std, dtype=torch.float64).to(DEV),
        LABEL_TO_CLASS.to(DEV), cs.to(DEV), ncnt.to(DEV))
    rows, cls = rows.cpu(), cls.cpu()
    for b, (lab, smp) in enumerate(trajs):
        r, c, nv, ns = F.records(torch.as_tensor(lab), torch.as_tensor(smp, dtype=torch.float32), mean_std,
                                 LABEL_TO_CLASS, cs, ncnt[b])
        n = len(r)
        assert (int(n_rows[b]), int(n_valid[b]), int(n_special[b])) == (n, nv, ns), b
        assert rows[b, :n].tolist() == [list(v) for v in r] and cls[b, :n].tolist() == c, b       # bitwise
        assert rows[b, n:].abs().sum() == 0 and cls[b, n:].abs().sum() == 0 and rows.shape[1] == S
    return rows, cls, n_rows.cpu()


def test_box_records_hand_worked_bitwise():
    cases = list(hand_cases().values())
    _, _, n_rows = _records_vs_oracle([(c[0], c[1]) for c in cases], MEAN_STD_ID, cases[0][3],
                                      torch.stack([c[2] for c in cases]))
    assert int(n_rows.max()) >= 4


def test_box_records_reference_trajectories_bitwise():
    trajs = [([t[0] for t in tr], [t[1:] for t in tr]) for tr in LAYOUT_TRAJ]
    _records_vs_oracle(trajs, MEAN_STD, COUNT_STATS, layout_noise_cnt())


def test_box_records_txt_boundary_bitwise():
    _records_vs_oracle([EDGE_TRAJ, EDGE_TRAJ], MEAN_STD_EDGE, COUNT_STATS, torch.zeros(2, 80))


def _decoder_trajs(B, seed, ms):
    bg = boxgen.BoxGenerator(_pre(), _dec(BIAS), ms, COUNT_STATS, LABEL_TO_CLASS)
    lens = torch.randint(1, 31, (B,), generator=torch.Generator().manual_seed(seed))
    caps, _ = captions_for(lens, 30, NTOK, seed + 1)
    nb, nc = ops.box_noise(seed, 0, B, 10, 80, DEV)
    out = bg.sample(caps.to(DEV), lens.to(DEV), 30, nb, nc)
    return out, nc


def test_box_records_decoder_samples_bitwise():
    out, nc = _decoder_trajs(65, 12, MEAN_STD_FULL)
    trajs = [(out["labels"][b, :int(out["steps"][b])].cpu(), out["samples"][b, :int(out["steps"][b])].cpu())
             for b in range(65)]
    _, _, n_rows = _records_vs_oracle(trajs, MEAN_STD_FULL, COUNT_STATS, nc.cpu())
    assert int(n_rows.max()) >= 2


def _parse_boxes_txt(text, boxes_num=10, min_size=10, imsizes=(64, 128, 256)):
    """load_gen_insanns' reading of a boxes.txt (image_generation/miscc/load.py:653-776): int of each value, the
    ROI_MIN_SIZE filter, the three scales."""
    rois = np.zeros((3, boxes_num, 6))
    n = 0
    for line in text.splitlines():
        f = line.split(",")
        v = [int(float(q)) for q in f[:4]]
        c = NAMES.index(f[4])
        if (v[2] < min_size and v[3] < min_size) or n >= boxes_num:
            continue
        for k, s in enumerate(imsizes):
            rois[k, n, :4] = np.array(v, dtype=np.float64) * (s / float(imsizes[-1]))
            rois[k, n, 4] = c
        n += 1
    return rois, n


@pytest.mark.parametrize("ms", ["integer", "full_mantissa"])
def test_written_rows_read_back_equal_layout(ms):
    """The two device paths agree: og_box_records' rows written as boxes.txt and read back by the loader's rules are
    og_box_layout's tables, bit for bit, on the same trajectories and noise_cnt."""
    mean_std = MEAN_STD if ms == "integer" else MEAN_STD_FULL
    out, nc = _decoder_trajs(130, 31, mean_std)
    args = (out["labels"], out["samples"], out["steps"], torch.tensor(mean_std, dtype=torch.float64, device=DEV),
            LABEL_TO_CLASS.to(DEV), COUNT_STATS.to(DEV), nc)
    rows, cls, n_rows, _, _ = (t.cpu() for t in ops.box_records(*args))
    rois, fm, roi_cls, num = ops.boxes_to_layout(*args)
    for b in range(130):
        n = int(n_rows[b])
        text = boxgen.box_rows_text(list(zip(rows[b, :n].tolist(), cls[b, :n].tolist())), NAMES)
        want, k = _parse_boxes_txt(text)
        assert k == int(num[b]), b
        for s in range(3):
            assert np.array_equal(rois[s][b].cpu().numpy(), want[s]), (b, s)
    assert int(num.max()) >= 2


def test_box_noise_matches_restatement_and_is_per_caption():
    nb, nc = ops.box_noise(77, 1000, 64, 10, 80, DEV)
    for q in (0, 1, 33, 63):
        wb, wc = F.noise(77, 1000 + q, 10, 80)
        got = nb[q].cpu().double()
        assert torch.equal(got[:, 0::3], torch.from_numpy(wb[:, 0::3]))                    # uniforms exact
        torch.testing.assert_close(got, torch.from_numpy(wb), atol=2e-6, rtol=1e-6)
        torch.testing.assert_close(nc[q].cpu().double(), torch.from_numpy(wc), atol=2e-6, rtol=1e-6)
    for first, b in ((1000, 1), (1033, 7), (990, 200)):                  # any chunk gives a caption the same draws
        ob, oc = ops.box_noise(77, first, b, 10, 80, DEV)
        lo, hi = max(first, 1000), min(first + b, 1064)
        assert torch.equal(ob[lo - first:hi - first], nb[lo - 1000:hi - 1000])
        assert torch.equal(oc[lo - first:hi - first], nc[lo - 1000:hi - 1000])
    assert not torch.equal(ops.box_noise(78, 1000, 1, 10, 80, DEV)[0][0], nb[0])
    u = nb[:, :, 0::3]
    assert float(u.min()) >= 0.0 and float(u.max()) < 1.0
    z = torch.cat([nb[:, :, [1, 2, 4, 5]].flatten(), nc.flatten()])
    assert abs(float(z.mean())) < 0.1 and abs(float(z.std()) - 1.0) < 0.1


# ---------------------------------------------------------------------------------------------------------------------
# boxgen.Evaluator end to end
# ---------------------------------------------------------------------------------------------------------------------
def _evaluator(root, output_opt=0, **kw):
    gd = {c: (float(COUNT_STATS[i, 0]), float(COUNT_STATS[i, 1])) for i, c in enumerate(CAT_IDS)}
    return boxgen.Evaluator(1, 10, str(root), types.SimpleNamespace(word2index=W2I, index2word={i: w for w, i in
                                                                                                   W2I.items()}),
                            types.SimpleNamespace(word2index=L2I, index2word=I2W), *[tuple(r) for r in MEAN_STD], gd,
                            str(root) + "/gen_masks/", output_opt, device=DEV, **kw)


def synthetic_split(n_keys=7, per_key=5, max_len=70, seed=5):
    """n_keys keys with per_key captions each, then key 0 repeated with per_key more; caption lengths 1 .. max_len."""
    keys = [f"{400000 + k}" for k in range(n_keys) for _ in range(per_key)] + ["400000"] * per_key
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, max_len + 1, (len(keys),), generator=g)
    lens[0], lens[1] = 1, max_len
    data = [[[f"w{int(t)}" for t in torch.randint(1, NTOK, (int(n),), generator=g)], "", "", "", "", ""]
            for n in lens]
    return data, keys


def _tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def test_evaluator_end_to_end_vs_oracle(tmp_path):
    data, keys = synthetic_split()
    ev = _evaluator(tmp_path, chunk=16, seed=3)
    ev.evaluate(_pre(), _dec(BIAS), data, keys)
    tree = _tree(tmp_path / "gen_masks")
    n = len(keys)
    assert len(tree) == n and sorted({k.split("/")[0] for k in tree}) == sorted(set(keys))
    jidx = boxgen.caption_indices(keys)
    assert sum(1 for k in tree if k.startswith("400000/")) == 10
    # the oracle composition: encoder state -> free-running decoder on the same noise -> rows -> text.  The device
    # trajectories are recomputed chunk by chunk as evaluate() ran them
    seqs = boxgen.caption_sequences(data, keys, W2I)
    width = max(len(q) for q in seqs)
    lens = torch.tensor([len(q) for q in seqs])
    caps = torch.zeros(n, width, dtype=torch.int64)
    for i, q in enumerate(seqs):
        caps[i, :len(q)] = torch.tensor(q)
    enc, dec = _pre(), _dec(BIAS)
    parts = []
    for lo in range(0, n, 16):
        hi = min(lo + 16, n)
        w = int(lens[lo:hi].max())
        _, hc, cc = enc.encode_state(caps[lo:hi, :w].contiguous().to(DEV), lens[lo:hi].to(DEV), w)
        nbc, ncc = ops.box_noise(3, lo, hi - lo, 10, 80, DEV)
        parts.append((hc, cc, nbc, ncc, *dec.sample_state(hc, cc, nbc, 10, debug=True)))
    h, c, nb, nc, labels, samples, steps, dbg = (torch.cat(t) for t in zip(*parts))
    h0, c0 = O.encoder_state(enc_sd(), caps, lens)
    torch.testing.assert_close(h.cpu(), h0, atol=1e-5, rtol=1e-5)
    diverged = _check_decode(dec_sd(BIAS), h.cpu(), c.cpu(), nb.cpu(), 10, labels, samples, steps, dbg)
    print(f"{diverged} of {n} samples took a different discrete choice at an oracle margin below the EPS rule")
    exact = 0
    for i in range(n):
        st = int(steps[i])
        ref = O.decode(dec_sd(BIAS), h[i].cpu(), c[i].cpu(), nb[i].cpu(), 10, SOS, EOS, dec_means())
        r, cl, nv, _ = F.records(torch.as_tensor(ref["labels"]), torch.stack(ref["samples"]), MEAN_STD, LABEL_TO_CLASS,
                                 COUNT_STATS, nc[i].cpu())
        want = F.files_text(r, cl, NAMES, keys[i], [], nv)[0]
        got = tree[f"{keys[i]}/{jidx[i]}/boxes.txt"].decode()
        exact += got == want
        if got != want:
            # the oracle's fp32 decoder sums in another order: a value may round to the neighbouring hundredth
            assert ref["labels"] == labels[i, :st].tolist(), i
            gl, wl = got.splitlines(), want.splitlines()
            assert len(gl) == len(wl), i
            for a, b in zip(gl, wl):
                fa, fb = a.split(","), b.split(",")
                assert fa[4:] == fb[4:] and all(abs(float(x) - float(y)) <= 0.0101 for x, y in zip(fa[:4], fb[:4])), \
                    (i, a, b)
        # and the file is exactly the rows of the device's own trajectory
        r, cl, nv, _ = F.records(labels[i, :st].cpu(), samples[i, :st].cpu(), MEAN_STD, LABEL_TO_CLASS, COUNT_STATS,
                                 nc[i].cpu())
        assert got == F.files_text(r, cl, NAMES, keys[i], [], nv)[0], i
    print(f"{exact} of {n} files equal the oracle composition's text byte for byte; the others differ by one "
          f"hundredth in a value")
    assert exact >= n // 2
    assert sum(v.count(b"\n") for v in tree.values()) >= n


def dec_means():
    from test_box_gen import MEANS
    return MEANS


def test_evaluator_chunk_independent(tmp_path):
    data, keys = synthetic_split()
    trees, lines = [], []
    for chunk in (1, 7, 256):
        root = tmp_path / f"c{chunk}"
        root.mkdir()
        _evaluator(root, chunk=chunk, seed=9).evaluate(_pre(), _dec(BIAS), data, keys)
        _evaluator(root, 1, chunk=chunk, seed=9).evaluate(_pre(), _dec(BIAS), data, keys)
        trees.append(_tree(root / "gen_masks"))
        lines.append(open(root / "dev_bbox_test.txt", "rb").read())
    assert trees[0] == trees[1] == trees[2] and lines[0] == lines[1] == lines[2]
    assert len(trees[0]) == len(keys) and lines[0].count(b"\n") > 0


def test_evaluator_5000_captions(tmp_path):
    data, keys = synthetic_split(n_keys=1000, per_key=5, max_len=40, seed=6)
    data, keys = data[:5000], keys[:5000]
    _evaluator(tmp_path, chunk=1024, seed=1).evaluate(_pre(), _dec(BIAS), data, keys)
    tree = _tree(tmp_path / "gen_masks")
    assert len(tree) == 5000
    rows = 0
    for text in tree.values():
        _, n = _parse_boxes_txt(text.decode())
        for line in text.decode().splitlines():
            f = line.split(",")
            assert len(f) == 6 and f[5] == "0" and f[4] in NAMES and all(1.0 <= float(v) <= 256.0 for v in f[:2])
            rows += 1
    assert rows > 5000
