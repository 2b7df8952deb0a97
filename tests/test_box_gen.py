"""Box generator for caption-to-image sampling (CPU): the oracle (oracle/box_oracle.py) against the reference's own
PreEncoderRNN / DecoderRNN, Evaluator.evaluate and load_gen_insanns; hand-worked layout cases; the state_dict layouts;
the reference checkpoint loader in both pickle formats; the unsupported-configuration and input-check errors; and the
library calls of the box stage (DRY_RUN: host logic only).

The reference side is stored in tests/golden/reference/box_*.  Re-record with the reference importable:

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_box_gen.py
"""
import gzip
import io
import json
import os
import pickle
import sys
import types

import numpy as np
import pytest
import torch

import reference_fixtures as fixtures
import refimport
from dry import dry, record  # noqa: F401
from objgan_b200 import boxgen, model, synth
from objgan_b200.config import cfg
from objgan_b200.sampler import GSampler
from oracle import box_oracle as O
from test_text_encoder import NTOK, _layout, captions_for, enc_sd

BOX_REF = "/root/reference/box_generation"
# the 80 COCO category ids in categories.txt order
CAT_IDS = [*range(1, 12), *range(13, 26), 27, 28, *range(31, 45), *range(46, 66), 67, 70, *range(72, 83),
           *range(84, 91)]
SPECIAL = ["<pad>", "<sos>", "<eos>", "<unk>"]
L2I = {**{w: i for i, w in enumerate(SPECIAL)}, **{str(c): 4 + i for i, c in enumerate(CAT_IDS)}}
NL = len(L2I)                                   # 84
MEANS = (0.5, 0.4, 0.3, 1.1)                    # x_mean, y_mean, w_mean, r_mean of the recorded decoder
SOS, EOS = 1, 2
# name -> (caption length, early_stop_len, added to l_out.bias[<eos>], numpy seed)
DEC_CASES = {"len1": (1, 10, 0.0, 11), "len9": (9, 10, 0.0, 12), "len23": (23, 10, 0.0, 13),
             "no_eos": (9, 10, -12.0, 14), "eos_step1": (5, 10, 12.0, 15)}
LABEL_TO_CLASS = torch.tensor([-1] * 4 + list(range(80)))


# ---------------------------------------------------------------------------------------------------------------------
# the reference's box_generation modules (read-only, CPU)
# ---------------------------------------------------------------------------------------------------------------------
def ref_box():
    if not os.path.isdir(BOX_REF):
        raise RuntimeError("reference not mounted")
    for name in ("nltk", "nltk.tokenize"):
        m = sys.modules.setdefault(name, types.ModuleType(name))
        m.RegexpTokenizer = object
    sys.modules["nltk"].tokenize = sys.modules["nltk.tokenize"]
    if BOX_REF not in sys.path:
        sys.path.insert(0, BOX_REF)
    import seq2seq.models as M
    from seq2seq.evaluator import evaluator as E
    return M, E


def dec_sd(eos_bias=0.0):
    """A DecoderRNN state_dict (n_labels = 84) with every weight uniform(-0.08, 0.08) as sample.py:141 initialises
    them, from a seeded generator; ``eos_bias`` is added to l_out.bias[<eos>]."""
    g = torch.Generator().manual_seed(21)
    net = model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2, use_attention=False, bidirectional=True)
    sd = {k: (torch.rand(v.shape, generator=g) * 0.16 - 0.08) for k, v in net.state_dict().items()}
    sd["l_out.bias"][EOS] += eos_bias
    return sd


def dec_case(name):
    n, _, _, _ = DEC_CASES[name]
    caps, lens = captions_for([n], n, NTOK, 300 + n)
    return caps, lens


def dec_fixture(name):
    def produce():
        M, _ = ref_box()
        n, stop, bias, seed = DEC_CASES[name]
        caps, lens = dec_case(name)
        enc = M.PreEncoderRNN(NTOK, nhidden=256)
        enc.load_state_dict(enc_sd(), strict=True)
        dec = M.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2, use_attention=False, bidirectional=True)
        dec.load_state_dict(dec_sd(bias), strict=True)
        enc.eval(), dec.eval()
        params = []
        real = dec.sample_next_state

        def rec(*a):                                 # sample_bivariate_normal scales sigma in place: clone first
            params.append(torch.cat([t[0].clone() for t in a]))
            return real(*a)
        dec.sample_next_state = rec
        np.random.seed(seed)
        with torch.no_grad():
            out, hid = enc(caps, [n])
            z = torch.zeros(1, 3)
            lout, _, _, _, other = dec(hid, out, torch.ones(1, 3, dtype=torch.long), z, z, z, z, is_training=0,
                                       early_stop_len=stop)
        steps = len(other["sequence"])
        samples = torch.tensor([[*map(float, xy), *map(float, wh)] for xy, wh in zip(other["xy"], other["wh"])],
                               dtype=torch.float64)
        return {"in__captions": caps, "labels": torch.cat(other["sequence"]).float(), "steps": steps,
                "samples": samples, "p": torch.cat(lout), "xy": torch.stack(params[0::2]),
                "wh": torch.stack(params[1::2]), "h_n": hid[0], "c_n": hid[1], "enc_out": out}

    path = os.path.join(fixtures.GOLD, f"box_decoder_{name}.npz")
    if fixtures.RECORD:
        out = produce()
        np.savez_compressed(path, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()})
    z = np.load(path)
    return {k: torch.from_numpy(z[k]) for k in z.files}


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs reference: encoder state and decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(DEC_CASES))
def test_oracle_decoder_matches_reference(name):
    want = dec_fixture(name)
    n, stop, bias, _ = DEC_CASES[name]
    caps, lens = dec_case(name)
    assert torch.equal(want["in__captions"], caps)
    h0, c0 = O.encoder_state(enc_sd(), caps, lens)
    # _cat_directions of the reference's (h_n, c_n)
    assert torch.allclose(h0[0], torch.cat([want["h_n"][0, 0], want["h_n"][1, 0]]), atol=1e-6)
    assert torch.allclose(c0[0], torch.cat([want["c_n"][0, 0], want["c_n"][1, 0]]), atol=1e-6)
    assert want["enc_out"].shape == (1, n, 256)
    sd = dec_sd(bias)
    labels, samples = want["labels"].long(), want["samples"]
    p, xy, wh = O.teacher_forced(sd, h0[0], c0[0], labels, samples, SOS, MEANS)
    torch.testing.assert_close(p, want["p"], atol=2e-6, rtol=1e-5)
    torch.testing.assert_close(xy, want["xy"], atol=2e-6, rtol=1e-5)
    torch.testing.assert_close(wh, want["wh"], atol=2e-6, rtol=1e-5)
    assert torch.equal(p.argmax(1), labels)                  # the reference's labels
    steps = int(want["steps"])
    assert steps == len(labels)
    ends = labels[-1] == EOS
    assert steps == (stop if not ends else int((labels == EOS).nonzero()[0]) + 1)
    if name == "no_eos":
        assert steps == stop and not ends
    if name == "eos_step1":
        assert steps == 1 and ends


def test_oracle_decode_free_running_matches_teacher_forced():
    """The free-running oracle and the teacher-forced one agree on their own trajectory."""
    caps, lens = dec_case("len9")
    h0, c0 = O.encoder_state(enc_sd(), caps, lens)
    noise = torch.randn(10, 6, generator=torch.Generator().manual_seed(3))
    noise[:, 0::3] = torch.rand(10, 2, generator=torch.Generator().manual_seed(4))
    sd = dec_sd()
    out = O.decode(sd, h0[0], c0[0], noise, 10, SOS, EOS, MEANS)
    p, xy, wh = O.teacher_forced(sd, h0[0], c0[0], out["labels"], torch.stack(out["samples"]), SOS, MEANS)
    assert torch.equal(p, torch.stack(out["p"])) and torch.equal(xy, torch.stack(out["xy"]))
    assert torch.equal(wh, torch.stack(out["wh"]))


def test_component_rule():
    """numpy's choice rule: #{k : cdf_k <= u}, clamped to K - 1."""
    pi = torch.tensor([0.2, 0.2, 0.2, 0.2, 0.2])
    assert [O.component(pi, u)[0] for u in (0.0, 0.19, 0.2, 0.99, 1.0)] == [0, 0, 1, 4, 4]
    rng = np.random.RandomState(5)
    for _ in range(200):
        pi = torch.softmax(torch.tensor(rng.randn(5), dtype=torch.float32), 0)
        u = rng.rand()
        q = np.log(pi.numpy()) / np.float32(0.4)
        q = np.exp(q - q.max())
        q /= q.sum()
        assert O.component(pi, u)[0] == min(int(np.searchsorted(np.cumsum(q.astype(np.float64)) /
                                                                 np.cumsum(q.astype(np.float64))[-1], u, "right")), 4)


# ---------------------------------------------------------------------------------------------------------------------
# layout: the reference's Evaluator.evaluate + load_gen_insanns
# ---------------------------------------------------------------------------------------------------------------------
MEAN_STD = [[120.0, 60.0], [110.0, 55.0], [70.0, 40.0], [1.0, 0.5]]
# trajectories (label index, x, y, w, r normalised); the last step of each ends at <eos> unless noted
LAYOUT_TRAJ = [
    [(4, 0.1, 0.2, 0.3, 0.1), (5, -0.5, 0.4, 0.2, -0.2), (4, 0.3, -0.1, 0.5, 0.3), (4, 0.8, 0.7, -0.2, 0.0),
     (4, 0.0, 0.0, 0.0, 0.0), (2, 0.2, 0.2, 0.2, 0.2)],                                     # a capped class
    [(10, 2.1, 2.2, 1.5, 0.6), (11, -2.5, -2.4, 0.1, 0.1), (12, 0.2, 0.1, -1.7, 0.0), (2, -3.0, 0.0, 0.0, 0.0)],
    [(20, 0.3, 0.3, 0.3, 0.3), (21, 0.1, 0.1, 0.1, 0.1), (22, 0.5, 0.5, 0.5, 0.5)],           # no <eos>: drops a box
    [(30, 0.0, 0.0, 0.0, 0.0), (2, -3.0, 0.0, 0.0, 0.0)],                                    # one kept step: none
    [(2, 0.0, 0.0, 0.0, 0.0)],                                                               # <eos> at once
]
# distinct per class (the recording tells the classes apart by their statistics) and with full 53-bit mantissas
COUNT_STATS = torch.tensor([[2.0 + c / 37.0, 0.3 + c / 101.0] for c in range(80)], dtype=torch.float64)
# a mean / std table with full 53-bit mantissas: the de-normalisation must round its product and sum separately
MEAN_STD_FULL = [[120.0 + 1 / 3, 60.0 + 1 / 7], [110.0 + 1 / 11, 55.0 + 1 / 13], [70.0 + 1 / 17, 40.0 + 1 / 19],
                 [1.0 + 1 / 23, 0.5 + 1 / 29]]


def layout_noise_cnt():
    return torch.randn(len(LAYOUT_TRAJ), 80, generator=torch.Generator().manual_seed(9)) * 2.0


def layout_fixture():
    def produce(tmp):
        _, E = ref_box()
        ncnt = layout_noise_cnt()
        keys = [f"img{i}" for i in range(len(LAYOUT_TRAJ))]
        i2w = {i: w for w, i in L2I.items()}
        gdict = {c: (float(COUNT_STATS[i, 0]), float(COUNT_STATS[i, 1])) for i, c in enumerate(CAT_IDS)}
        draws = []
        state = {"b": 0}

        class Dec:
            def __call__(self, *a, **kw):
                traj = LAYOUT_TRAJ[state["b"]]
                seq = [torch.tensor([t[0]]) for t in traj]
                return None, None, None, None, {"sequence": seq, "xy": [(np.float32(t[1]), np.float32(t[2])) for t in traj],
                                                "wh": [(np.float32(t[3]), np.float32(t[4])) for t in traj]}

        ev = E.Evaluator(1, 10, tmp, types.SimpleNamespace(index2word={}),
                         types.SimpleNamespace(index2word=i2w), *[tuple(r) for r in MEAN_STD], gdict,
                         tmp + "/gen_masks/", 0)
        real_rb, real_normal = E.random_batch, np.random.normal

        def rb(*a, select_index, **kw):
            state["b"] = select_index
            return (None,) * 8

        def logged(mu, sigma, size=None):      # the logged draws: mu + sigma * noise_cnt[b, class]
            cat = [c for c, v in gdict.items() if v == (mu, sigma)]
            assert len(cat) == 1
            row = CAT_IDS.index(cat[0])
            v = mu + sigma * float(ncnt[state["b"], row])
            draws.append((state["b"], row, v))
            return np.array([v])
        E.random_batch, np.random.normal = rb, logged
        try:
            ev.evaluate(lambda *a: (None, None), Dec(), [0] * len(keys), keys)
        finally:
            E.random_batch, np.random.normal = real_rb, real_normal
        ref = refimport.load()
        for name in ("pycocotools", "pycocotools.coco", "torchtext", "spacy", "skimage.io"):
            m = sys.modules.setdefault(name, types.ModuleType(name))
            m.COCO = object
        sys.modules["spacy"].load = lambda *a, **kw: None
        sys.modules["skimage.transform"].resize = None
        from miscc import load as L
        ins = L.load_gen_insanns(tmp, keys, "test", [64, 128, 256], 16, {c: i for i, c in enumerate(CAT_IDS)})
        out = {"draws": np.array(draws, dtype=np.float64)}
        files = []
        for i, k in enumerate(keys):
            a = ins[k][0]
            for s in range(3):
                out[f"rois{s}_{i}"] = np.asarray(a["rois"][s], dtype=np.float64)
            out[f"fm_rois_{i}"] = np.asarray(a["fm_rois"], dtype=np.float64)
            out[f"num_rois_{i}"] = np.asarray(a["num_rois"])
            files.append(open(f"{tmp}/gen_masks/{k}/0/boxes.txt").read())
        out["boxes_txt"] = np.array(files)
        return out

    path = os.path.join(fixtures.GOLD, "box_layout.npz")
    if fixtures.RECORD:
        import tempfile
        with tempfile.TemporaryDirectory() as tmp:
            np.savez_compressed(path, **produce(tmp))
    return dict(np.load(path))


def _traj(i):
    t = torch.tensor(LAYOUT_TRAJ[i], dtype=torch.float64)
    return t[:, 0].long(), t[:, 1:].float()


def test_oracle_layout_matches_reference():
    want = layout_fixture()
    ncnt = layout_noise_cnt()
    for i in range(len(LAYOUT_TRAJ)):
        labels, samples = _traj(i)
        rois, fm, cls, n = O.layout(labels, samples, MEAN_STD, LABEL_TO_CLASS, COUNT_STATS, ncnt[i])
        assert n == int(want[f"num_rois_{i}"]), i
        for s in range(3):
            assert np.array_equal(rois[s].numpy(), want[f"rois{s}_{i}"]), (i, s)
        assert np.array_equal(fm.numpy(), want[f"fm_rois_{i}"]), i
        assert torch.equal(cls[:n], rois[0, :n, 4].long())
    assert want["num_rois_3"] == 0 and want["num_rois_4"] == 0 and want["num_rois_0"] >= 2
    assert want["boxes_txt"][3] == "" and want["boxes_txt"][4] == ""
    assert (want["rois2_0"][:int(want["num_rois_0"]), 4] == 0).sum() == 2       # class 0: four boxes, capped at two
    assert sorted(int(r) for b, r, _ in want["draws"] if b == 2) == [16, 17]
    # the draws were mu + sigma * noise_cnt[b, class], one per distinct class and sample
    for b, row, v in want["draws"]:
        assert v == float(COUNT_STATS[int(row), 0]) + float(COUNT_STATS[int(row), 1]) * float(ncnt[int(b), int(row)])


# ---------------------------------------------------------------------------------------------------------------------
# hand-worked layout cases: one sample per case, with MEAN_STD_ID (samples are the de-normalised values)
# ---------------------------------------------------------------------------------------------------------------------
MEAN_STD_ID = [[0.0, 1.0], [0.0, 1.0], [0.0, 1.0], [0.0, 1.0]]


def hand_cases():
    """name -> (labels, samples (x, y, w, r) in pixels / aspect, noise_cnt (80,), count_stats, want rois[2][:n, :4],
    want classes).  The last step is an <eos> step with a valid box (the drop-last rule removes it)."""
    eos = (2, 50.0, 50.0, 20.0, 1.0)
    z = torch.zeros(80)
    cs = torch.tensor([[3.0, 1.0]] * 80, dtype=torch.float64)
    f32 = lambda v: float(np.float32(v))
    cases = {
        # x - w/2 = 12.996... -> '12.99'? no: 12.996 -> '13.00' -> 13; 12.994 -> '12.99' -> 12
        "txt_round": ([4, 5, 2], [(f32(22.996), 40.0, 20.0, 1.0), (f32(22.994), 40.0, 20.0, 1.0), eos[1:]], z, cs,
                      None, [0, 1]),
        "clip": ([4, 5, 2], [(3.0, 250.0, 30.0, 1.0), (250.0, 3.0, 40.0, 0.5), eos[1:]], z, cs,
                 [[1, 235, 30, 21], [230, 1, 26, 20]], [0, 1]),
        "min_size_one": ([4, 5, 2], [(100.0, 100.0, 9.0, 2.0), (100.0, 100.0, 30.0, 0.2), eos[1:]], z, cs,
                         None, [0, 1]),
        "min_size_both": ([4, 5, 2], [(100.0, 100.0, 9.0, 1.0), (100.0, 100.0, 30.0, 1.0), eos[1:]], z, cs,
                          None, [1]),
        "negative_threshold": ([4, 4, 4, 2], [(60.0, 60.0, 20.0, 1.0)] * 3 + [eos[1:]],
                               torch.full((80,), -50.0), cs, None, [0, 0]),
        "cap": ([4, 4, 4, 4, 4, 5, 2], [(60.0 + k, 60.0, 20.0, 1.0) for k in range(6)] + [eos[1:]],
                torch.tensor([0.9] + [0.0] * 79), cs, None, [0, 0, 0, 1]),
        "drop_last_no_eos": ([4, 5, 6], [(60.0, 60.0, 20.0, 1.0)] * 3, z, cs, None, [0, 1]),
        "drop_last_invalid_eos": ([4, 5, 2], [(60.0, 60.0, 20.0, 1.0), (60.0, 60.0, 20.0, 1.0), (-1.0, 5.0, 5.0, 1.0)],
                                  z, cs, None, [0]),
        "special_mid": ([4, 3, 0, 5, 1, 2], [(60.0, 60.0, 20.0, 1.0)] * 5 + [eos[1:]], z, cs, None, [0, 1]),
        "empty": ([4, 2], [(60.0, 60.0, 20.0, 1.0), (-5.0, 60.0, 20.0, 1.0)], z, cs, None, []),
    }
    return cases


@pytest.mark.parametrize("name", list(hand_cases()))
def test_layout_hand_worked(name):
    labels, samples, ncnt, cs, want_box, want_cls = hand_cases()[name]
    rois, fm, cls, n = O.layout(torch.tensor(labels), torch.tensor(samples), MEAN_STD_ID, LABEL_TO_CLASS, cs, ncnt)
    assert n == len(want_cls) and cls[:n].tolist() == want_cls
    assert rois[:, n:].abs().sum() == 0 and fm[n:].abs().sum() == 0 and cls[n:].abs().sum() == 0
    assert torch.equal(fm[:n, :4], rois[0, :n, :4] / 2) and torch.equal(rois[1, :n, :4], rois[2, :n, :4] / 2)
    assert torch.equal(rois[0, :n, :4], rois[2, :n, :4] / 4) and torch.equal(rois[:, :n, 4], cls[:n].double().expand(3, n))
    assert (rois[2, :n, :4] == rois[2, :n, :4].round()).all()
    if want_box is not None:
        assert rois[2, :n, :4].tolist() == want_box
    if name == "txt_round":                            # 22.996 - 10 = 12.996 -> 13; 12.994 -> 12
        assert rois[2, 0, 0] == 13 and rois[2, 1, 0] == 12


# '%.2f' boundaries reached exactly: x = mean + 0 * std, then x - w / 2 with w = 20 lands on the double just below
# (x) or just above (y) 12.995, which '%.2f' writes as 12.99 and 13.00
MEAN_STD_EDGE = [[float(np.nextafter(22.995, 0)), 1.0], [float(np.nextafter(22.995, 30)), 1.0], [20.0, 1.0],
                 [1.0, 1.0]]
EDGE_TRAJ = ([4, 5, 2], [(0.0, 0.0, 0.0, 0.0), (1.0, 1.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0)])


def test_layout_txt_boundary_exact():
    labels, samples = EDGE_TRAJ
    rois, _, _, n = O.layout(torch.tensor(labels), torch.tensor(samples), MEAN_STD_EDGE, LABEL_TO_CLASS,
                             COUNT_STATS, torch.zeros(80))
    assert n == 2
    assert MEAN_STD_EDGE[0][0] - 10.0 < 12.995 < MEAN_STD_EDGE[1][0] - 10.0
    assert rois[2, 0, :2].tolist() == [12, 13] and rois[2, 1, :2].tolist() == [13, 14]


def test_txt_round_trip_boundaries():
    """int(float('%.2f' % v)) against the kernel's rule floor(v) + (frac(v) > 0.995) on values around every boundary."""
    vals = [k + f for k in (1, 12, 254) for f in (0.994999, 0.995, 0.99500000001, 0.9951, 0.999, 0.0, 0.5)]
    vals += list(np.nextafter(np.float64(12.995), 0)[None]) + [np.nextafter(np.float64(12.995), 20)]
    for v in vals:
        v = float(v)
        f = np.floor(v)
        assert int(float("%.2f" % v)) == int(f + (1.0 if v - f > 0.995 else 0.0)), v


# ---------------------------------------------------------------------------------------------------------------------
# module API, layouts, loader
# ---------------------------------------------------------------------------------------------------------------------
def box_layouts():
    """{"decoder": [[key, shape]], "encoder": [[key, shape]], sha256s} of the reference's modules."""
    path = os.path.join(fixtures.GOLD, "box_layout.json")
    if fixtures.RECORD:
        M, _ = ref_box()
        d = M.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2, use_attention=False, bidirectional=True)
        e = M.PreEncoderRNN(NTOK, nhidden=256)
        json.dump({n: {"state": _layout(m.state_dict()), "keys": [[k, list(v.shape)] for k, v in m.state_dict().items()]}
                   for n, m in (("decoder", d), ("encoder", e))}, open(path, "w"), indent=0)
    return json.load(open(path))


def test_state_dict_layouts_match_reference():
    ref = box_layouts()
    d = model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2, use_attention=False, bidirectional=True)
    e = model.PreEncoderRNN(NTOK, nhidden=256)
    for name, m in (("decoder", d), ("encoder", e)):
        sd = m.state_dict()
        assert [[k, list(v.shape)] for k, v in sd.items()] == ref[name]["keys"]
        assert _layout(sd) == ref[name]["state"]
    e.load_state_dict(enc_sd(), strict=True)             # the text encoder's snapshot loads as is


def reference_checkpoints():
    """{"zip": bytes, "legacy": bytes} of a reference-made ``torch.save(decoder)`` (checkpoint.py:91) of a DecoderRNN
    with 6 labels and a patterned state, gzip-compressed, and that state."""
    l2i = {**{w: i for i, w in enumerate(SPECIAL)}, "1": 4, "3": 5}
    pattern = lambda v, i: ((torch.arange(v.numel()) * (i + 3)) % 17 - 8).float().view(v.shape) * 0.01
    path = os.path.join(fixtures.GOLD, "box_decoder_checkpoint.npz")
    if fixtures.RECORD:
        M, _ = ref_box()
        d = M.DecoderRNN(l2i, 0.5, 0.4, 0.3, 1.1, 1, 150, 256, 5, dropout_p=0.2, use_attention=False,
                         bidirectional=True)
        d.load_state_dict({k: pattern(v, i) for i, (k, v) in enumerate(d.state_dict().items())})
        blobs = {}
        for fmt, zipf in (("zip", True), ("legacy", False)):
            buf = io.BytesIO()
            torch.save(d, buf, _use_new_zipfile_serialization=zipf)
            blobs[fmt] = np.frombuffer(gzip.compress(buf.getvalue(), 9), dtype=np.uint8)
        idx = io.BytesIO()
        pickle.dump({i: w for w, i in l2i.items()}, idx)
        blobs["label_index2word"] = np.frombuffer(idx.getvalue(), dtype=np.uint8)
        np.savez(path, **blobs)
    z = np.load(path)
    return {k: z[k].tobytes() for k in z.files}, l2i, pattern


@pytest.mark.parametrize("fmt", ["zip", "legacy"])
def test_reference_checkpoint_loader(fmt, tmp_path):
    blobs, l2i, pattern = reference_checkpoints()
    p = tmp_path / "model.pt"
    p.write_bytes(gzip.decompress(blobs[fmt]))
    dec = boxgen.load_reference_decoder(str(p))
    assert dec.l_output_size == 6 and dec.l_sos_id == 1 and dec.l_eos_id == 2 and not dec.training
    assert (dec.x_mean, dec.y_mean, dec.w_mean, dec.r_mean) == (0.5, 0.4, 0.3, 1.1)
    for i, (k, v) in enumerate(dec.state_dict().items()):
        assert torch.equal(v, pattern(v, i)), k


class _AsCall:
    """Pickles as fn(*args) (a REDUCE on the global fn)."""

    def __init__(self, fn, *args):
        self.fn, self.args = fn, args

    def __reduce__(self):
        return self.fn, self.args


class _AsObject:
    """Pickles as an instance of ``cls`` with ``state`` (NEWOBJ + BUILD), the way torch.save(module) writes a module."""

    def __init__(self, cls, state):
        self._cls, self._state = cls, state

    @property
    def __class__(self):
        return self._cls

    def __reduce_ex__(self, proto):
        import copyreg
        return copyreg.__newobj__, (self._cls,), self._state


def _torch04_pickle(dec, l2i):
    """A legacy-format torch.save(decoder) as torch 0.4 (the reference's pin) writes it: every module has a
    ``_backend`` pickled through torch.nn.backends.thnn._get_thnn_function_backend, and every Parameter is pickled as
    torch.nn.parameter.Parameter(tensor, requires_grad)."""
    import collections
    import copyreg  # noqa: F401
    backend = _AsCall(torch.nn.backends.thnn._get_thnn_function_backend)

    def module(cls, params, children=(), **attrs):
        st = dict(_backend=backend, training=False, _buffers=collections.OrderedDict(),
                  _backward_hooks=collections.OrderedDict(), _forward_hooks=collections.OrderedDict(),
                  _forward_pre_hooks=collections.OrderedDict(), _state_dict_hooks=collections.OrderedDict(),
                  _load_state_dict_pre_hooks=collections.OrderedDict(),
                  _parameters=collections.OrderedDict((k, _AsCall(torch.nn.parameter.Parameter, v.clone(), True))
                                                      for k, v in params.items()),
                  _modules=collections.OrderedDict(children), **attrs)
        return _AsObject(cls, st)
    sd = dec.state_dict()
    sub = lambda p: {k[len(p) + 1:]: v for k, v in sd.items() if k.startswith(p + ".")}
    lin = lambda p: module(torch.nn.Linear, sub(p), in_features=sub(p)["weight"].shape[1],
                           out_features=sub(p)["weight"].shape[0])
    names = ["weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"]
    children = [("input_dropout", module(torch.nn.Dropout, {}, p=0.0, inplace=False)),
                ("l_embedding", module(torch.nn.Embedding, sub("l_embedding"), num_embeddings=len(l2i),
                                       embedding_dim=256, padding_idx=None, max_norm=None, norm_type=2,
                                       scale_grad_by_freq=False, sparse=False)),
                ("xy_embedding", lin("xy_embedding")), ("wh_embedding", lin("wh_embedding")),
                ("next_xy_embedding", lin("next_xy_embedding")),
                ("rnn", module(torch.nn.LSTM, sub("rnn"), mode="LSTM", input_size=356, hidden_size=256, num_layers=1,
                               bias=True, batch_first=True, dropout=0.2, bidirectional=False, _all_weights=[names],
                               _data_ptrs=[], dropout_state={})),
                ("l_out", lin("l_out")), ("xy_out", lin("xy_out")), ("wh_out", lin("wh_out"))]
    stub = type("DecoderRNN", (), {"__module__": "seq2seq.models.DecoderRNN"})
    top = module(stub, {}, children, vocab_size=len(l2i), max_len=150, hidden_size=256, n_layers=1,
                 input_dropout_p=0, dropout_p=0.2, rnn_cell=torch.nn.LSTM, bidirectional_encoder=True,
                 l_output_size=len(l2i), aug_size=50, batch_size=1, max_length=150, gmm_comp_num=5,
                 gmm_param_num=6, clip_val=0.01, use_attention=False, l_eos_id=l2i["<eos>"], l_sos_id=l2i["<sos>"],
                 x_mean=dec.x_mean, y_mean=dec.y_mean, w_mean=dec.w_mean, r_mean=dec.r_mean, temperature=0.4,
                 init_input=None, l_softmax=torch.nn.functional.log_softmax)
    mods = {n: types.ModuleType(n) for n in ("seq2seq", "seq2seq.models", "seq2seq.models.DecoderRNN")}
    mods["seq2seq.models.DecoderRNN"].DecoderRNN = stub
    saved = {n: sys.modules.get(n) for n in mods}
    sys.modules.update(mods)
    try:
        buf = io.BytesIO()
        torch.save(top, buf, _use_new_zipfile_serialization=False, pickle_protocol=2)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n)
            else:
                sys.modules[n] = m
    return buf.getvalue()


def test_reference_checkpoint_loader_torch04_pickle(tmp_path):
    """A 0.4-era pickle names Parameter and the thnn backend function; it loads, and the state_dict is exact."""
    l2i = {**{w: i for i, w in enumerate(SPECIAL)}, "1": 4, "3": 5}
    want = model.DecoderRNN(l2i, 0.5, 0.4, 0.3, 1.1, 1, 150, 256, 5, dropout_p=0.2, bidirectional=True)
    with torch.no_grad():
        for i, p in enumerate(want.parameters()):
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(i)))
    data = _torch04_pickle(want, l2i)
    assert b"torch.nn.parameter" in data and b"_get_thnn_function_backend" in data
    assert b"_rebuild_parameter" not in data
    (tmp_path / "model.pt").write_bytes(data)
    dec = boxgen.load_reference_decoder(str(tmp_path / "model.pt"))
    assert dec.l_output_size == 6 and dec.l_eos_id == 2 and (dec.x_mean, dec.r_mean) == (0.5, 1.1)
    got, ref = dec.state_dict(), want.state_dict()
    assert list(got) == list(ref) and all(torch.equal(got[k], ref[k]) for k in ref)


def test_checkpoint_loader_refuses_other_globals(tmp_path):
    class Evil:
        def __reduce__(self):
            return (os.system, ("true",))
    for payload in (Evil(), {"a": Evil()}):
        p = tmp_path / "model.pt"
        torch.save(payload, str(p))
        with pytest.raises(pickle.UnpicklingError, match="refusing"):
            boxgen.load_reference_decoder(str(p))
    buf = io.BytesIO()
    pickle.dump(types.SimpleNamespace(a=1), buf)
    (tmp_path / "ns.pt").write_bytes(buf.getvalue())
    with pytest.raises(pickle.UnpicklingError, match="refusing"):
        boxgen.load_reference_decoder(str(tmp_path / "ns.pt"))


def test_from_reference_files(tmp_path):
    blobs, l2i, _ = reference_checkpoints()
    d = tmp_path / "checkpoints" / "ck"
    d.mkdir(parents=True)
    (d / "model.pt").write_bytes(gzip.decompress(blobs["zip"]))
    (d / "label_index2word.pt").write_bytes(blobs["label_index2word"])
    torch.save({"module." + k: v for k, v in enc_sd().items()}, tmp_path / "text_encoder.pth")
    (tmp_path / "mean_std.txt").write_text("120.0 60.0\n110.0 55.0\n70.0 40.0\n1.0 0.5\n")
    np.save(tmp_path / "gaussian_dict.npy", {1: (3.0, 1.0), 3: (2.5, 0.5), 7: (4.0, 2.0)})
    bg = boxgen.BoxGenerator.from_reference(str(d), str(tmp_path / "text_encoder.pth"), str(tmp_path / "mean_std.txt"),
                                            str(tmp_path / "gaussian_dict.npy"), [1, 7, 3], device="cpu")
    assert bg.label_to_class.tolist() == [-1, -1, -1, -1, 0, 2]
    assert bg.count_stats.tolist() == [[3.0, 1.0], [4.0, 2.0], [2.5, 0.5]]
    assert bg.mean_std.tolist() == [[120.0, 60.0], [110.0, 55.0], [70.0, 40.0], [1.0, 0.5]]
    with pytest.raises(ValueError, match="no statistics"):
        boxgen.BoxGenerator.from_reference(str(d), str(tmp_path / "text_encoder.pth"), str(tmp_path / "mean_std.txt"),
                                           str(tmp_path / "gaussian_dict.npy"), [1, 7, 3, 9], device="cpu")


def _gen(early_stop_len=10, **kw):
    enc = model.PreEncoderRNN(NTOK, nhidden=256)
    dec = model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, bidirectional=True)
    args = dict(mean_std=MEAN_STD, count_stats=COUNT_STATS, label_to_class=LABEL_TO_CLASS)
    args.update(kw)
    return boxgen.BoxGenerator(enc, dec, early_stop_len=early_stop_len, **args)


def test_unsupported_and_input_checks(dry):
    mk = lambda **kw: model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, **{"bidirectional": True, **kw})
    for kw in ({"use_attention": True}, {"rnn_cell": "gru"}, {"n_layers": 2}):
        with pytest.raises(NotImplementedError):
            mk(**kw)
    for kw in ({"nhidden": 128}, {"nlayers": 2}, {"bidirectional": False}):
        with pytest.raises(NotImplementedError):
            model.PreEncoderRNN(NTOK, **{"nhidden": 256, **kw})
    for bad in (0, 12):
        with pytest.raises(ValueError, match="early_stop_len"):
            _gen(bad)
    _gen(11)
    with pytest.raises(ValueError, match="count_stats"):
        _gen(count_stats=COUNT_STATS[:, :1])
    nan = COUNT_STATS.clone()
    nan[5, 1] = float("nan")
    with pytest.raises(ValueError, match="count_stats"):
        _gen(count_stats=nan)
    with pytest.raises(ValueError, match="outside"):
        _gen(count_stats=COUNT_STATS[:40])
    bad = LABEL_TO_CLASS.clone()
    bad[1] = 0
    with pytest.raises(ValueError, match="special token"):
        _gen(label_to_class=bad)
    with pytest.raises(ValueError, match="one entry per"):
        _gen(label_to_class=LABEL_TO_CLASS[:50])
    # inference only
    dec = mk()
    h = torch.zeros(2, 256)
    nz = torch.zeros(2, 10, 6)
    with pytest.raises(RuntimeError, match=r"call \.eval\(\)"):
        dec.sample_state(h, h, nz, 10)
    dec.eval()
    with pytest.raises(RuntimeError, match="inference only"):
        dec.sample_state(h, h, nz, 10)
    with torch.no_grad():
        labels, samples, steps, dbg = dec.sample_state(h, h, nz, 10, debug=True)
    assert labels.shape == (2, 10) and samples.shape == (2, 10, 4) and steps.shape == (2,) and dbg.shape == (2, 10, 144)
    enc = model.PreEncoderRNN(NTOK, nhidden=256)
    caps, lens = captions_for([4, 2], 6, NTOK, 1)
    with pytest.raises(RuntimeError, match=r"call \.eval\(\)"):
        enc(caps, lens)
    enc.eval()
    with torch.no_grad():
        out, (h_n, c_n) = enc(caps, lens)
    assert out.shape == (2, 4, 256) and h_n.shape == c_n.shape == (2, 2, 128)


def _trace(fn):
    return [name for name, _ in record(fn)]


@pytest.mark.parametrize("B,L", [(1, 1), (5, 40)])
def test_box_stage_call_sequence(dry, B, L):
    """The box stage is five library calls whatever B and the caption length; the derived weights are made once."""
    bg = _gen()
    caps, lens = captions_for([L] * B, L, NTOK, 2)
    nb, nc = bg.draw_noise(B)
    first = _trace(lambda: bg.sample(caps, lens, L, nb, nc))
    assert first.count("og_box_label_table") == 1
    calls = _trace(lambda: bg.sample(caps, lens, L, nb, nc))
    assert calls == ["og_gather_rows", "og_conv2d_simt", "og_lstm_bidir_state", "og_box_decode", "og_box_layout"]
    out = bg.sample(caps, lens, L, nb, nc)
    assert [r.shape for r in out["rois"]] == [(B, 10, 6)] * 3 and out["fm_rois"].shape == (B, 10, 6)
    assert out["roi_cls"].shape == (B, 10) and out["num_rois"].shape == (B,) and out["labels"].shape == (B, 10)


def test_sampler_box_checks(dry):
    bg = _gen()
    x = {"captions": captions_for([4, 6], 18, NTOK, 3)[0], "cap_lens": torch.tensor([4, 6]),
         "glove_captions": captions_for([4, 6], 18, 40, 4)[0]}
    s = GSampler(model.G_NET(80), text_encoder=model.RNN_ENCODER(NTOK, nhidden=256), glove=torch.randn(40, 50),
                 box_generator=bg)
    with pytest.raises(ValueError, match="shape generator"):
        s.sample_eager(x)
    with pytest.raises(ValueError, match="no box generator"):
        GSampler(model.G_NET(80), model.SHP_G_NET(80), text_encoder=model.RNN_ENCODER(NTOK, nhidden=256),
                 glove=torch.randn(40, 50)).sample_eager(x)
    s = GSampler(model.G_NET(80), model.SHP_G_NET(80), text_encoder=model.RNN_ENCODER(NTOK, nhidden=256),
                 glove=torch.randn(40, 50), box_generator=bg)
    for k, v, msg in (("box_cap_lens", torch.tensor([0, 3]), "lengths"), ("box_cap_lens", torch.tensor([19, 3]), "lengths"),
                      ("noise_box", torch.zeros(2, 9, 6), "noise_box")):
        bad = dict(x, box_captions=x["captions"], box_cap_lens=x["cap_lens"])
        bad[k] = v
        with pytest.raises(ValueError, match=msg):
            s.sample_layout(bad)
    with pytest.raises(ValueError, match="give both or neither"):
        s.sample_layout(dict(x, box_captions=x["captions"]))
    bad = dict(x, box_captions=x["captions"].clone())
    bad["box_captions"][0, 0] = NTOK
    bad["box_cap_lens"] = x["cap_lens"]
    with pytest.raises(ValueError, match="token ids"):
        s.sample_layout(bad)
