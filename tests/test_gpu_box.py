"""GPU tests of the box stage of caption-to-image sampling: the encoder's final state (og_lstm_bidir_state), og_box_decode
and og_box_layout against the CPU oracle (oracle/box_oracle.py, pinned to the reference by tests/test_box_gen.py),
bitwise repeatability and batch invariance, and GSampler on caption-only batches (graph replay, the oracle composition
box -> shape -> G, from_snapshot with a reference-format box checkpoint, a full-size batch)."""
import gzip

import numpy as np
import pytest
import torch

from objgan_b200 import boxgen, model, ops, synth
from objgan_b200.sampler import GSampler
from oracle import box_oracle as O
from oracle import text_oracle as T
from test_box_gen import (COUNT_STATS, EDGE_TRAJ, EOS, L2I, LABEL_TO_CLASS, LAYOUT_TRAJ, MEAN_STD, MEAN_STD_EDGE,
                          MEAN_STD_FULL, MEAN_STD_ID, MEANS, SOS, dec_sd, hand_cases, layout_noise_cnt,
                          reference_checkpoints)
from test_gpu_sample import _flat, _same, close
from test_gpu_shape import _g_eval, _shp
from test_gpu_text import _enc, _glove, ragged_lens
from test_shape_gen import shp_sd
from test_text_encoder import NTOK, caption_batch, captions_for, enc_sd

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]
NGLOVE = 70
EPS = 1e-4            # a discrete choice may differ from the oracle's only where the oracle's margin is below this


def _frozen(net):
    for p in net.parameters():
        p.requires_grad_(False)
    return net.to(DEV).eval()


def _pre(sd=None):
    net = model.PreEncoderRNN(NTOK, nhidden=256)
    net.load_state_dict(sd or enc_sd(), strict=True)
    return _frozen(net)


def _dec(bias=0.0):
    net = model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2, use_attention=False, bidirectional=True)
    net.load_state_dict(dec_sd(bias), strict=True)
    return _frozen(net)


def _noise(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    nz = torch.randn(B, S, 6, generator=g)
    nz[:, :, 0::3] = torch.rand(B, S, 2, generator=g)
    return nz


def _box_gen(bias=0.0, early_stop_len=10):
    return boxgen.BoxGenerator(_pre(), _dec(bias), MEAN_STD, COUNT_STATS, LABEL_TO_CLASS, early_stop_len)


# ---------------------------------------------------------------------------------------------------------------------
# encoder state
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,L", [(1, 1), (7, 23), (65, 64)])
def test_encoder_state_vs_oracle(B, L):
    enc = _pre()
    lens = ragged_lens(B, L, B + L)
    caps, _ = captions_for(lens, L, NTOK, 7 * B + L)
    words, h, c = enc.encode_state(caps.to(DEV), lens.to(DEV), L)
    h_ref, c_ref = O.encoder_state(enc_sd(), caps, lens)
    close(h, h_ref, 1e-5, "h")
    close(c, c_ref, 1e-5, "c")
    # the text encoder's entry point is unchanged: same words / sent, bit for bit
    words0, sent0 = RNNE(enc)(caps.to(DEV), lens.to(DEV), L)
    assert torch.equal(words0, words) and torch.equal(sent0, h)
    out, (h_n, c_n) = enc(caps.to(DEV), lens.to(DEV))
    assert out.shape == (B, int(lens.max()), 256) and h_n.shape == (2, B, 128)
    assert torch.equal(h_n.transpose(0, 1).reshape(B, 256), h) and torch.equal(c_n.transpose(0, 1).reshape(B, 256), c)


def RNNE(pre):
    net = model.RNN_ENCODER(NTOK, nhidden=256)
    net.load_state_dict(pre.state_dict(), strict=True)
    return _frozen(net)


# ---------------------------------------------------------------------------------------------------------------------
# the decoder
# ---------------------------------------------------------------------------------------------------------------------
def _check_decode(sd, h0, c0, nz, S, labels, samples, steps, dbg):
    """Each sample step by step against the free-running oracle on the same noise; where a discrete choice differs the
    oracle's margin there must be below EPS, and the sample is then checked teacher-forced on its own trajectory.
    Returns the number of such samples."""
    nl = len(L2I)
    diverged = 0
    labels, samples, steps, dbg = labels.cpu(), samples.cpu(), steps.cpu(), dbg.cpu()
    for b in range(h0.shape[0]):
        ref = O.decode(sd, h0[b], c0[b], nz[b], S, SOS, EOS, MEANS)
        n = int(steps[b])
        assert 1 <= n <= S and (labels[b, n:] == -1).all() and samples[b, n:].abs().sum() == 0
        assert n == S or int(labels[b, n - 1]) == EOS
        assert (labels[b, :n - 1] != EOS).all()
        split = None
        for t in range(min(n, len(ref["labels"]))):
            close(dbg[b, t, :nl], ref["p"][t], 1e-4, f"p {b} {t}")
            close(dbg[b, t, nl:nl + 30], ref["xy"][t], 1e-4, f"xy {b} {t}")
            same = int(labels[b, t]) == ref["labels"][t]
            if not same:
                assert ref["margin"][t][0] < EPS, (b, t, ref["margin"][t])
                split = t
                break
            if not torch.allclose(samples[b, t, :2], ref["samples"][t][:2], atol=1e-3, rtol=1e-3):
                assert ref["margin"][t][1] < EPS, (b, t, ref["margin"][t])
                split = t
                break
            close(dbg[b, t, nl + 30:], ref["wh"][t], 1e-4, f"wh {b} {t}")
            if not torch.allclose(samples[b, t, 2:], ref["samples"][t][2:], atol=1e-3, rtol=1e-3):
                assert ref["margin"][t][2] < EPS, (b, t, ref["margin"][t])
                split = t
                break
        if split is None:
            assert n == len(ref["labels"]), b
            continue
        diverged += 1
        p, xy, wh = O.teacher_forced(sd, h0[b], c0[b], labels[b, :n], samples[b, :n], SOS, MEANS)
        close(dbg[b, :n, :nl], p, 1e-4, f"teacher-forced p {b}")
        close(dbg[b, :n, nl:nl + 30], xy, 1e-4, f"teacher-forced xy {b}")
        close(dbg[b, :n, nl + 30:], wh, 1e-4, f"teacher-forced wh {b}")
    return diverged


@pytest.mark.parametrize("S", [1, 10])
@pytest.mark.parametrize("B", [1, 7, 64, 65])
def test_box_decode_vs_oracle(B, S):
    bias = 0.3                                        # some samples stop early at <eos>, some run to early_stop_len
    enc, dec = _pre(), _dec(bias)
    lens = ragged_lens(B, 20, B + S)
    caps, _ = captions_for(lens, 20, NTOK, B * 3 + S)
    _, h, c = enc.encode_state(caps.to(DEV), lens.to(DEV), 20)
    nz = _noise(B, S, 40 + B)
    labels, samples, steps, dbg = dec.sample_state(h, c, nz.to(DEV), S, debug=True)
    n = _check_decode(dec_sd(bias), h.cpu(), c.cpu(), nz, S, labels, samples, steps, dbg)
    print(f"B={B} S={S}: {n} of {B} samples took a different discrete choice at an oracle margin < {EPS}")
    if S == 10:
        st = steps.cpu()
        assert B < 7 or (st < S).any()


def test_box_decode_repeatable_and_batch_invariant():
    dec, enc = _dec(0.3), _pre()
    B = 64
    lens = ragged_lens(B, 30, 5)
    caps, _ = captions_for(lens, 30, NTOK, 6)
    _, h, c = enc.encode_state(caps.to(DEV), lens.to(DEV), 30)
    nz = _noise(B, 10, 7).to(DEV)
    first = dec.sample_state(h, c, nz, 10, debug=True)
    again = dec.sample_state(h, c, nz, 10, debug=True)
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    no_dbg = dec.sample_state(h, c, nz, 10)
    assert all(torch.equal(a, b) for a, b in zip(first[:3], no_dbg[:3]))
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1)).to(DEV)
    pl = dec.sample_state(h[perm], c[perm], nz[perm], 10, debug=True)
    assert all(torch.equal(a, b[perm]) for a, b in zip(pl, first))
    for i in (0, 33, 63):                              # a sample alone gives what it gives inside B = 64
        one = dec.sample_state(h[i:i + 1], c[i:i + 1], nz[i:i + 1], 10, debug=True)
        assert all(torch.equal(a[0], b[i]) for a, b in zip(one, first))


# ---------------------------------------------------------------------------------------------------------------------
# the layout
# ---------------------------------------------------------------------------------------------------------------------
def _pad(trajs):
    """Trajectories of different lengths as (labels (B, S) with -1 after the end, samples (B, S, 4), steps)."""
    S = max(len(t[0]) for t in trajs)
    B = len(trajs)
    labels = torch.full((B, S), -1, dtype=torch.int64)
    samples = torch.zeros(B, S, 4)
    steps = torch.zeros(B, dtype=torch.int64)
    for b, (lab, smp) in enumerate(trajs):
        labels[b, :len(lab)] = torch.as_tensor(lab)
        samples[b, :len(lab)] = torch.as_tensor(smp, dtype=torch.float32)
        steps[b] = len(lab)
    return labels, samples, steps


def _layout_vs_oracle(trajs, mean_std, cs, ncnt):
    labels, samples, steps = _pad(trajs)
    rois, fm, cls, num = ops.boxes_to_layout(labels.to(DEV), samples.to(DEV), steps.to(DEV),
                                             torch.tensor(mean_std, dtype=torch.float64).to(DEV),
                                             LABEL_TO_CLASS.to(DEV), cs.to(DEV), ncnt.to(DEV))
    for b, (lab, smp) in enumerate(trajs):
        r, f, c, n = O.layout(torch.as_tensor(lab), torch.as_tensor(smp, dtype=torch.float32), mean_std,
                              LABEL_TO_CLASS, cs[b] if cs.dim() == 3 else cs, ncnt[b])
        assert int(num[b]) == n, b
        for s in range(3):
            assert torch.equal(rois[s][b].cpu(), r[s]), (b, s)
        assert torch.equal(fm[b].cpu(), f) and torch.equal(cls[b].cpu(), c), b


def test_box_layout_hand_worked_bitwise():
    cases = list(hand_cases().values())
    cs = cases[0][3]
    assert all(torch.equal(c[3], cs) for c in cases)
    _layout_vs_oracle([(c[0], c[1]) for c in cases], MEAN_STD_ID, cs, torch.stack([c[2] for c in cases]))


def test_box_layout_reference_trajectories_bitwise():
    trajs = [([t[0] for t in tr], [t[1:] for t in tr]) for tr in LAYOUT_TRAJ]
    _layout_vs_oracle(trajs, MEAN_STD, COUNT_STATS, layout_noise_cnt())


def test_box_layout_txt_boundary_bitwise():
    """Values on either side of the exact '%.2f' boundary 12.995 (the doubles next to it)."""
    _layout_vs_oracle([EDGE_TRAJ], MEAN_STD_EDGE, COUNT_STATS, torch.zeros(1, 80))
    _layout_vs_oracle([EDGE_TRAJ, EDGE_TRAJ], MEAN_STD_EDGE, COUNT_STATS, torch.zeros(2, 80))


@pytest.mark.parametrize("mean_std", ["integer", "full_mantissa"])
def test_box_layout_decoder_samples_bitwise(mean_std):
    """The layout of real decoder trajectories (B = 65) against the oracle, bit for bit; with full 53-bit mean / std
    and count statistics a fused multiply-add would differ from the oracle's separately rounded product and sum."""
    ms = MEAN_STD if mean_std == "integer" else MEAN_STD_FULL
    bg = boxgen.BoxGenerator(_pre(), _dec(), ms, COUNT_STATS, LABEL_TO_CLASS)
    lens = ragged_lens(65, 30, 9)
    caps, _ = captions_for(lens, 30, NTOK, 10)
    nb, nc = _noise(65, 10, 11).to(DEV), torch.randn(65, 80, generator=torch.Generator().manual_seed(12)).to(DEV)
    out = bg.sample(caps.to(DEV), lens.to(DEV), 30, nb, nc)
    trajs = [(out["labels"][b, :int(out["steps"][b])].cpu(), out["samples"][b, :int(out["steps"][b])].cpu())
             for b in range(65)]
    _layout_vs_oracle(trajs, ms, COUNT_STATS, nc.cpu())
    assert int(out["num_rois"].max()) >= 2


# ---------------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------------
def _sampler(g=None, box_bias=0.0):
    return GSampler(g or _g_eval(), _shp(shp_sd()), text_encoder=_enc(enc_sd()), glove=_glove(),
                    box_generator=_box_gen(box_bias))


def caption_only(B, seed, lens, box_len=None):
    x = caption_batch(B, seed, lens, NTOK, NGLOVE, parity=True)
    keep = {k: x[k] for k in ("captions", "cap_lens", "glove_captions", "z", "eps")}
    g = torch.Generator().manual_seed(seed)
    keep["noise_shp"] = torch.randn(B, 10, 320, generator=g)
    keep["noise_box"] = _noise(B, 10, seed + 1)
    keep["noise_cnt"] = torch.randn(B, 80, generator=g)
    keep["clabels_emb"] = x["clabels_emb"]
    if box_len is not None:
        bl = ragged_lens(B, box_len, seed)
        keep["box_captions"], keep["box_cap_lens"] = captions_for(bl, box_len, NTOK, seed + 2)
    return keep


def oracle_box_sample(sd_g, x):
    """text oracle -> shape oracle -> form_hmaps -> eval-mode G_NET oracle on the layout in x."""
    import oracle_eval
    from oracle import shape_oracle as S
    n = int(x["cap_lens"].max())
    words, sent = T.rnn_encoder_forward(enc_sd(), x["captions"], x["cap_lens"], n)
    gw, mask = T.text_inputs(x["captions"], x["glove_captions"], _glove(), n)
    r = int(x["glb_max_num_roi"])
    b = x["z"].shape[0]
    slabels = torch.zeros(b, r, x["clabels_emb"].shape[1])
    for i in range(b):
        k = int(x["num_rois"][i])
        slabels[i, :k] = x["clabels_emb"][x["roi_cls"][i, :k]]
    fwd, bwd, fm = S.bbox_maps(x["rois"][0], x["fm_rois"], x["num_rois"], r, 80)
    raw = S.shp_g_net_forward(shp_sd(), x["noise_shp"][:, :r], fwd, bwd, fm)
    hm, bt, fmb = S.form_hmaps(raw[:, :, 0], x["num_rois"], x["roi_cls"])
    inp = dict(z=x["z"], eps=x["eps"], sent_emb=sent, words_embs=words, glove_words_embs=gw, mask=mask,
               slabels_feat=slabels.transpose(1, 2).unsqueeze(3).contiguous(), hmaps=hm, rois=x["rois"],
               fm_rois=x["fm_rois"], num_rois=x["num_rois"], bt_masks=bt, fm_bt_masks=fmb, glb_max_num_roi=r)
    return oracle_eval.g_net_forward_eval(sd_g, inp)


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_caption_only_vs_layout_and_oracle(engine, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    g = _g_eval()
    s = _sampler(g)
    x = caption_only(3, 33, [9, 14, 3], box_len=40)
    lay = s.sample_layout(x)
    got = s.sample(x)
    with_layout = dict(x, **{k: lay[k] for k in ("rois", "fm_rois", "num_rois", "roi_cls")})
    with_layout["glb_max_num_roi"] = int(lay["num_rois"].max())
    assert _same(s.sample(with_layout), got, 1e-6, what="layout given") is True
    assert _same(s.sample(x), got, 1e-6, what="replay") is True
    # the oracle composition: box oracle (layout, bitwise above) -> text oracle -> shape oracle -> G oracle
    sd_g = {k: v.detach().cpu().clone() for k, v in g.state_dict().items()}
    ref_in = {k: (v.cpu() if torch.is_tensor(v) else [t.cpu() for t in v] if isinstance(v, list) else v)
              for k, v in with_layout.items()}
    with torch.no_grad():
        ref = oracle_box_sample(sd_g, ref_in)
    for i, (a, b) in enumerate(zip(_flat(got), _flat(ref))):
        close(a, b, 1e-3, f"output {i}")


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_box_graph_replay_mixed(engine, monkeypatch):
    """Caption-only batches interleaved with the three existing kinds (embeddings, captions + boxes with masks,
    generated shapes): every replay equals the eager pass bit for bit."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    s = _sampler()
    box_a = caption_only(2, 61, [18, 6])
    box_b = caption_only(2, 62, [4, 12], box_len=30)
    emb = synth.compact(synth.make_inputs(2, seed=61, parity=True))
    cap = caption_batch(2, 63, [12, 7], NTOK, NGLOVE, parity=True)
    gen = dict(emb)
    for k in ("bt_masks", "fm_bt_masks"):
        gen.pop(k)
    gen["noise_shp"] = torch.randn(2, 10, 320, generator=torch.Generator().manual_seed(64))
    batches = (box_a, emb, cap, gen, box_b)
    first = [s.sample(b) for b in batches]
    n_graphs, n_box = len(s._graphs), len(s._box_graphs)
    assert n_box == 2
    for _ in range(2):
        for b, f in zip(batches, first):
            assert _same(s.sample(b), f, 1e-6, what="replay") is True
            assert _same(s.sample_eager(b), f, 1e-6, what="eager") is True
    assert len(s._graphs) == n_graphs and len(s._box_graphs) == n_box
    other = dict(box_a, noise_box=_noise(2, 10, 99))
    assert _same(s.sample(other), s.sample_eager(other), 1e-6, what="other noise") is True


def test_sampler_box_graph_caption_widths():
    """Box captions of width 24 with max length 18, then a batch of the same B whose box stage reads its (width 18)
    captions: both map to the box graph of (B, 18), and each replay equals the eager box stage."""
    s = _sampler()
    wide = caption_only(2, 75, [18, 9])
    wide["box_captions"] = torch.cat([wide["captions"], torch.zeros(2, 6, dtype=torch.int64)], 1)
    wide["box_cap_lens"] = wide["cap_lens"].clone()
    narrow = caption_only(2, 76, [5, 18])
    assert wide["box_captions"].shape[1] == 24 and narrow["captions"].shape[1] == 18
    la = s.sample_layout(wide)
    lb = s.sample_layout(narrow)
    assert list(s._box_graphs) == [(2, 18)]
    for x, lay in ((wide, la), (narrow, lb), (wide, la)):
        again = s.sample_layout(x)
        assert all(torch.equal(torch.stack(again[k]) if k == "rois" else again[k],
                               torch.stack(lay[k]) if k == "rois" else lay[k]) for k in lay)
    eager = s._layout({k: v.to(DEV) for k, v in narrow.items() if k != "clabels_emb"}, eager=True)
    assert torch.equal(eager["labels"], lb["labels"]) and torch.equal(eager["fm_rois"], lb["fm_rois"])
    assert _same(s.sample(wide), s.sample_eager(wide), 1e-6, what="wide") is True


def test_sampler_eager_runs_box_stage_eagerly(monkeypatch):
    """sample_eager launches the box stage's kernels itself instead of replaying its graph."""
    s = _sampler()
    x = caption_only(2, 77, [6, 11])
    s.sample(x)
    assert len(s._box_graphs) == 1
    replays = []
    real = torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (replays.append(g), real(g))[1])
    s.sample_eager(x)
    assert replays == []
    s.sample(x)
    assert len(replays) == 2                           # the box graph, then the image graph


def test_sampler_all_empty_raises():
    s = _sampler()
    x = caption_only(2, 71, [5, 9])
    x["noise_box"][:] = 0.0
    bg = s.box_generator
    bg.mean_std = torch.tensor([[-500.0, 1.0]] * 4, dtype=torch.float64, device=DEV)   # every box invalid
    s._box_graphs.clear()
    lay = s.sample_layout(x)
    assert lay["num_rois"].tolist() == [0, 0]
    with pytest.raises(ValueError, match=r"samples \[0, 1\]"):
        s.sample(x)


def test_sampler_from_snapshot_box(tmp_path):
    g = _g_eval()
    blobs, l2i, _ = reference_checkpoints()
    d = tmp_path / "checkpoints" / "ck"
    d.mkdir(parents=True)
    (d / "model.pt").write_bytes(gzip.decompress(blobs["legacy"]))
    (d / "label_index2word.pt").write_bytes(blobs["label_index2word"])
    torch.save({k: v.cpu() for k, v in g.state_dict().items()}, tmp_path / "netG.pth")
    torch.save(shp_sd(), tmp_path / "netShpG.pth")
    torch.save({"module." + k: v for k, v in enc_sd().items()}, tmp_path / "text_encoder.pth")
    (tmp_path / "mean_std.txt").write_text("120.0 60.0\n110.0 55.0\n70.0 40.0\n1.0 0.5\n")
    cat_ids = [1, 3] + [c for c in range(5, 83)]
    np.save(tmp_path / "gaussian_dict.npy", {c: (3.0, 1.0) for c in cat_ids})
    s = GSampler.from_snapshot(str(tmp_path / "netG.pth"), device=DEV, shape_snapshot=str(tmp_path / "netShpG.pth"),
                               text_snapshot=str(tmp_path / "text_encoder.pth"), glove=_glove(),
                               box_checkpoint=str(d), mean_std=str(tmp_path / "mean_std.txt"),
                               gaussian_dict=str(tmp_path / "gaussian_dict.npy"), cat_ids=cat_ids)
    assert s.box_generator.label_to_class.tolist() == [-1, -1, -1, -1, 0, 1]
    x = caption_only(2, 81, [7, 11])
    x["noise_cnt"] = torch.randn(2, 80, generator=torch.Generator().manual_seed(2))
    lay = s.sample_layout(x)
    want = boxgen.BoxGenerator(_pre(), _frozen(boxgen.load_reference_decoder(str(d / "model.pt"))),
                               [[120.0, 60.0], [110.0, 55.0], [70.0, 40.0], [1.0, 0.5]], [[3.0, 1.0]] * 80,
                               [-1, -1, -1, -1, 0, 1])
    ref = want.sample(x["captions"].to(DEV), x["cap_lens"].to(DEV), 11, x["noise_box"].to(DEV),
                      x["noise_cnt"].to(DEV))
    for k in ("fm_rois", "num_rois", "roi_cls", "labels", "samples", "steps"):
        assert torch.equal(lay[k], ref[k]), k
    if int(lay["num_rois"].max()) > 0:
        assert all(torch.isfinite(t).all() for t in _flat(s.sample(x)))


def test_sampler_boxes_full_size():
    """Batch 16, untruncated box captions of up to 64 tokens, early_stop_len 10."""
    s = _sampler()
    x = caption_only(16, 91, ragged_lens(16, 18, 5).tolist(), box_len=64)
    lay = s.sample_layout(x)
    assert lay["labels"].shape == (16, 10) and int(lay["num_rois"].max()) >= 2
    got = s.sample(x)
    again = s.sample(x)
    assert all(torch.isfinite(t).all() for t in _flat(got))
    assert _same(again, got, 1e-6, what="B=16 replay") is True
    assert _same(s.sample_eager(x), got, 1e-6, what="B=16 eager") is True
