"""GPU tests of caption-conditioned sampling: og_lstm_bidir and RNN_ENCODER against the CPU oracle (oracle/text_oracle.py,
pinned to the reference's RNN_ENCODER by tests/test_text_encoder.py) and against the reference fixtures, bitwise
repeatability and batch-permutation invariance, the GloVe lookups / mask and class label embeddings, the whole
caption-driven GSampler.sample against the oracle composition (text oracle -> eval-mode G_NET, with ground-truth or
generated shapes), and graph replay."""
import pytest
import torch

import oracle_eval
from objgan_b200 import model, ops, synth
from objgan_b200.sampler import GSampler
from oracle import shape_oracle as S
from oracle import text_oracle as T
from test_gpu_sample import _flat, _same, close
from test_gpu_shape import _g_eval, _shp
from test_shape_gen import shp_sd
from test_text_encoder import (NTOK, TEXT_CASES, caption_batch, captions_for, cat_label_case, enc_sd, text_case,
                               text_fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]
NGLOVE = 70


def _enc(sd):
    net = model.RNN_ENCODER(sd["encoder.weight"].shape[0], nhidden=256)
    net.load_state_dict(sd, strict=True)
    net.to(DEV).eval()
    for p in net.parameters():
        p.requires_grad_(False)
    return net


def _glove(n=NGLOVE, seed=3):
    return 0.5 * torch.randn(n, 50, generator=torch.Generator().manual_seed(seed))


def ragged_lens(B, L, seed):
    """Unsorted lengths in [1, L], with 1 and L present when B allows."""
    lens = torch.randint(1, L + 1, (B,), generator=torch.Generator().manual_seed(seed))
    lens[B // 2] = L
    if B > 1:
        lens[B - 1] = 1
    return lens


# ---------------------------------------------------------------------------------------------------------------------
# the recurrence and the encoder
# ---------------------------------------------------------------------------------------------------------------------
def test_lstm_bidir_kernel_vs_loop():
    """og_lstm_bidir alone on seeded gate inputs against an explicit per-sample loop."""
    g = torch.Generator().manual_seed(8)
    B, L, H = 6, 9, 128
    lens = torch.tensor([9, 1, 4, 9, 2, 7])
    gx = torch.randn(B * L, 8 * H, generator=g)
    whh = [0.1 * torch.randn(4 * H, H, generator=g) for _ in range(2)]
    words, sent = ops.lstm_bidir(gx.to(DEV), whh[0].to(DEV), whh[1].to(DEV), lens.to(DEV), L)
    want = torch.zeros(B, 2 * H, L)
    want_s = torch.zeros(B, 2 * H)
    for d in range(2):
        for b in range(B):
            h, c = torch.zeros(H), torch.zeros(H)
            n = int(lens[b])
            for t in (range(n - 1, -1, -1) if d else range(n)):
                z = gx[b * L + t, d * 4 * H:(d + 1) * 4 * H] + whh[d] @ h
                i, f, gg, o = z.chunk(4)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
                h = torch.sigmoid(o) * torch.tanh(c)
                want[b, d * H:(d + 1) * H, t] = h
            want_s[b, d * H:(d + 1) * H] = h
    close(words, want, 1e-5, "words")
    close(sent, want_s, 1e-5, "sent")
    for b in range(B):
        assert words[b, :, int(lens[b]):].abs().max().item() == 0 if lens[b] < L else True


@pytest.mark.parametrize("L", [1, 12, 18])
@pytest.mark.parametrize("B", [1, 5, 16, 64, 65])
def test_rnn_encoder_vs_oracle(B, L):
    sd = enc_sd()
    enc = _enc(sd)
    lens = ragged_lens(B, L, 100 * B + L)
    caps, _ = captions_for(lens, 18, NTOK, B + L)
    words_ref, sent_ref = T.rnn_encoder_forward(sd, caps, lens, L)
    cd, ld = caps.to(DEV), lens.to(DEV)
    words, sent = enc(cd, ld, L)
    close(words, words_ref, 1e-5, "words_emb")
    close(sent, sent_ref, 1e-5, "sent_emb")
    w = words.cpu()
    for b in range(B):                                 # the columns past each caption are exactly zero
        n = int(lens[b])
        assert n == L or w[b, :, n:].abs().max().item() == 0
    again = enc(cd, ld, L)
    assert torch.equal(again[0], words) and torch.equal(again[1], sent)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(B))
    pw, ps = enc(cd[perm.to(DEV)], ld[perm.to(DEV)], L)
    assert torch.equal(pw, words[perm.to(DEV)]) and torch.equal(ps, sent[perm.to(DEV)])
    if B > 1:                                          # a sample alone gives what it gives inside the batch
        one = enc(cd[B // 2:B // 2 + 1], ld[B // 2:B // 2 + 1], L)
        assert torch.equal(one[0][0], words[B // 2]) and torch.equal(one[1][0], sent[B // 2])


@pytest.mark.parametrize("name", list(TEXT_CASES))
def test_rnn_encoder_vs_reference_fixture(name):
    want = text_fixture(name)
    caps, lens, max_len = text_case(name)
    words, sent = _enc(enc_sd())(caps.to(DEV), lens.to(DEV), max_len)
    from test_text_encoder import WORDS_CAP, _close
    _close(words.cpu(), want["words"], 1e-5, WORDS_CAP)
    _close(sent.cpu(), want["sent"], 1e-5, WORDS_CAP)


def test_text_inputs_and_class_labels():
    caps, lens = captions_for([5, 18, 1], 18, NTOK, 2)
    gcaps, _ = captions_for([5, 18, 1], 18, NGLOVE, 3)
    glove = _glove()
    gw, mask = ops.text_inputs(caps.to(DEV), gcaps.to(DEV), glove.to(DEV), 14)
    gw_ref, mask_ref = T.text_inputs(caps, gcaps, glove, 14)
    assert torch.equal(gw.cpu(), gw_ref) and torch.equal(mask.cpu(), mask_ref)
    glove, labels, lens, order, want = cat_label_case()
    got = ops.class_label_emb(glove.to(DEV), labels.to(DEV), lens.to(DEV), order.to(DEV))
    assert torch.equal(got.cpu(), want)


# ---------------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------------
def oracle_caption_sample(sd_g, sd_e, glove, x, sd_s=None):
    """text oracle -> (shape oracle -> form_hmaps) -> eval-mode G_NET oracle."""
    n = int(x["cap_lens"].max())
    words, sent = T.rnn_encoder_forward(sd_e, x["captions"], x["cap_lens"], n)
    gw, mask = T.text_inputs(x["captions"], x["glove_captions"], glove, n)
    inp = synth.make_inputs(x["z"].shape[0], seed=x["_seed"], parity=True)
    inp.update(words_embs=words, sent_emb=sent, glove_words_embs=gw, mask=mask, z=x["z"], eps=x["eps"])
    if sd_s is not None:
        r = int(x["glb_max_num_roi"])
        fwd, bwd, fm = S.bbox_maps(x["rois"][0], x["fm_rois"], x["num_rois"], r, 80)
        raw = S.shp_g_net_forward(sd_s, x["noise_shp"][:, :r], fwd, bwd, fm)
        hm, bt, fmb = S.form_hmaps(raw[:, :, 0], x["num_rois"], x["roi_cls"])
        inp.update(hmaps=hm, bt_masks=bt, fm_bt_masks=fmb)
    return oracle_eval.g_net_forward_eval(sd_g, inp), (words, sent, mask, gw)


@pytest.mark.parametrize("gen", [False, True])
@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_captions_vs_oracle(engine, gen, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    g = _g_eval()
    sd_g = {k: v.detach().cpu().clone() for k, v in g.state_dict().items()}
    sd_e, sd_s, glove = enc_sd(), shp_sd(), _glove()
    s = GSampler(g, _shp(sd_s) if gen else None, text_encoder=_enc(sd_e), glove=glove)
    x = caption_batch(3, 33, [9, 14, 3], NTOK, NGLOVE, parity=True)
    x["_seed"] = 33
    if gen:
        for k in ("bt_masks", "fm_bt_masks"):
            x.pop(k)
        x["noise_shp"] = torch.randn(3, 10, 320, generator=torch.Generator().manual_seed(33))
    with torch.no_grad():
        ref, (words, sent, mask, gw) = oracle_caption_sample(sd_g, sd_e, glove, x, sd_s if gen else None)
    enc = s.encode_text(x)
    close(enc["words_embs"], words, 1e-5, "words_embs")
    close(enc["sent_emb"], sent, 1e-5, "sent_emb")
    assert torch.equal(enc["mask"].cpu(), mask) and torch.equal(enc["glove_words_embs"].cpu(), gw)
    got = s.sample(x)
    for i, (a, b) in enumerate(zip(_flat(got), _flat(ref))):
        close(a, b, 1e-3, f"output {i}")
    assert _same(s.sample(x), got, 1e-6, what="replay") is True


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_caption_graph_replay_mixed(engine, monkeypatch):
    """Caption batches of two max_len and an embedding batch, interleaved: every replay equals the eager pass bit for
    bit, and each max_len has its own graph."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    s = GSampler(_g_eval(), text_encoder=_enc(enc_sd()), glove=_glove())
    ca = caption_batch(2, 61, [18, 6], NTOK, NGLOVE, parity=True)
    ca2 = caption_batch(2, 62, [4, 18], NTOK, NGLOVE, parity=True)
    cb = caption_batch(2, 63, [12, 7], NTOK, NGLOVE, parity=True)
    emb = synth.compact(synth.make_inputs(2, seed=61, parity=True))
    first = [s.sample(b) for b in (ca, emb, cb)]
    assert len(s._graphs) == 3
    for _ in range(2):
        for b, f in zip((ca, emb, cb), first):
            assert _same(s.sample(b), f, 1e-6, what="replay") is True
        assert _same(s.sample(ca2), s.sample_eager(ca2), 1e-6, what="replay, other captions") is True
    assert len(s._graphs) == 3
    assert not torch.equal(s.sample(ca)[0][0], s.sample(ca2)[0][0])


def test_sampler_from_snapshot_text(tmp_path):
    g = _g_eval()
    sd_e, glove = enc_sd(), _glove()
    torch.save({k: v.cpu() for k, v in g.state_dict().items()}, tmp_path / "netG.pth")
    torch.save({"module." + k: v for k, v in sd_e.items()}, tmp_path / "text_encoder.pth")
    labels, lens, order = torch.tensor([[5, 6, 7], [8, 9, 0]] + [[k % 60 + 1, 0, 0] for k in range(78)]), \
        torch.tensor([3, 2] + [1] * 78), torch.arange(80).flip(0)
    s = GSampler.from_snapshot(str(tmp_path / "netG.pth"), device=DEV, text_snapshot=str(tmp_path / "text_encoder.pth"),
                               glove=glove, cat_labels=labels, cat_label_lens=lens, cat_label_order=order)
    clabels = T.prepare_cat_emb(glove, labels, lens, order)
    assert torch.equal(s.clabels_emb.cpu(), clabels)
    x = caption_batch(2, 71, [10, 3], NTOK, NGLOVE, parity=True)
    want = GSampler(g, text_encoder=_enc(sd_e), glove=glove)
    with_c = dict(x, clabels_emb=clabels)
    x.pop("clabels_emb")                               # the sampler's own label embeddings stand in
    _same(s.sample(x), want.sample(with_c), 1e-6, what="from_snapshot")
    _same(s.sample(x), want.sample_eager(with_c), 1e-6, what="from_snapshot, replayed")
    with pytest.raises(ValueError, match="no text encoder"):
        GSampler(g).sample(x)


def test_sampler_captions_full_size():
    """Batch 16, WORDS_NUM = 18, 10 rois per image and a vocabulary of 30,000 tokens."""
    sd = {k: v for k, v in enc_sd(30000).items()}
    glove = _glove(30000, 4)
    s = GSampler(_g_eval(), text_encoder=_enc(sd), glove=glove)
    lens = ragged_lens(16, 18, 5)
    x = caption_batch(16, 91, lens, 30000, 30000)
    assert x["glb_max_num_roi"] == 10 and x["captions"].max() > 20000
    s.sample(x)
    got = s.sample(x)
    assert all(torch.isfinite(t).all() for t in _flat(got))
    _same(got, s.sample_eager(x), 1e-6, what="B=16 captions")
    enc = s.encode_text(x)
    words, sent = T.rnn_encoder_forward(sd, x["captions"], x["cap_lens"], 18)
    close(enc["words_embs"], words, 1e-5, "words_embs")
    close(enc["sent_emb"], sent, 1e-5, "sent_emb")
