"""Text encoder for caption-conditioned sampling (CPU): the oracle's RNN_ENCODER forward (oracle/text_oracle.py) against
the reference's own module, the state_dict layout and loading, the inference-only and unsupported-configuration errors,
GSampler's caption input checks, prepare_cat_emb on hand-worked labels, and the library calls of the text stage
(DRY_RUN: host logic only).

The reference side is stored in tests/golden/reference/rnn_encoder_*.npz and rnn_encoder_layout.json.  Re-record with
the reference importable (tests/refimport.py):

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_text_encoder.py
"""
import hashlib
import json
import os

import pytest
import torch

import reference_fixtures as fixtures
import refimport
from dry import dry, record  # noqa: F401
from objgan_b200 import model, ops, synth
from objgan_b200.config import cfg
from objgan_b200.sampler import GSampler, strip_module_prefix
from oracle import text_oracle as T

NTOK = 60               # vocabulary of the recorded cases
WORDS_CAP = 4096        # stored elements per words_emb
# name -> (cap_lens, caption width, max_len); the reference needs the lengths sorted (testDataset.py:120-145)
TEXT_CASES = {"B1": ([11], 18, 11), "B5": ([18, 14, 9, 3, 1], 18, 18), "B3_pad": ([12, 7, 2], 18, 15)}


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fixtures
# ---------------------------------------------------------------------------------------------------------------------
_sd = {}


def enc_sd(ntoken=NTOK):
    """state_dict of objgan_b200's RNN_ENCODER(ntoken, nhidden=256) under torch.manual_seed(0)."""
    if ntoken not in _sd:
        torch.manual_seed(0)
        net = model.RNN_ENCODER(ntoken, nhidden=cfg.TEXT.EMBEDDING_DIM)
        _sd[ntoken] = {k: v.clone() for k, v in net.state_dict().items()}
    return {k: v.clone() for k, v in _sd[ntoken].items()}


def captions_for(lens, width, ntoken, seed):
    """(B, width) int64 token ids in [1, ntoken) for t < lens[b], 0 (the padding id) after."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.as_tensor(lens, dtype=torch.int64)
    ids = torch.randint(1, ntoken, (lens.shape[0], width), generator=g)
    return ids * (torch.arange(width).view(1, -1) < lens.view(-1, 1)), lens


def text_case(name):
    lens, width, max_len = TEXT_CASES[name]
    caps, lens = captions_for(lens, width, NTOK, 900 + len(lens))
    return caps, lens, max_len


def text_fixture(name):
    def produce():
        ref = refimport.load()
        caps, lens, max_len = text_case(name)
        net = ref.model.RNN_ENCODER(NTOK, nhidden=256)
        net.load_state_dict(enc_sd(), strict=True)
        net.eval()
        with torch.no_grad():
            words, sent = net(caps, lens, max_len)
        return {"in__captions": caps, "in__cap_lens": lens, "words": words, "sent": sent,
                "words_absmax": words.abs().max()}
    return fixtures.recorded(f"rnn_encoder_{name}", produce, cap=WORDS_CAP)


def _layout(state_dict):
    return hashlib.sha256(json.dumps([[k, list(v.shape), str(v.dtype)] for k, v in state_dict.items()]).encode()).hexdigest()


def enc_layout():
    """{"state": sha256 of (key, shape, dtype) in order, "keys": [[key, shape]]} of the reference's
    RNN_ENCODER(NTOK, nhidden=256)."""
    path = os.path.join(fixtures.GOLD, "rnn_encoder_layout.json")
    if fixtures.RECORD:
        sd = refimport.load().model.RNN_ENCODER(NTOK, nhidden=256).state_dict()
        json.dump({"state": _layout(sd), "keys": [[k, list(v.shape)] for k, v in sd.items()]}, open(path, "w"), indent=0)
    return json.load(open(path))


def _close(a, b, tol, cap):
    """a (full tensor) against the stored sample b, within tol of max|b|."""
    a = torch.from_numpy(fixtures.sample(a, cap)).reshape(-1)
    b = torch.as_tensor(b).float().reshape(-1)
    assert a.numel() == b.numel() and torch.isfinite(a).all()
    err = (a - b).abs().max().item()
    assert err <= tol * max(b.abs().max().item(), 1e-12), err


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(TEXT_CASES))
def test_rnn_encoder_oracle_matches_reference(name):
    want = text_fixture(name)
    caps, lens, max_len = text_case(name)
    assert torch.equal(caps.float(), want["in__captions"]) and torch.equal(lens.float(), want["in__cap_lens"])
    words, sent = T.rnn_encoder_forward(enc_sd(), caps, lens, max_len)
    assert words.shape == (len(lens), 256, max_len) and sent.shape == (len(lens), 256)
    _close(words, want["words"], 1e-5, WORDS_CAP)
    _close(sent, want["sent"], 1e-5, WORDS_CAP)
    assert abs(words.abs().max().item() - float(want["words_absmax"])) <= 1e-6
    for b, n in enumerate(lens.tolist()):                  # zero columns past each caption, exactly
        assert words[b, :, n:].abs().max() == 0 if n < max_len else True
    # sent_emb = [forward h after the last token, backward h after token 0]
    assert torch.equal(sent[:, :128], words[torch.arange(len(lens)), :128, lens - 1])
    assert torch.equal(sent[:, 128:], words[:, 128:, 0])


def test_rnn_encoder_oracle_is_per_sample():
    """The oracle runs every sample on its own: an unsorted batch gives each sample the result it has alone."""
    caps, lens = captions_for([3, 18, 1, 9], 18, NTOK, 5)
    words, sent = T.rnn_encoder_forward(enc_sd(), caps, lens, 18)
    for b in range(4):
        w1, s1 = T.rnn_encoder_forward(enc_sd(), caps[b:b + 1], lens[b:b + 1], 18)
        assert torch.equal(w1[0], words[b]) and torch.equal(s1[0], sent[b])


# ---------------------------------------------------------------------------------------------------------------------
# module API
# ---------------------------------------------------------------------------------------------------------------------
def test_rnn_encoder_state_dict_matches_reference():
    ref = enc_layout()
    net = model.RNN_ENCODER(NTOK, nhidden=256)
    sd = net.state_dict()
    assert _layout(sd) == ref["state"]
    assert [[k, list(v.shape)] for k, v in sd.items()] == ref["keys"]
    assert [k for k, _ in ref["keys"]][:2] == ["encoder.weight", "rnn.weight_ih_l0"]
    other = {k: torch.randn(v.shape) for k, v in sd.items()}
    net.load_state_dict(strip_module_prefix({"module." + k: v for k, v in other.items()}), strict=True)
    assert all(torch.equal(net.state_dict()[k], v) for k, v in other.items())
    net.load_state_dict(strip_module_prefix(other), strict=True)
    with pytest.raises(RuntimeError):
        net.load_state_dict(strip_module_prefix({"module." + k: v for k, v in list(other.items())[1:]}), strict=True)


def test_text_snapshot_loads_with_and_without_module_prefix(dry, tmp_path):
    torch.save(model.G_NET(80).state_dict(), tmp_path / "netG.pth")
    sd = enc_sd(75)
    torch.save({"module." + k: v for k, v in sd.items()}, tmp_path / "text_encoder.pth")
    torch.save(sd, tmp_path / "text_encoder_bare.pth")
    for name in ("text_encoder.pth", "text_encoder_bare.pth"):
        s = GSampler.from_snapshot(str(tmp_path / "netG.pth"), device="cpu", text_snapshot=str(tmp_path / name),
                                   glove=torch.randn(40, 50))
        assert s.text_encoder.ntoken == 75 and not s.text_encoder.training
        got = s.text_encoder.state_dict()
        assert all(torch.equal(got[k], v) for k, v in sd.items()), name
        assert not any(p.requires_grad for p in s.text_encoder.parameters())
    assert GSampler.from_snapshot(str(tmp_path / "netG.pth"), device="cpu").text_encoder is None


def test_inference_only_and_unsupported(dry):
    net = model.RNN_ENCODER(NTOK, nhidden=256)
    caps, lens = captions_for([4, 2], 18, NTOK, 1)
    with pytest.raises(RuntimeError, match=r"call \.eval\(\)"):
        net(caps, lens, 4)
    net.eval()
    with pytest.raises(RuntimeError, match="inference only"):
        net(caps, lens, 4)
    with torch.no_grad():
        words, sent = net(caps, lens, 4)
    assert words.shape == (2, 256, 4) and sent.shape == (2, 256)
    for p in net.parameters():
        p.requires_grad_(False)
    assert net(caps, lens, 4)[0].shape == (2, 256, 4)
    with pytest.raises(NotImplementedError):
        model.RNN_ENCODER(NTOK, nlayers=2)
    with pytest.raises(NotImplementedError):
        model.RNN_ENCODER(NTOK, bidirectional=False)
    saved = cfg.RNN_TYPE
    cfg.RNN_TYPE = "GRU"
    try:
        with pytest.raises(NotImplementedError):
            model.RNN_ENCODER(NTOK)
    finally:
        cfg.RNN_TYPE = saved


def caption_batch(B, seed, lens, ntoken, nglove, **kw):
    """A compact batch whose words come from captions: ``captions`` / ``glove_captions`` (B, WORDS_NUM) with the padding
    id 0 past ``lens`` (unsorted allowed), and no words_embs / sent_emb / glove_words_embs / mask."""
    x = synth.compact(synth.make_inputs(B, seed=seed, **kw))
    for k in ("words_embs", "sent_emb", "glove_words_embs", "mask"):
        x.pop(k)
    x["captions"], x["cap_lens"] = captions_for(lens, cfg.TEXT.WORDS_NUM, ntoken, seed)
    x["glove_captions"], _ = captions_for(lens, cfg.TEXT.WORDS_NUM, nglove, seed + 1)
    return x


def _text_sampler(**kw):
    enc = model.RNN_ENCODER(NTOK, nhidden=256)
    return GSampler(model.G_NET(80), text_encoder=enc, glove=torch.randn(40, 50), **kw)


def test_sampler_caption_input_checks(dry):
    s = _text_sampler()
    good = caption_batch(2, 3, [5, 18], NTOK, 40)
    key = GSampler._key(s._prepare(good))
    assert key[1] == 18 and key[4:] == (True, False)
    cases = [("cap_lens", torch.tensor([0, 3]), "cap_lens"), ("cap_lens", torch.tensor([19, 3]), "cap_lens"),
             ("captions", None, "caption token ids"), ("glove_captions", None, "GloVe token ids")]
    for key, val, msg in cases:
        bad = dict(good)
        if val is None:
            bad[key] = good[key].clone()
            bad[key][1, 0] = NTOK if key == "captions" else 40
        else:
            bad[key] = val
        with pytest.raises(ValueError, match=msg):
            s.sample_eager(bad)
        neg = dict(good)
        if val is None:
            neg[key] = good[key].clone()
            neg[key][0, 1] = -1
            with pytest.raises(ValueError, match=msg):
                s.sample_eager(neg)
    with pytest.raises(ValueError, match="no text encoder"):
        GSampler(model.G_NET(80)).sample_eager(good)
    with pytest.raises(ValueError, match="no text encoder"):
        GSampler(model.G_NET(80)).encode_text(good)


def _trace(fn):
    return [name for name, _ in record(fn)]


@pytest.mark.parametrize("lens", [[1], [7, 18, 3, 1, 12]])
def test_text_stage_call_sequence(dry, lens):
    """The text stage is four library calls whatever B and max_len: the token lookup, the x-part of the gates of both
    directions for all steps, the recurrence, and the GloVe lookups + mask; the padded weight copies are made once."""
    s = _text_sampler()
    x = caption_batch(len(lens), 4, lens, NTOK, 40)
    first = _trace(lambda: s.encode_text(x))
    assert first.count("og_zero_bytes") == 1 and first.count("og_add") == 2 and first.count("og_pack_weights") == 1
    calls = _trace(lambda: s.encode_text(x))
    assert calls == ["og_gather_rows", "og_conv2d_simt", "og_lstm_bidir", "og_text_inputs"]
    out = s.encode_text(x)
    n = max(lens)
    assert out["words_embs"].shape == (len(lens), 256, n) and out["sent_emb"].shape == (len(lens), 256)
    assert out["mask"].shape == (len(lens), n) and out["mask"].dtype == torch.bool
    assert out["glove_words_embs"].shape == (len(lens), 50, n)
    full = _trace(lambda: s.sample_eager(x))
    i = full.index("og_lstm_bidir")                 # the text stage runs inside the same forward, once
    assert full[i - 2:i + 2] == calls and full.count("og_lstm_bidir") == 1 and i < full.index("og_words_proj")
    with torch.no_grad():
        s.text_encoder.rnn.bias_hh_l0.add_(1.0)       # a weight change refreshes the derived copies
    again = _trace(lambda: s.encode_text(x))
    assert again == ["og_zero_bytes", "og_copy_channels", "og_add", "og_add", "og_gather_rows", "og_pack_weights",
                     *calls[1:]]


def test_sampler_caption_key_and_clabels(dry):
    clabels = torch.randn(80, 50)
    s = _text_sampler(clabels_emb=clabels)
    x = caption_batch(3, 6, [4, 9, 2], NTOK, 40)
    x.pop("clabels_emb")
    dev = s._prepare(x)
    assert dev["slabels_feat"].shape == (3, 50, x["glb_max_num_roi"], 1)     # built from the sampler's clabels_emb
    key = GSampler._key(dev)
    assert key[0] == 3 and key[1] == 9 and key[4:] == (True, False)
    assert all(k not in dev for k in ("words_embs", "sent_emb", "glove_words_embs", "mask"))
    emb = synth.compact(synth.make_inputs(3, seed=6))
    assert GSampler._key(s._prepare(emb))[4:] == (False, False)


# ---------------------------------------------------------------------------------------------------------------------
# prepare_cat_emb
# ---------------------------------------------------------------------------------------------------------------------
def cat_label_case():
    """Five labels sorted by length (3, 2, 2, 1, 1 tokens) over a GloVe table of exactly representable values, the
    resort order of load.py:346, and the hand-worked result: 3-token labels are zero rows, 2-token ones the mean."""
    glove = torch.arange(8 * 4, dtype=torch.float32).view(8, 4) / 4.0
    labels = torch.tensor([[1, 2, 3], [4, 5, 0], [6, 1, 0], [7, 0, 0], [3, 0, 0]])
    lens = torch.tensor([3, 2, 2, 1, 1])
    order = torch.tensor([3, 0, 4, 2, 1])
    rows = [torch.zeros(4), (glove[4] + glove[5]) / 2, (glove[6] + glove[1]) / 2, glove[7], glove[3]]
    want = torch.stack([rows[k] for k in order.tolist()])
    return glove, labels, lens, order, want


def test_prepare_cat_emb_hand_worked():
    glove, labels, lens, order, want = cat_label_case()
    got = T.prepare_cat_emb(glove, labels, lens, order)
    assert torch.equal(got, want)
    assert torch.equal(want[1], torch.zeros(4)) and torch.equal(want[0], glove[7])
    assert torch.equal(want[4], torch.tensor([4.5, 4.75, 5.0, 5.25]))   # (glove[4] + glove[5]) / 2


def test_class_label_emb_checks():
    glove, labels, lens, order, _ = cat_label_case()
    with pytest.raises(ValueError, match="GloVe table"):
        ops.class_label_emb(glove[:5], labels, lens, order)
    with pytest.raises(ValueError, match="cat_label_order"):
        ops.class_label_emb(glove, labels, lens, torch.tensor([0, 1, 2, 3, 5]))
    with pytest.raises(ValueError, match="cat_label_lens"):
        ops.class_label_emb(glove, labels[:, :1], torch.tensor([2, 1, 1, 1, 1]), order)
