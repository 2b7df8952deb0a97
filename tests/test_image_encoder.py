"""DAMSM image encoder (CPU): the oracle's CNN_ENCODER forward and input gradient (oracle/image_encoder_oracle.py)
against the reference's own module, the state_dict layout and loading, the eval-only / frozen guards, the library
calls of one forward (DRY_RUN: host logic only) and the R-precision pooling.

The reference side is stored in tests/golden/reference/cnn_encoder_*.npz and cnn_encoder_layout.json.  Re-record with
the reference and torchvision importable (tests/refimport.py):

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_image_encoder.py
"""
import json
import os
from unittest import mock

import pytest
import torch

import reference_fixtures as fixtures
import refimport
from objgan_b200 import lib, losses, model
from oracle import image_encoder_oracle as E

LAYOUT = os.path.join(fixtures.GOLD, "cnn_encoder_layout.json")
CASES = {"B2_256": (2, 256), "B1_200": (1, 200)}

_sd = []


def enc_sd():
    """The test weights (oracle.test_state_dict over CNN_ENCODER's keys), fixed by their seed."""
    if not _sd:
        _sd.append(E.test_state_dict(model.CNN_ENCODER(256).state_dict(), seed=0))
    return {k: v.clone() for k, v in _sd[0].items()}


def case_inputs(name):
    b, s = CASES[name]
    g = torch.Generator().manual_seed(100 + s)
    x = torch.rand(b, 3, s, s, generator=g) * 2 - 1
    a = torch.randn(b, 256, 17, 17, generator=g)       # L = <a, features> + <c, cnn_code>
    c = torch.randn(b, 256, generator=g)
    return x, a, c


def _reference_encoder():
    R = refimport.load()
    import torchvision
    R.cfg.TRAIN.FLAG = True
    R.cfg.TRAIN.NET_E = "text_encoder100.pth"
    torch.manual_seed(0)
    imagenet = torchvision.models.inception_v3(init_weights=True, aux_logits=True).state_dict()
    with mock.patch("torch.load", lambda *a, **k: imagenet):     # the ImageNet file the constructor reads
        net = R.model.CNN_ENCODER(256)
    return net


def encoder_fixture(name):
    def produce():
        net = _reference_encoder()
        net.load_state_dict(enc_sd(), strict=True)
        net.eval()
        x, a, c = case_inputs(name)
        x.requires_grad_(True)
        f, code = net(x)
        ((f * a).sum() + (code * c).sum()).backward()
        return {"features": f, "code": code, "grad": x.grad}
    return fixtures.recorded(f"cnn_encoder_{name}", produce, cap=4096)


def oracle_case(name, dtype=torch.float64):
    x, a, c = case_inputs(name)
    sd = {k: v.to(dtype) if v.is_floating_point() else v for k, v in enc_sd().items()}
    x = x.to(dtype).requires_grad_(True)
    f, code = E.cnn_encoder_forward(sd, x)
    ((f * a.to(dtype)).sum() + (code * c.to(dtype)).sum()).backward()
    return f.detach(), code.detach(), x.grad


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    ref = encoder_fixture(name)
    f, code, grad = oracle_case(name, torch.float32)      # same precision: a max-pool argmax can flip in float64
    for key, t in (("features", f), ("code", code), ("grad", grad)):
        assert _rel(torch.from_numpy(fixtures.sample(t.float(), 4096)), ref[key]) <= 1e-5, key


def test_oracle_activations_stay_order_one():
    x, _, _ = case_inputs("B1_200")
    stats = []
    with torch.no_grad():
        E.cnn_encoder_forward(enc_sd(), x, stats)
    assert len(stats) == 94
    m = [v for _, v in stats]
    assert min(m) > 0.3 and max(m) < 20, (min(m), max(m))


def test_state_dict_layout_matches_reference():
    if fixtures.RECORD:
        net = _reference_encoder()
        with open(LAYOUT, "w") as f:
            json.dump({k: list(v.shape) for k, v in net.state_dict().items()}, f, indent=0)
    layout = json.load(open(LAYOUT))
    ours = {k: list(v.shape) for k, v in model.CNN_ENCODER(256).state_dict().items()}
    assert ours == layout
    assert sum(1 for k in layout if k.endswith(".conv.weight")) == 94


@pytest.mark.parametrize("prefix", ["", "module."])
@pytest.mark.parametrize("with_nbt", [True, False])
def test_load_variants(prefix, with_nbt):
    sd = {prefix + k: v for k, v in enc_sd().items() if with_nbt or not k.endswith("num_batches_tracked")}
    net = model.CNN_ENCODER(256)
    net.load_state_dict(sd, strict=True)
    assert torch.equal(net.Mixed_6e.branch7x7dbl_3.conv.weight, enc_sd()["Mixed_6e.branch7x7dbl_3.conv.weight"])
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop(prefix + "emb_features.weight")
        net.load_state_dict(bad, strict=True)


def test_guards():
    net = model.CNN_ENCODER(256)
    x = torch.zeros(1, 3, 64, 64)
    net.train()
    with pytest.raises(RuntimeError, match="eval mode only"):
        net(x)
    net.eval()
    net.Mixed_5b.branch1x1.conv.weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="frozen"):
        net(x)


def test_dry_run_call_sequence():
    """One forward issues a fixed list of library calls and no torch compute; with the input requiring grad the
    backward adds the input-gradient calls."""
    net = model.CNN_ENCODER(256)
    prog = net.program()
    convs = [st for st in prog.steps if st[0] == "conv"]
    # 94 BasicConv2d + emb_features, with 11 groups of sibling 1x1 convs fused (3 x 3 + 4 x 3 + 2 + 2 x 3 -> 11)
    assert sum(len(st[1].weights) for st in convs) == 95
    assert len(convs) == 95 - (3 * 2 + 4 * 2 + 1 + 2 * 2)
    lib.DRY_RUN = True
    try:
        first = lib.get().launches
        net(torch.zeros(2, 3, 256, 256))                     # folds BatchNorm and packs the weights
        first = lib.get().launches - first
        n0 = lib.get().launches
        with mock.patch("torch.nn.functional.conv2d", side_effect=AssertionError("torch compute")):
            f, code = net(torch.zeros(2, 3, 256, 256))
        fwd = lib.get().launches - n0
        assert first - fwd >= 94                             # one og_bn_fold per BasicConv2d, once
        assert f.shape == (2, 256, 17, 17) and code.shape == (2, 256)
        x = torch.zeros(2, 3, 256, 256, requires_grad=True)
        n0 = lib.get().launches
        f, code = net(x)
        (f.sum() + code.sum()).backward()
        assert x.grad.shape == x.shape
        assert lib.get().launches - n0 > 2 * fwd          # the input gradient costs more calls than the forward
    finally:
        lib.DRY_RUN = False


class _RecordingRP(losses.RPrecision):
    def _score(self):
        self.scored.append([int(c[0, 0]) for c in self.sets["cnn_code"]])


def test_rprecision_pooling_hand_worked():
    """7 batches of 16 fill a pool of 100 (112 >= 100); the 8th scores the pool and is dropped; the 9th starts the
    next pool."""
    rp = _RecordingRP(100)
    rp.scored = []
    for i in range(1, 17):
        code = torch.full((16, 4), float(i))
        rp.add(torch.zeros(16, 4, 17, 17), code, torch.zeros(16, 4, 5), torch.zeros(16, 4), [5] * 16)
        if i == 8:
            assert rp.scored == [[1, 2, 3, 4, 5, 6, 7]] and rp.count == 0
        if i == 9:
            assert rp.count == 16
    assert rp.scored == [[1, 2, 3, 4, 5, 6, 7], [9, 10, 11, 12, 13, 14, 15]]


def test_rprecision_pool_cut_and_padding():
    rp = losses.RPrecision(10)
    for i, width in enumerate((3, 6)):
        lens = [width if j == 0 else 2 for j in range(8)]
        rp.add(torch.zeros(8, 4, 17, 17), torch.full((8, 4), float(i)), torch.ones(8, 4, width), torch.zeros(8, 4),
               lens)
    pool = rp._pool()
    assert pool["cnn_code"].shape == (10, 4) and pool["words_embs"].shape == (10, 4, 6)
    assert pool["words_embs"][0, 0, 3:].abs().sum() == 0 and pool["words_embs"][8, 0].sum() == 6


# ---------------------------------------------------------------------------------------------------------------------
# R-precision at the evaluator's pool size (cfg.TEST.RP_POOL_SIZE = 100): 100 x 100 image-caption pairs
# ---------------------------------------------------------------------------------------------------------------------
def pool_case(seed=2024, n=100, T=12):
    """A seeded pool of n samples whose region features and image codes are noisy copies of their own caption's words
    and sentence embedding (accuracies near 45 %, far from both chance and 100 %); class ids repeat, so the
    same-class mask is exercised.  Returns (region (n, 256, 17, 17), code, words (n, 256, T), sent, cap_lens,
    class_ids)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(3, T + 1, (n,), generator=g)
    words = torch.randn(n, 256, T, generator=g) * (torch.arange(T).view(1, 1, T) < lens.view(n, 1, 1))
    idx = (torch.arange(289).view(1, 289) % lens.view(n, 1)).view(n, 1, 289).expand(n, 256, 289)
    region = torch.gather(words, 2, idx) + 25.0 * torch.randn(n, 256, 289, generator=g)
    sent = torch.randn(n, 256, generator=g)
    code = sent + 8.0 * torch.randn(n, 256, generator=g)
    cls = torch.randint(0, 60, (n,), generator=g).numpy()
    return region.view(n, 256, 17, 17), code, words, sent, lens, cls


def rprecision_fixture():
    """The reference's words_loss / sent_loss(is_training=False) accuracies on pool_case() (evaluator.py:401-405)."""
    def produce():
        R = refimport.load(words_num=12)
        region, code, words, sent, lens, cls = pool_case()
        labels = torch.arange(100)
        import numpy as np
        # torch 2's masked_fill_ needs a boolean mask: the reference's ByteTensor of its 0/1 numpy mask, as bool
        with mock.patch("torch.ByteTensor", lambda a: torch.from_numpy(np.asarray(a)).bool()):
            w = R.losses.words_loss(region, words, labels, lens, cls, 100, is_training=False)[3]
            s = R.losses.sent_loss(code, sent, labels, cls, 100, is_training=False)[2]
        return {"w_accuracy": float(w), "s_accuracy": float(s)}
    return fixtures.recorded("rprecision_pool100", produce)


def test_rprecision_pool100_oracle_matches_reference():
    from oracle import objgan_oracle as O
    ref = rprecision_fixture()
    region, code, words, sent, lens, cls = pool_case()
    w = O.words_loss(region, words, torch.arange(100), lens.tolist(), cls, 100)[3]
    s = O.sent_loss(code, sent, torch.arange(100), cls, 100)[2]
    assert 20 < float(ref["w_accuracy"]) < 80 and 20 < float(ref["s_accuracy"]) < 80
    assert float(w) == float(ref["w_accuracy"]) and float(s) == float(ref["s_accuracy"])
