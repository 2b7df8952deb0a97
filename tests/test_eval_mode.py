"""Eval-mode BatchNorm (CPU): the oracle's eval-mode generator against the reference's own G_NET after netG.eval()
(ref: evaluator.py:108-138), and the library calls G_NET.eval() issues (DRY_RUN: host logic only).

The reference side is stored in tests/golden/reference/g_net_forward_eval_B{1,3}.npz.  The running statistics in it
come from 10 train-mode forwards of the reference's G_NET on seeded batches (fresh statistics saturate most pixels
and make a weak test); they are stored whole (keys ``in__rs__*``), so the GPU tests load them without the reference.
Re-record with the reference importable (tests/refimport.py):

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_eval_mode.py
"""
import numpy as np
import pytest
import torch

import oracle_eval
import reference_fixtures as fixtures
import refimport
from objgan_b200 import lib, model, ops, synth

CAP = fixtures.CAP
TRAIN_PASSES = 10


def _g_sd():
    """state_dict of objgan_b200's G_NET(80) after weights_init under torch.manual_seed(0) (as test_g_net_forward)."""
    torch.manual_seed(0)
    g = model.G_NET(80)
    g.apply(model.weights_init)
    return {k: v.clone() for k, v in g.state_dict().items()}


def _ref_forward(g, inp, seed):
    """The reference's G_NET forward with its CA_NET draw taken under a fixed seed; returns (outputs, eps)."""
    torch.manual_seed(seed)
    eps = torch.FloatTensor(inp["z"].shape[0], 100).normal_()      # CA_NET.reparametrize's draw (model.py:473-477)
    torch.manual_seed(seed)
    out = g(inp["z"], inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"], inp["slabels_feat"], inp["mask"],
            inp["hmaps"], inp["rois"], inp["fm_rois"], inp["num_rois"], inp["bt_masks"], inp["fm_bt_masks"],
            inp["glb_max_num_roi"])
    return out, eps


_trained = {}


def _trained_ref_g(ref):
    """The reference's G_NET with _g_sd() weights after TRAIN_PASSES train-mode forwards on seeded batches of 3."""
    if "g" not in _trained:
        g = ref.model.G_NET(80)
        g.load_state_dict(_g_sd(), strict=True)
        g.train()
        with torch.no_grad():
            for i in range(TRAIN_PASSES):
                _ref_forward(g, synth.make_inputs(3, seed=200 + i, parity=True), 300 + i)
        _trained["g"] = g
    return _trained["g"]


def _buffers(sd):
    return {k: v for k, v in sd.items() if "running" in k or "num_batches" in k}


def eval_fixture(B, monkeypatch=None):
    """{key: tensor} of g_net_forward_eval_B{B}: in__rs__<buffer> (running statistics, whole), in__eps, the eval-mode
    outputs, and after__<buffer> (the buffers after the eval forward)."""
    def produce():
        if monkeypatch is not None:      # torch 2 masks need bool: the reference's ByteTensor mask, as bool
            monkeypatch.setattr(torch, "ByteTensor", lambda a: torch.from_numpy(np.asarray(a)).bool())
        ref = refimport.load()
        g = _trained_ref_g(ref)
        before = {k: v.clone() for k, v in _buffers(g.state_dict()).items()}
        g.eval()
        with torch.no_grad():
            out, eps = _ref_forward(g, eval_inputs(B), 7)
        g.train()
        r = {"in__eps": eps, "mu": out[4], "logvar": out[5]}
        r.update({"in__rs__" + k: v for k, v in before.items()})
        r.update({f"fake{i}": out[0][i] for i in range(3)})
        r.update({f"out{j}_{i}": out[j][i] for j in (1, 2, 3) for i in range(2)})
        r.update({"after__" + k: v for k, v in _buffers(g.state_dict()).items()})
        return r
    return fixtures.recorded(f"g_net_forward_eval_B{B}", produce)


def eval_inputs(B):
    return synth.make_inputs(B, seed=40 + B, parity=True)


def eval_state_dict(want):
    """_g_sd() with the fixture's running statistics."""
    sd = _g_sd()
    for k in _buffers(sd):
        sd[k] = want["in__rs__" + k].to(sd[k].dtype).reshape(sd[k].shape)
    return sd


def _close(a, b, tol=1e-4, cap=CAP):
    a = torch.from_numpy(fixtures.sample(a, cap)) if torch.as_tensor(a).numel() > cap else torch.as_tensor(a).float()
    b = torch.as_tensor(b).float()
    assert a.numel() == b.numel()
    a, b = a.reshape(-1), b.reshape(-1)
    assert torch.isfinite(a).all()
    err = (a - b).abs().max().item()
    ref = max(b.abs().max().item(), 1e-6)
    assert err <= tol * max(ref, 1.0), (err, ref)


@pytest.mark.parametrize("B", [1, 3])
def test_g_net_forward_eval(B, monkeypatch):
    """The oracle's eval-mode G forward equals the reference's G_NET after eval() (same budget as
    test_oracle_vs_reference.py::test_g_net_forward); the reference left its buffers as they were, and so does the
    oracle."""
    want = eval_fixture(B, monkeypatch)
    sd = eval_state_dict(want)
    sd0 = {k: v.clone() for k, v in sd.items()}
    inp = eval_inputs(B)
    inp["eps"] = want["in__eps"]
    with torch.no_grad():
        o = oracle_eval.g_net_forward_eval(sd, inp)
    for i in range(3):
        _close(o[0][i], want[f"fake{i}"])
    for j in (1, 2, 3):
        for i in range(2):
            _close(o[j][i], want[f"out{j}_{i}"])
    _close(o[4], want["mu"])
    _close(o[5], want["logvar"])
    for k in _buffers(sd):
        assert torch.equal(sd[k], sd0[k]), k
        after = want["after__" + k]
        assert np.array_equal(fixtures.sample(sd0[k]).reshape(-1), after.numpy().reshape(-1)), k
    assert int(want["in__rs__h_net1_sent.fc.1.num_batches_tracked"]) == TRAIN_PASSES


# ---------------------------------------------------------------------------------------------------
# library calls (DRY_RUN: no kernels run, the call sequence and argument counts are what is checked)
# ---------------------------------------------------------------------------------------------------
@pytest.fixture()
def dry():
    lib.DRY_RUN = True
    model.FAST_INIT = True
    yield
    lib.DRY_RUN = False
    model.FAST_INIT = False


def _trace(monkeypatch, fn):
    calls = []
    real = ops._call

    def rec(name, *args):
        calls.append((name, len(args)))
        return real(name, *args)
    monkeypatch.setattr(ops, "_call", rec)
    fn()
    monkeypatch.setattr(ops, "_call", real)
    return calls


def test_eval_call_sequence(dry, monkeypatch):
    g = model.G_NET(80)
    inp = synth.make_inputs(2, parity=True)

    def fwd():
        with torch.no_grad():
            g(inp["z"], inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"], inp["slabels_feat"], inp["mask"],
              inp["hmaps"], inp["rois"], inp["fm_rois"], inp["num_rois"], inp["bt_masks"], inp["fm_bt_masks"],
              inp["glb_max_num_roi"])
    fwd()                                   # the first pass also packs the weights
    train = _trace(monkeypatch, fwd)
    bufs = {k: v.clone() for k, v in g.named_buffers()}
    g.eval()
    ev = _trace(monkeypatch, fwd)
    count = lambda calls, name: sum(1 for n, _ in calls if n == name)
    assert count(train, "og_norm_stats") == 35 and count(ev, "og_norm_stats") == 29
    assert count(train, "og_bn_eval_coef") == 0 and count(ev, "og_bn_eval_coef") == 6
    assert len(ev) == len(train)            # one coefficient call in place of each BatchNorm statistics call
    for k, v in g.named_buffers():
        assert torch.equal(v, bufs[k]), k
    g.train()
    assert _trace(monkeypatch, fwd) == train


def test_eval_backward_wiring(dry):
    """Gradients w.r.t. z through the eval-mode generator reach og_bn_eval_backward, and the parameters of the
    BatchNorm layers receive gradients too."""
    g = model.G_NET(80).eval()
    inp = synth.make_inputs(2, parity=True)
    z = inp["z"].clone().requires_grad_(True)
    g.ca_net.eps_override = inp["eps"]
    out = g(z, inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"], inp["slabels_feat"], inp["mask"],
            inp["hmaps"], inp["rois"], inp["fm_rois"], inp["num_rois"], inp["bt_masks"], inp["fm_bt_masks"],
            inp["glb_max_num_roi"])
    sum(f.sum() for f in out[0]).backward()
    assert z.grad is not None and z.grad.shape == z.shape
    assert g.h_net1_sent.fc[1].weight.grad is not None
