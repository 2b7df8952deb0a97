"""Dry runs for the CPU tests.  Under lib.DRY_RUN the host code takes the GPU's dispatch on CPU tensors, and ops._call
checks each library call's argument count against the header and counts it instead of launching, so no kernel runs and
outputs stay uninitialised.

  dry        fixture: a dry run with model.FAST_INIT (values are never looked at), both restored after the test
  record     the library calls a function issues
  workload   the recorded library calls and convolution layers of one of the networks' runs, once per session
"""
import functools
import random
from collections import namedtuple

import pytest
import torch

from objgan_b200 import lib, losses, model, ops, synth, trainer
from objgan_b200.lib import ACT_LRELU


@pytest.fixture()
def dry(monkeypatch):
    monkeypatch.setattr(lib, "DRY_RUN", True)
    monkeypatch.setattr(model, "FAST_INIT", True)


def record(fn, calls=None):
    """Runs ``fn()`` and returns ``calls`` (a new list by default) with (name, args) appended for each library call it
    issued; a test may append its own events to the same list to interleave them.  The calls still go through ops._call,
    so a dry run checks their argument counts."""
    calls = [] if calls is None else calls
    real = ops._call

    def rec(name, *args):
        calls.append((name, args))
        return real(name, *args)
    ops._call = rec
    try:
        fn()
    finally:
        ops._call = real
    return calls


# ---------------------------------------------------------------------------------------------------------------------
# the networks' runs whose shapes the *_cases.py tables list
# ---------------------------------------------------------------------------------------------------------------------
def _step_b(encoder):
    t = trainer.StepBTrainer(device="cpu", seed=0, image_encoder=model.CNN_ENCODER(256) if encoder else None)
    inp = synth.make_inputs(16)
    random.seed(1)
    t.step(inp)


def _eval_g(batch):
    g = model.G_NET(80).eval()
    inp = synth.make_inputs(batch, seed=7, parity=batch > 1)
    with torch.no_grad():
        g(inp["z"], inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"], inp["slabels_feat"], inp["mask"],
          inp["hmaps"], inp["rois"], inp["fm_rois"], inp["num_rois"], inp["bt_masks"], inp["fm_bt_masks"],
          inp["glb_max_num_roi"])


def _inception():
    imgs = torch.zeros(16, 3, 256, 256)
    with torch.no_grad():
        model.INCEPTION_V3()(imgs)
        model.INCEPTION_V3_FID().activations(imgs)


def _rprecision():
    """Seven batches of 16 fill the pool of 100, the eighth call scores it (like the evaluator)."""
    rp = losses.RPrecision(100)
    for i in range(8):
        b = synth.make_inputs(16, seed=300 + i)
        rp.add(torch.zeros(16, 256, 17, 17), torch.zeros(16, 256), b["words_embs"], b["sent_emb"], b["cap_lens"])
    assert len(rp.w_accuracy) == 1


WORKLOADS = {
    "step_b": lambda: _step_b(False),                   # a batch-16 StepBTrainer.step
    "step_b_encoder": lambda: _step_b(True),            # the same with the DAMSM image encoder CNN_ENCODER(256)
    "eval_g1": lambda: _eval_g(1),                      # an eval-mode G_NET forward (GSampler) at batch 1
    "eval_g16": lambda: _eval_g(16),
    "inception": _inception,                            # INCEPTION_V3 and INCEPTION_V3_FID at batch 16
    "rprecision": _rprecision,                          # an R-precision pool of 100
}

# calls: record()'s (name, args) list.  convs: per ops.conv2d, a conv_cases.CASES row without its path; encs: per
# ops.enc_conv_fwd / enc_conv_dgrad, a conv_cases.ENC_CASES row without its path
Workload = namedtuple("Workload", "calls convs encs")


@functools.lru_cache(maxsize=None)
def workload(name):
    """The Workload of WORKLOADS[name] under a dry run, recorded on first use."""
    assert lib.DRY_RUN and model.FAST_INIT, "workloads are recorded under the dry fixture"
    convs, encs = [], []
    real_fwd, real_efwd, real_edgrad = ops._Conv2d.forward, ops.enc_conv_fwd, ops.enc_conv_dgrad

    def fwd(ctx, x, weight, bias, cache, stride, pad, mode, act, split):
        n, h, w, _ = x.shape
        co, ci, k, _ = weight.shape
        convs.append((n, h, w, ci, co, k, stride, pad, mode, act, bias is not None, split))
        return real_fwd(ctx, x, weight, bias, cache, stride, pad, mode, act, split)

    def enc(d, layer, n, h, w, yoff, cy):
        encs.append((d, n, h, w, layer.cin, layer.cout, layer.kh, layer.kw, layer.stride, layer.padh, layer.padw,
                     layer.act == ACT_LRELU, layer.bns is not None or len(layer.weights) > 1, yoff, cy))

    def efwd(layer, x, y, yoff=0):
        enc("fwd", layer, *x.shape[:3], yoff, y.shape[3])
        return real_efwd(layer, x, y, yoff)

    def edgrad(layer, gp, h, w):
        enc("dgrad", layer, gp.shape[0], h, w, 0, ops.cpad(layer.cin))
        return real_edgrad(layer, gp, h, w)

    ops._Conv2d.forward, ops.enc_conv_fwd, ops.enc_conv_dgrad = staticmethod(fwd), efwd, edgrad
    try:
        calls = record(WORKLOADS[name])
    finally:
        ops._Conv2d.forward, ops.enc_conv_fwd, ops.enc_conv_dgrad = staticmethod(real_fwd), real_efwd, real_edgrad
    return Workload(calls, convs, encs)
