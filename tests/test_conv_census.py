"""CPU guard of tests/conv_cases.py: every convolution shape a batch-16 Step-B step (DAMSM image encoder attached), an
eval-mode G_NET forward (batch 1 and 16) and the Inception forwards (batch 16) issue is a row of CASES / ENC_CASES, no
row is stale, and each row's path is the one the GPU takes, so a new layer or a dispatch change cannot bring a shape or
a route that tests/test_gpu_conv.py never ran.  lib.DRY_RUN: the host code issues its library calls (argument lists
checked against the header), no kernel runs."""
import random

import pytest
import torch

from conv_cases import CASES, EDGE_CASES, ENC_CASES, conv_needs, enc_path, path_of, stale, uncovered
from objgan_b200 import lib, model, synth, trainer


@pytest.fixture()
def dry():
    lib.DRY_RUN = True
    model.FAST_INIT = True
    yield
    lib.DRY_RUN = False
    model.FAST_INIT = False


def _step_b():
    t = trainer.StepBTrainer(device="cpu", seed=0, image_encoder=model.CNN_ENCODER(256))
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


def test_step_b_shapes_are_cases(dry):
    needs = conv_needs(_step_b)
    assert len(needs) > 60
    assert {n[-1] for n in needs} >= {"s1", "s2", "narrow", "simt", "tc"}
    assert uncovered(needs) == []


@pytest.mark.parametrize("batch", [1, 16])
def test_eval_generator_shapes_are_cases(dry, batch):
    assert uncovered(conv_needs(lambda: _eval_g(batch))) == []


def test_inception_shapes_are_cases(dry):
    assert uncovered(conv_needs(_inception)) == []


def test_no_case_is_stale(dry):
    """Each row of CASES / ENC_CASES is issued by one of the runs, so the tables stay the list of what the networks run
    (deleting any row makes one of the tests above fail)."""
    needs = conv_needs(_step_b) | conv_needs(lambda: _eval_g(1)) | conv_needs(lambda: _eval_g(16)) | \
        conv_needs(_inception)
    assert stale(needs) == []


def test_paths_are_the_gpu_rule():
    """The path column of every row is what ops.conv_path picks (its general form for ENC_CASES):
    a change of TC_MIN_PIXELS or of the dispatch moves rows, and shows up as a table edit."""
    assert [r for r in CASES + EDGE_CASES if path_of(*r[:9], r[11]) != r[12]] == []
    assert [r for r in ENC_CASES if enc_path(*r[1:4], *r[6:11]) != r[15]] == []
    assert len(set(CASES)) == len(CASES) and len(set(ENC_CASES)) == len(ENC_CASES)
