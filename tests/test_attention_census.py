"""CPU guard of tests/attention_cases.py: every attention, mask-paint and word-projection shape a batch-16 Step-B step and
an eval-mode G_NET forward (batch 1 and 16) issue is a row of CASES, so a new layer cannot bring a shape that
tests/test_gpu_attention.py never ran.
lib.DRY_RUN: the host code issues its library calls (argument lists checked against the header), no kernel runs."""
import random

import pytest
import torch

from attention_cases import ENTRIES, att_needs, stale, uncovered
from objgan_b200 import lib, model, synth, trainer


@pytest.fixture()
def dry():
    lib.DRY_RUN = True
    model.FAST_INIT = True
    yield
    lib.DRY_RUN = False
    model.FAST_INIT = False


def _step_b():
    t = trainer.StepBTrainer(device="cpu", seed=0)
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


def test_step_b_shapes_are_cases(dry):
    needs = att_needs(_step_b)
    assert {e for e, _ in needs} == set(ENTRIES)       # the step runs every entry point, forward and backward
    assert uncovered(needs) == []


@pytest.mark.parametrize("batch", [1, 16])
def test_eval_generator_shapes_are_cases(dry, batch):
    needs = att_needs(lambda: _eval_g(batch))
    assert any(e == "og_att_general_fwd" for e, _ in needs)
    assert uncovered(needs) == []


def test_every_case_is_issued(dry):
    """No row of CASES is stale: each is issued by one of the three runs, so the table stays the list of what the
    networks run (deleting any row makes one of the tests above fail)."""
    needs = att_needs(_step_b) | att_needs(lambda: _eval_g(1)) | att_needs(lambda: _eval_g(16))
    assert stale(needs) == []
