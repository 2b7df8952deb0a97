"""CPU guard of tests/damsm_cases.py: every DAMSM matching and encoder-gather shape that a batch-16 Step-B step (DAMSM
image encoder attached) and an R-precision pool of 100 issue is a row of CASES, and no row is stale, so a new layer or
a new caller cannot bring a shape that tests/test_gpu_damsm.py never ran.
lib.DRY_RUN: the host code issues its library calls (argument lists checked against the header), no kernel runs."""
import random

import pytest
import torch

from damsm_cases import ENTRIES, damsm_needs, stale, uncovered
from objgan_b200 import lib, losses, model, synth, trainer


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


def _rprecision():
    """Seven batches of 16 fill the pool of 100, the eighth call scores it (like the evaluator)."""
    rp = losses.RPrecision(100)
    for i in range(8):
        b = synth.make_inputs(16, seed=300 + i)
        rp.add(torch.zeros(16, 256, 17, 17), torch.zeros(16, 256), b["words_embs"], b["sent_emb"], b["cap_lens"])
    assert len(rp.w_accuracy) == 1


def test_step_b_shapes_are_cases(dry):
    needs = damsm_needs(_step_b)
    assert {e for e, _ in needs} == set(ENTRIES)       # the step runs every entry point of the tables
    assert uncovered(needs) == []


def test_rprecision_shapes_are_cases(dry):
    needs = damsm_needs(_rprecision)
    assert {e for e, _ in needs} == {"og_words_pairs_fwd", "og_cosine_matrix_fwd", "og_ce_pair"}
    assert uncovered(needs) == []


def test_every_case_is_issued(dry):
    """No row of CASES is stale: each is issued by one of the two runs, so the table stays the list of what the
    networks run (deleting any row makes one of the tests above fail)."""
    assert stale(damsm_needs(_step_b) | damsm_needs(_rprecision)) == []
