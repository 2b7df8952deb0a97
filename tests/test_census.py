"""CPU guard of the shape tables of the kernel tests: every normalisation, convolution, attention and DAMSM shape the
networks' runs issue is a row of tests/{norm,conv,attention,damsm}_cases.py, no row is stale, and each convolution
row's path is the one the GPU takes, so a new layer, a new caller or a dispatch change cannot bring a shape or a route
that tests/test_gpu_{norm,conv,attention,damsm}.py never ran.  The runs are the dry-run workloads of tests/dry.py,
recorded once per session: the host code takes the GPU's dispatch, no kernel runs."""
import pytest

import attention_cases
import conv_cases
import damsm_cases
import norm_cases
from dry import dry, workload  # noqa: F401


def _union(needs, *runs):
    """The needs of several workloads together."""
    return set().union(*(needs(workload(r)) for r in runs))


def test_norm_step_b_shapes_are_cases(dry):
    needs = norm_cases.norm_needs(workload("step_b"))
    assert len(needs) > 30
    assert norm_cases.uncovered(needs) == []


def test_conv_step_b_shapes_are_cases(dry):
    needs = conv_cases.conv_needs(workload("step_b_encoder"))
    assert len(needs) > 60
    assert {n[-1] for n in needs} >= {"s1", "s2", "narrow", "simt", "tc"}
    assert conv_cases.uncovered(needs) == []


def test_attention_step_b_shapes_are_cases(dry):
    needs = attention_cases.att_needs(workload("step_b"))
    assert {e for e, _ in needs} == set(attention_cases.ENTRIES)       # every entry point, forward and backward
    assert attention_cases.uncovered(needs) == []


def test_damsm_step_b_shapes_are_cases(dry):
    needs = damsm_cases.damsm_needs(workload("step_b_encoder"))
    assert {e for e, _ in needs} == set(damsm_cases.ENTRIES)           # the step runs every entry point
    assert damsm_cases.uncovered(needs) == []


# table: (its needs of a workload, its uncovered, what an eval-mode G_NET forward must also show)
EVAL_G = {
    "norm": (norm_cases.norm_needs, norm_cases.uncovered, lambda needs: any(n[0] == "bn_eval" for n in needs)),
    "conv": (conv_cases.conv_needs, conv_cases.uncovered, lambda needs: True),
    "attention": (attention_cases.att_needs, attention_cases.uncovered,
                  lambda needs: any(e == "og_att_general_fwd" for e, _ in needs)),
}


@pytest.mark.parametrize("batch", [1, 16])
@pytest.mark.parametrize("table", EVAL_G)
def test_eval_generator_shapes_are_cases(dry, table, batch):
    needs_of, uncovered, shows = EVAL_G[table]
    needs = needs_of(workload(f"eval_g{batch}"))
    assert shows(needs)
    assert uncovered(needs) == []


def test_inception_shapes_are_cases(dry):
    assert conv_cases.uncovered(conv_cases.conv_needs(workload("inception"))) == []


def test_rprecision_shapes_are_cases(dry):
    needs = damsm_cases.damsm_needs(workload("rprecision"))
    assert {e for e, _ in needs} == {"og_words_pairs_fwd", "og_cosine_matrix_fwd", "og_ce_pair"}
    assert damsm_cases.uncovered(needs) == []


# No row of a table is stale: each is issued by one of the runs above, so the table stays the list of what the networks
# run (deleting any row makes one of the tests above fail).
def test_norm_no_case_is_stale(dry):
    assert norm_cases.stale(_union(norm_cases.norm_needs, "step_b", "eval_g1", "eval_g16")) == []


def test_conv_no_case_is_stale(dry):
    needs = _union(conv_cases.conv_needs, "step_b_encoder", "eval_g1", "eval_g16", "inception")
    assert conv_cases.stale(needs) == []


def test_attention_no_case_is_stale(dry):
    assert attention_cases.stale(_union(attention_cases.att_needs, "step_b", "eval_g1", "eval_g16")) == []


def test_damsm_no_case_is_stale(dry):
    assert damsm_cases.stale(_union(damsm_cases.damsm_needs, "step_b_encoder", "rprecision")) == []


def test_paths_are_the_gpu_rule():
    """The path column of every conv row is what ops.conv_path picks (its general form for ENC_CASES):
    a change of TC_MIN_PIXELS or of the dispatch moves rows, and shows up as a table edit."""
    C = conv_cases
    assert [r for r in C.CASES + C.EDGE_CASES if C.path_of(*r[:9], r[11]) != r[12]] == []
    assert [r for r in C.ENC_CASES if C.enc_path(*r[1:4], *r[6:11]) != r[15]] == []
    assert len(set(C.CASES)) == len(C.CASES) and len(set(C.ENC_CASES)) == len(C.ENC_CASES)
