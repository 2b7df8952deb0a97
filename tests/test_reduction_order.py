"""Run-to-run determinism of the Step-A step, checked without a GPU.

The step amplifies rounding by 10^3 - 10^4 per step, so a sum whose order depends on thread scheduling makes two runs
diverge.  Cross-CTA reductions therefore store per-CTA partials to planes of a workspace and add the planes in a fixed
order.  The only atomic adds left are the scatter adds of Step-B's object and DAMSM path (ALLOWED): this file checks
that csrc/ has no other, and that a Step-A step issues none of the entry points that launch them.
"""
import glob
import os
import re

from dry import dry, record  # noqa: F401
from objgan_b200 import synth, trainer

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "obj-gan_b200", "csrc")
ALLOWED = {                 # kernel: (file, entry point that launches it) -- fp32 scatter adds of Step-B's backward
    "roi_align_bwd_kernel": ("roi_align.cu", "ROIAlignBackwardLaucher"),
    "roi_align_avg_bwd_kernel": ("roi_align.cu", "og_roi_align_avg_bwd"),
    "roi_align_avg_nhwc_bwd_kernel": ("roi_align.cu", "og_roi_align_avg_nhwc_bwd"),
    "scatter_rows_add_kernel": ("elementwise.cu", "og_scatter_rows_add"),
    "bilinear_bwd_kernel": ("elementwise.cu", "og_bilinear_bwd"),
    "words_pairs_bwd_kernel": ("words_pairs.cu", "og_words_pairs_bwd"),
}
# the name of a kernel or device function definition
_FUNC = re.compile(r"(?:__global__|__device__)[^;{}=()]*?(?:__launch_bounds__\([^)]*\)[^;{}=()]*?)?\b(\w+)\s*\(")


def _sources():
    """(file name, source without its // comments) of csrc/*.cu and *.cuh"""
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        with open(path) as f:
            yield os.path.basename(path), re.sub(r"//[^\n]*", "", f.read())


def _atomic_sites():
    """(file, line, enclosing function) of every atomicAdd: the last kernel or device function defined before it."""
    for name, src in _sources():
        for m in re.finditer(r"\batomicAdd\b", src):
            funcs = _FUNC.findall(src, 0, m.start())
            yield name, src.count("\n", 0, m.start()) + 1, funcs[-1] if funcs else None


def test_atomics_only_in_step_b_scatter_kernels():
    found = list(_atomic_sites())
    bad = [(f, line, k) for f, line, k in found if ALLOWED.get(k, (None,))[0] != f]
    assert not bad, "atomicAdd outside the allowed scatter kernels (file, line, kernel): %s" % bad
    assert {k for _, _, k in found} == set(ALLOWED), "an allowed kernel lost its atomics: update ALLOWED"


def test_step_a_issues_no_atomic_entry(dry):
    entries = {e for _, e in ALLOWED.values()}
    t = trainer.StepATrainer(device="cpu", seed=0)
    inp = synth.make_inputs(16, seed=1234, parity=False)
    issued = {name for name, _ in record(lambda: t.step(inp))}
    assert "og_norm_stats" in issued and "og_att_general_bwd" in issued    # the record covers the step's reductions
    assert not issued & entries, sorted(issued & entries)
