"""What ptxas makes of the tensor-core convolutions (conv_tc.cu), checked without a GPU.

Every wgmma of a pipeline stage must issue back to back: ptxas serializes them (a wait after each one) when the issue
window holds a branch it cannot prove warp-uniform, a run-time choice of how many MMAs to issue, or a read of the
accumulator registers, and it says so with a "Potential Performance Loss" / "injected" (C75xx) note.  The tests
compile conv_tc.cu exactly as build.py does plus -Xptxas -v and assert: no C75xx note, no spills, and in the SASS a
stage's MMAs as one group that ends in the only wait of the stage."""
import os
import re
import shutil
import subprocess

import pytest

from objgan_b200 import build

NVCC = build.NVCC
pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which(NVCC)), reason="nvcc not available")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("conv_sass")
    obj = str(d / "conv_tc.o")
    cmd = [NVCC, "-Xptxas=-v", *build.FLAGS, "-c", os.path.join(build.CSRC, "conv_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


def _demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    if r.returncode != 0:
        return list(names)
    return r.stdout.splitlines()


def test_no_serialization_warnings_or_spills(compiled):
    _, log = compiled
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln)]
    assert not notes, "\n".join(notes[:10])
    # per function: "Compiling entry function '<f>'" ... "<n> bytes stack frame, <s> bytes spill stores, <l> ... loads"
    cur, seen = None, {}
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur:
            seen[cur] = (int(m.group(1)), int(m.group(2)))
    conv = {k: v for k, v in seen.items() if "conv_tc" in k}
    assert len(conv) >= 10, sorted(seen)
    spills = {n: v for n, v in zip(_demangle(list(conv)), conv.values()) if v != (0, 0)}
    assert not spills, spills


def _stage_groups(sass_lines):
    """Sizes of the HGMMA runs between two WARPGROUP.DEPBAR waits."""
    groups, n = [], 0
    for ln in sass_lines:
        if "HGMMA" in ln:
            n += 1
        elif "WARPGROUP.DEPBAR" in ln:
            groups.append(n)
            n = 0
    return groups


def test_stage_of_three_products_issues_as_one_group(compiled):
    """The widest HGMMA group of each kernel is a whole stage: 4 k-steps x 3 products, or x 2 in the stacked form
    (one wide MMA per product and k-step in the fprop / dgrad and in the weight-gradient kernel)."""
    obj, _ = compiled
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    if not cuobjdump:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(ln)
    names = dict(zip(funcs, _demangle(list(funcs))))
    checked = 0
    for f, lines in funcs.items():
        name = names[f]
        m = re.search(r"conv_tc_kernel<(\d+), (\d+), (true|false)>", name)
        w = re.search(r"conv_tc_wgrad_wide_kernel<(\d+), (\d+), (\d+)>", name)
        if m:
            want = 4 * (2 if m.group(3) == "true" else 3)
        elif w:
            want = 4 * 3
        else:
            continue
        groups = _stage_groups(lines)
        assert groups and max(groups) == want, (name, groups)
        checked += 1
    assert checked >= 10, checked
