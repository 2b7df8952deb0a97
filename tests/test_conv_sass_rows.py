"""What ptxas makes of the row-run forward kernel (conv_tc_rows_kernel in conv_tc.cu), checked without a GPU.

The kernel reads each stage's A operand from a resident slot instead of a per-stage tile, but its consumer issues the
same stage windows as conv_tc_kernel: a stage's MMAs must go out back to back and end in the stage's only wait, with
no C75xx "Potential Performance Loss" note and no spills (see tests/test_conv_sass.py for why)."""
import os
import re
import shutil
import subprocess

import pytest

from objgan_b200 import build

NVCC = build.NVCC
pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which(NVCC)), reason="nvcc not available")

KERNEL = re.compile(r"conv_tc_rows_kernel<(\d+), (true|false)>")
WIDTHS = {("32", "false"), ("48", "false"), ("64", "false"), ("96", "false"), ("104", "false"), ("112", "false"),
          ("128", "false"), ("32", "true"), ("64", "true")}


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("conv_sass_rows")
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


def test_rows_kernel_no_serialization_notes_or_spills(compiled):
    _, log = compiled
    # a C75xx note names the (mangled) function it is about
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln) and "conv_tc_rows_kernel" in ln]
    assert not notes, "\n".join(notes[:10])
    cur, spills = None, {}
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
    rows = {n: v for n, v in zip(_demangle(list(spills)), spills.values()) if KERNEL.search(n)}
    assert {KERNEL.search(n).groups() for n in rows} == WIDTHS, sorted(rows)
    assert all(v == (0, 0) for v in rows.values()), rows


def test_rows_kernel_stage_issues_as_one_group(compiled):
    """The widest HGMMA group between two waits is a whole stage: 4 k-steps x 3 products, x 2 in the stacked form."""
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
    seen = set()
    for f, lines in funcs.items():
        m = KERNEL.search(names[f])
        if not m:
            continue
        groups, n = [], 0
        for ln in lines:
            if "HGMMA" in ln:
                n += 1
            elif "WARPGROUP.DEPBAR" in ln:
                groups.append(n)
                n = 0
        want = 4 * (2 if m.group(2) == "true" else 3)
        assert groups and max(groups) == want, (names[f], groups)
        seen.add(m.groups())
    assert seen == WIDTHS, sorted(seen)
