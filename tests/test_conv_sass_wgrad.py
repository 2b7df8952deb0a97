"""The weight-gradient kernel of conv_tc.cu in SASS, checked without a GPU: every instantiated ci width issues one
wgmma over its whole (MN-major, several-slab) B extent per product and k-step, so a stage is 4 x 3 HGMMAs in
one run that ends in its own wait (twice per stage when two entries share the G tile), with no C75xx serialization
note and no spills."""
import os
import re
import shutil
import subprocess

import pytest

from objgan_b200 import build

NVCC = build.NVCC
pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which(NVCC)), reason="nvcc not available")

WIDTHS = {32, 48, 64, 96, 104, 112, 128}


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("conv_sass_wgrad")
    obj = str(d / "conv_tc.o")
    cmd = [NVCC, "-Xptxas=-v", *build.FLAGS, "-c", os.path.join(build.CSRC, "conv_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


def _demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else list(names)


def _wgrad(name):
    """(ci width, entries per CTA) of a weight-gradient kernel instantiation."""
    m = re.search(r"conv_tc_wgrad\w*<(\d+), (\d+), (\d+)>", name)
    return (int(m.group(1)), int(m.group(3))) if m else None


# every width with one entry per CTA; widths up to 104 also with two entries sharing the G tile
KERNELS = {(w, t) for w in WIDTHS for t in (1, 2) if t == 1 or w <= 104}


def test_wgrad_kernels_no_serialization_or_spills(compiled):
    _, log = compiled
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln)]
    assert not notes, "\n".join(notes[:10])
    cur, spills = None, {}
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            cur = _demangle([m.group(1)])[0]
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur and _wgrad(cur):
            spills[cur] = (int(m.group(1)), int(m.group(2)))
    assert {_wgrad(n) for n in spills} == KERNELS, sorted(spills)
    assert all(v == (0, 0) for v in spills.values()), spills


def test_wgrad_stage_is_one_wide_mma_per_product_and_k_step(compiled):
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
    seen = set()
    for f, name in zip(funcs, _demangle(list(funcs))):
        key = _wgrad(name)
        if not key:
            continue
        bnw, _ = key
        groups, n, shapes = [], 0, set()
        for ln in funcs[f]:
            if "HGMMA" in ln:
                n += 1
                shapes.update(re.findall(r"HGMMA\.64x(\d+)x16", ln))
            elif "WARPGROUP.DEPBAR" in ln:
                groups.append(n)
                n = 0
        assert groups and max(groups) == 4 * 3, (name, groups)
        assert shapes == {str(bnw)}, (name, shapes)
        seen.add(key)
    assert seen == KERNELS, sorted(seen)
