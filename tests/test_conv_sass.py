"""What ptxas makes of the tensor-core convolutions (conv_tc.cu), checked without a GPU.

Every wgmma of a pipeline stage must issue back to back: ptxas serializes them (a wait after each one) when the issue
window holds a branch it cannot prove warp-uniform, a run-time choice of how many MMAs to issue, or a read of the
accumulator registers, and it says so with a "Potential Performance Loss" / "injected" (C75xx) note.  The tests
compile conv_tc.cu once, exactly as build.py does plus -Xptxas -v, and assert: no C75xx note, no spills, the exact set
of kernel instantiations, and in the SASS a stage's MMAs as one group that ends in the only wait of the stage."""
import os
import re
import shutil
import subprocess

import pytest

from objgan_b200 import build

NVCC = build.NVCC
pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which(NVCC)), reason="nvcc not available")

FORWARD = re.compile(r"conv_tc_kernel<(\d+), (\d+), (true|false)>")
ROWS = re.compile(r"conv_tc_rows_kernel<(\d+), (true|false)>")
WGRAD = re.compile(r"conv_tc_wgrad_wide_kernel<(\d+), (\d+), (\d+)>")

WIDTHS = (32, 48, 64, 96, 104, 112, 128)
# (BN, STAGES, STACKED): the operand ring is as deep as 200 KB holds, at most 4 stages
FORWARD_KERNELS = {(w, 4 if w <= 64 else 3, "false") for w in WIDTHS} | {(32, 4, "true"), (64, 4, "true")}
ROWS_KERNELS = {(w, "false") for w in WIDTHS} | {(32, "true"), (64, "true")}
# (BNW, STAGES, TAPS): every width with one entry per CTA; widths up to 104 also with two entries sharing the G tile
WGRAD_KERNELS = ({(w, 4 if w <= 64 else 3, 1) for w in WIDTHS}
                 | {(w, 3 if w <= 64 else 2, 2) for w in WIDTHS if w <= 104})


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("conv_sass")
    obj = str(d / "conv_tc.o")
    cmd = [NVCC, "-Xptxas=-v", *build.FLAGS, "-c", os.path.join(build.CSRC, "conv_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return obj, r.stderr


@pytest.fixture(scope="module")
def sass(compiled):
    """Demangled function name -> its SASS lines."""
    obj, _ = compiled
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    if not cuobjdump:
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(ln)
    return dict(zip(_demangle(list(funcs)), funcs.values()))


def _demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else list(names)


def _spills(log):
    """Demangled entry function -> (spill store bytes, spill load bytes), from the ptxas -v log."""
    cur, seen = None, {}
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur:
            seen[cur] = (int(m.group(1)), int(m.group(2)))
    return dict(zip(_demangle(list(seen)), seen.values()))


def _instances(names, pattern):
    return {tuple(int(g) if g.isdigit() else g for g in m.groups()) for m in map(pattern.search, names) if m}


def _stage_groups(lines):
    """Sizes of the HGMMA runs between two WARPGROUP.DEPBAR waits."""
    groups, n = [], 0
    for ln in lines:
        if "HGMMA" in ln:
            n += 1
        elif "WARPGROUP.DEPBAR" in ln:
            groups.append(n)
            n = 0
    return groups


def _check_spills(log, pattern, kernels):
    spills = {n: v for n, v in _spills(log).items() if pattern.search(n)}
    assert _instances(spills, pattern) == kernels, sorted(spills)
    assert all(v == (0, 0) for v in spills.values()), spills


def _check_stage_groups(sass, pattern, kernels, want):
    """want(match, lines) -> the widest HGMMA group between two waits that each instantiation must have."""
    seen = set()
    for name, lines in sass.items():
        m = pattern.search(name)
        if not m:
            continue
        groups = _stage_groups(lines)
        assert groups and max(groups) == want(m, lines), (name, groups)
        seen.add(name)
    assert _instances(seen, pattern) == kernels, sorted(seen)


def test_no_serialization_warnings_or_spills(compiled):
    _, log = compiled
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln)]
    assert not notes, "\n".join(notes[:10])
    conv = {n: v for n, v in _spills(log).items() if "conv_tc" in n}
    assert not {n: v for n, v in conv.items() if v != (0, 0)}, conv
    _check_spills(log, FORWARD, FORWARD_KERNELS)


def test_rows_kernel_no_serialization_notes_or_spills(compiled):
    _, log = compiled
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln) and "conv_tc_rows_kernel" in ln]
    assert not notes, "\n".join(notes[:10])
    _check_spills(log, ROWS, ROWS_KERNELS)


def test_wgrad_kernels_no_serialization_or_spills(compiled):
    _, log = compiled
    notes = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln)]
    assert not notes, "\n".join(notes[:10])
    _check_spills(log, WGRAD, WGRAD_KERNELS)


def test_stage_of_three_products_issues_as_one_group(sass):
    """The widest HGMMA group of each kernel is a whole stage: 4 k-steps x 3 products, or x 2 in the stacked form
    (one wide MMA per product and k-step in the fprop / dgrad and in the weight-gradient kernel)."""
    _check_stage_groups(sass, FORWARD, FORWARD_KERNELS, lambda m, _: 4 * (2 if m.group(3) == "true" else 3))
    _check_stage_groups(sass, WGRAD, WGRAD_KERNELS, lambda m, _: 4 * 3)


def test_rows_kernel_stage_issues_as_one_group(sass):
    """The row-run kernel issues the same stage windows as conv_tc_kernel: 4 k-steps x 3 products, x 2 stacked."""
    _check_stage_groups(sass, ROWS, ROWS_KERNELS, lambda m, _: 4 * (2 if m.group(2) == "true" else 3))


def test_wgrad_stage_is_one_wide_mma_per_product_and_k_step(sass):
    """Every weight-gradient width issues one wgmma over its whole (MN-major, several-slab) B extent per product and
    k-step: a stage is 4 x 3 HGMMAs in one run that ends in its own wait (twice per stage when two entries share the G
    tile)."""
    def want(m, lines):
        shapes = {s for ln in lines for s in re.findall(r"HGMMA\.64x(\d+)x16", ln)}
        assert shapes == {m.group(1)}, (m.group(0), shapes)
        return 4 * 3
    _check_stage_groups(sass, WGRAD, WGRAD_KERNELS, want)
