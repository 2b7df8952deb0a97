"""Shapes of the normalisation kernels (csrc/norm.cu), shared by tests/test_gpu_norm.py (which runs every row against a
float64 restatement) and tests/test_census.py (which checks that the networks issue no shape missing here).

A CASES row is (kind, groups, P, Cy, act, residual, affine):
  kind      "in"      InstanceNorm2d: groups = N, statistics per image (og_norm_stats / og_norm_apply / og_norm_backward)
            "bn"      train-mode BatchNorm: groups = 1, batch statistics, running buffers updated (same entry points)
            "bn_eval" eval-mode BatchNorm: og_bn_eval_coef + og_norm_apply + og_bn_eval_backward
  groups, P groups of P pixels each (P = H*W for InstanceNorm, N*H*W for BatchNorm2d, N for BatchNorm1d)
  Cy        channels of the normalised tensor (both halves for GLU; multiple of 4)
  act       lib.NA_NONE / NA_LRELU / NA_GLU
  residual  a residual is added after the activation
  affine    gamma / beta present
A SPLIT_CASES row is (instance, N, H, W, Cy, act, residual, pad) of og_norm_bound + og_norm_apply_split, the
producer-side operand split whose output feeds a tensor-core convolution (pad: that convolution's reflection halo).
Rows are kept at the size the networks run them (no batch is cut), so a shape the networks issue must be in the table
as it stands.  The EDGE_CASES and SPLIT_EDGE_CASES rows pin the kernels' code paths (see tests/test_gpu_norm.py).
"""
from objgan_b200.lib import NA_GLU, NA_LRELU, NA_NONE

# every distinct shape of one batch-16 StepBTrainer.step and of an eval-mode G_NET forward at batch 1 and 16
CASES = [
    # Step B, generator + discriminators, batch 16: BatchNorm
    ("bn", 1, 16, 24576, NA_GLU, False, True),          # INIT_STAGE_G: BatchNorm1d + GLU
    ("bn", 1, 16384, 96, NA_GLU, False, True),          # upBlocks 4x4 -> 128x128 ...
    ("bn", 1, 65536, 96, NA_GLU, False, True),
    ("bn", 1, 262144, 96, NA_GLU, False, True),
    ("bn", 1, 1048576, 96, NA_GLU, False, True),        # ... stage-3 upBlock at 256x256
    ("bn", 1, 4096, 192, NA_GLU, False, True),
    ("bn", 1, 240, 768, NA_LRELU, False, True),         # roi heads: P not a multiple of 32
    ("bn", 1, 256, 768, NA_LRELU, False, True),
    ("bn", 1, 768, 384, NA_LRELU, False, True),
    ("bn", 1, 784, 384, NA_LRELU, False, True),
    ("bn", 1, 960, 768, NA_LRELU, False, True),
    ("bn", 1, 1024, 384, NA_LRELU, False, True),
    ("bn", 1, 1024, 768, NA_LRELU, False, True),
    ("bn", 1, 3840, 768, NA_LRELU, False, True),
    ("bn", 1, 4096, 192, NA_LRELU, False, True),
    ("bn", 1, 4096, 384, NA_LRELU, False, True),
    ("bn", 1, 4096, 768, NA_LRELU, False, True),
    ("bn", 1, 16384, 192, NA_LRELU, False, True),
    ("bn", 1, 16384, 384, NA_LRELU, False, True),
    ("bn", 1, 16384, 768, NA_LRELU, False, True),
    ("bn", 1, 65536, 192, NA_LRELU, False, True),
    ("bn", 1, 65536, 384, NA_LRELU, False, True),
    ("bn", 1, 262144, 192, NA_LRELU, False, True),
    # Step B, batch 16: InstanceNorm
    ("in", 16, 1024, 400, NA_GLU, False, False),        # HmapResBlock conv1 (two halves of 194 -> 200 channels)
    ("in", 16, 4096, 400, NA_GLU, False, False),
    ("in", 16, 16384, 400, NA_GLU, False, False),
    ("in", 16, 1024, 200, NA_NONE, True, False),        # HmapResBlock conv2 + residual
    ("in", 16, 4096, 200, NA_NONE, True, False),
    ("in", 16, 16384, 200, NA_NONE, True, False),
    ("in", 16, 4096, 16, NA_LRELU, False, False),       # heat-map / shape encoders
    ("in", 16, 16384, 16, NA_LRELU, False, False),
    ("in", 16, 65536, 16, NA_LRELU, False, False),
    ("in", 16, 262144, 16, NA_LRELU, False, False),     # object discriminators at 512x512
    ("in", 16, 4096, 24, NA_LRELU, False, False),
    ("in", 16, 16384, 24, NA_LRELU, False, False),
    ("in", 16, 65536, 24, NA_LRELU, False, False),
]

# eval-mode G_NET forward (GSampler) at batch 1 and 16: running statistics, and InstanceNorm with a single image
CASES += [
    ("bn_eval", 1, 1, 24576, NA_GLU, False, True),      # BatchNorm1d at batch 1
    ("bn_eval", 1, 16, 24576, NA_GLU, False, True),
    ("bn_eval", 1, 256, 192, NA_GLU, False, True),
    ("bn_eval", 1, 1024, 96, NA_GLU, False, True),
    ("bn_eval", 1, 4096, 96, NA_GLU, False, True),
    ("bn_eval", 1, 4096, 192, NA_GLU, False, True),
    ("bn_eval", 1, 16384, 96, NA_GLU, False, True),
    ("bn_eval", 1, 65536, 96, NA_GLU, False, True),
    ("bn_eval", 1, 262144, 96, NA_GLU, False, True),
    ("bn_eval", 1, 1048576, 96, NA_GLU, False, True),
    ("in", 1, 1024, 200, NA_NONE, True, False),         # batch 1: one group
    ("in", 1, 4096, 200, NA_NONE, True, False),
    ("in", 1, 16384, 200, NA_NONE, True, False),
    ("in", 1, 4096, 24, NA_LRELU, False, False),
    ("in", 1, 16384, 24, NA_LRELU, False, False),
    ("in", 1, 65536, 24, NA_LRELU, False, False),
]

# rows that pin the kernels' code paths (not shapes the networks issue)
EDGE_CASES = [
    ("in", 1, 1024, 400, NA_GLU, False, False),         # HmapResBlock conv1 at batch 1 (the chains apply it split)
    ("in", 1, 4096, 400, NA_GLU, False, False),
    ("in", 1, 16384, 400, NA_GLU, False, False),
    ("bn", 1, 1, 8, NA_LRELU, False, True),             # P = 1: variance 0, unbiased variance undefined
    ("bn", 1, 7, 12, NA_NONE, False, True),             # P < 8: tail loop only; C/4 = 3
    ("in", 3, 37, 4, NA_LRELU, False, False),           # C/4 = 1, P < 64, P not a multiple of 8
    ("in", 2, 63, 264, NA_GLU, False, False),           # GLU with Co/4 = 33: partial second x block
    ("bn", 1, 200, 132, NA_LRELU, False, True),         # C/4 = 33; one chunk
    ("bn", 1, 1001, 128, NA_NONE, False, True),         # C/4 = 32; odd P
    ("bn", 1, 100003, 256, NA_GLU, False, True),        # many chunks, P prime (tails in every chunk)
    ("in", 64, 1024, 200, NA_NONE, True, False),        # wrapped apply walk: dp > P, dc != 0, many groups per trip
    ("in", 9, 40001, 20, NA_NONE, False, False),        # wrapped walk with C/4 = 5 and P odd: dp > P, dc = 4
    ("bn_eval", 1, 777, 132, NA_LRELU, False, True),    # eval: partial x block, P odd
    ("bn_eval", 1, 300001, 20, NA_NONE, False, True),   # eval: many fixed-order planes
]

# every producer-side operand split of the same runs: the HmapResBlock chains at batch 16 and 1
SPLIT_CASES = [
    (1, 16, 32, 32, 400, NA_GLU, False, 1),
    (1, 16, 32, 32, 200, NA_NONE, True, 1),
    (1, 16, 32, 32, 200, NA_NONE, True, 0),
    (1, 16, 64, 64, 400, NA_GLU, False, 1),
    (1, 16, 64, 64, 200, NA_NONE, True, 1),
    (1, 16, 64, 64, 200, NA_NONE, True, 0),
    (1, 16, 128, 128, 400, NA_GLU, False, 1),
    (1, 16, 128, 128, 200, NA_NONE, True, 1),
    (1, 16, 128, 128, 200, NA_NONE, True, 0),
    (1, 1, 32, 32, 400, NA_GLU, False, 1),
    (1, 1, 32, 32, 200, NA_NONE, True, 1),
    (1, 1, 32, 32, 200, NA_NONE, True, 0),
    (1, 1, 64, 64, 400, NA_GLU, False, 1),
    (1, 1, 64, 64, 200, NA_NONE, True, 1),
    (1, 1, 64, 64, 200, NA_NONE, True, 0),
    (1, 1, 128, 128, 400, NA_GLU, False, 1),
    (1, 1, 128, 128, 200, NA_NONE, True, 1),
    (1, 1, 128, 128, 200, NA_NONE, True, 0),
]

# the combinations the chains do not use
SPLIT_EDGE_CASES = [
    (0, 3, 9, 7, 32, NA_LRELU, False, 1),         # BatchNorm statistics, H, W odd
    (0, 2, 2, 2, 16, NA_GLU, True, 1),            # 2x2 maps: every halo position reflects
    (0, 4, 5, 6, 8, NA_NONE, False, 0),
    (0, 2, 6, 10, 16, NA_GLU, True, 0),           # BatchNorm + GLU with a residual, no halo
    (1, 2, 3, 2, 24, NA_LRELU, True, 0),
    (1, 3, 11, 13, 48, NA_NONE, False, 1),
]


def matches(need, row):
    return all(n is None or n == r for n, r in zip(need, row))


def norm_needs(work):
    """The set of CASES patterns the normalisation calls of a recorded workload (tests/dry.py) need: tuples shaped
    like a CASES row, None where the call does not fix the field; split needs as ("split",) + a SPLIT_CASES row."""
    needs = set()
    kind = None
    for name, a in work.calls:
        if name == "og_norm_stats":                       # x, groups, P, C, eps, stats, mean, rstd, rm, rv, ...
            kind = "bn" if a[8] else "in"
            needs.add((kind, a[1], a[2], a[3], None, None, None))
        elif name == "og_bn_eval_coef":
            kind = "bn_eval"
        elif name == "og_norm_apply":                     # y, groups, P, Cy, mean, rstd, gamma, beta, res, act, ...
            needs.add((kind, a[1], a[2], a[3], a[9], bool(a[8]), bool(a[6])))
        elif name == "og_norm_backward":                  # y, g, groups, P, Cy, mean, rstd, gamma, beta, act, ...
            needs.add(("bn" if a[7] else "in", a[2], a[3], a[4], a[9], None, bool(a[7])))
        elif name == "og_bn_eval_backward":               # y, g, P, Cy, mean, rstd, gamma, beta, act, ...
            needs.add(("bn_eval", 1, a[2], a[3], a[8], None, bool(a[6])))
        elif name == "og_norm_apply_split":               # y, N, H, W, Cy, instance, mean, rstd, gamma, beta, res, act, ..
            needs.add(("split", a[5], a[1], a[2], a[3], a[4], a[11], bool(a[10]), a[15]))
    return needs


def _split_stats(row):
    """The og_norm_stats pattern of a SPLIT_CASES row."""
    instance, n, h, w, cy = row[:5]
    return ("in", n, h * w, cy) if instance else ("bn", 1, n * h * w, cy)


def uncovered(needs):
    """The needs no row covers (split needs are looked up in SPLIT_CASES, and so are the statistics of a split)."""
    split = {("split",) + r for r in SPLIT_CASES}
    split_stats = {_split_stats(r) for r in SPLIT_CASES}

    def covered(n):
        if n[0] == "split":
            return n in split
        return any(matches(n, r) for r in CASES) or (n[4] is None and n[:4] in split_stats)
    return sorted((n for n in needs if not covered(n)), key=str)


def stale(needs):
    """The rows of CASES no normalisation pass (statistics alone do not count) and the rows of SPLIT_CASES no split
    need matches."""
    return ([r for r in CASES if not any(matches(n, r) and n[4] is not None for n in needs)] +
            [r for r in SPLIT_CASES if ("split",) + r not in needs])
