"""Shapes of the DAMSM matching kernels (csrc/words_pairs.cu, csrc/damsm.cu) and of the image encoder's backward
gathers that carry the DAMSM gradient back to the image (csrc/inception.cu), shared by tests/test_gpu_damsm.py (which
runs every row against a float64 restatement) and tests/test_census.py (which checks that the networks issue no
shape missing here).

One table of rows per C entry point:
  og_words_pairs_fwd / og_words_pairs_bwd   (B, NC, ndf, T, S, kind)
      B images x NC captions, ndf channels, T word slots, S regions; kind: "ragged" (caption lengths 1 .. T and one
      above T), "zero" (the same, plus an all-zero word column and an all-zero image: the eps-clamped cosine)
  og_cosine_matrix_fwd / og_cosine_matrix_bwd   (Ba, Bb, D, kind)       kind: "rand", "zero" (one zero row per side)
  og_ce_pair            (B, mask, labels, tie)
      mask: None, "zero" (a mask of zeros) or "class" (same-class pairs, as losses._class_masks builds it); labels:
      "arange" or "perm"; tie: one row of the scores holds an exact tie for its maximum
  og_ce_pair_bwd        (n, g0, g1)               g0 / g1: the scalar is passed (False: a null pointer)
  og_bilinear_bwd_gather  (N, IH, IW, C, OH, OW)  gx (N, IH, IW, C) from g (N, OH, OW, C)
  og_global_avg_bwd     (N, P, C)
  og_relu_grad_slice    (ldy, yoff, ldg, goff, ldo, ooff, nch, P, relu)

CASES holds the rows the networks issue, kept at the size they run: one batch-16 Step-B step with the DAMSM image
encoder attached, and losses.RPrecision(100) scoring a pool (seven batches of 16 added, the eighth scores it).  The
trainer's attention-map snapshot (condGANTrainer.save_img_results) calls og_words_pairs_fwd on the display batch,
which is a training batch: the step's row.  It is not driven here because it needs a whole condGANTrainer with saved
encoder and Inception weights.  EDGE_CASES holds rows that pin the paths and edges the networks do not reach; REFUSED
the argument lists each entry point must refuse before it launches anything.
"""
WP_FWD, WP_BWD = "og_words_pairs_fwd", "og_words_pairs_bwd"
COS_FWD, COS_BWD = "og_cosine_matrix_fwd", "og_cosine_matrix_bwd"
CE, CE_BWD = "og_ce_pair", "og_ce_pair_bwd"
BL_BWD, GAP_BWD, RELU_SLICE = "og_bilinear_bwd_gather", "og_global_avg_bwd", "og_relu_grad_slice"
ENTRIES = (WP_FWD, WP_BWD, COS_FWD, COS_BWD, CE, CE_BWD, BL_BWD, GAP_BWD, RELU_SLICE)

# CNN_ENCODER's conv epilogues, backward through the Inception stem and Mixed_5b .. Mixed_7c at batch 16 (slices of
# the concatenated block outputs: ldy = the block's width, yoff = the branch's first channel)
_RELU_STEP = [
    (32, 0, 32, 0, 32, 0, 32, 355216, 1), (32, 0, 32, 0, 32, 0, 32, 345744, 1), (64, 0, 64, 0, 64, 0, 64, 345744, 1),
    (80, 0, 80, 0, 80, 0, 80, 85264, 1), (192, 0, 192, 0, 192, 0, 192, 80656, 1),
    (64, 0, 64, 0, 64, 0, 64, 19600, 1), (96, 0, 96, 0, 96, 0, 96, 19600, 1), (176, 0, 176, 0, 176, 0, 176, 19600, 1),
    (256, 64, 256, 64, 64, 0, 64, 19600, 1), (256, 128, 256, 128, 96, 0, 96, 19600, 1),
    (256, 224, 256, 224, 32, 0, 32, 19600, 1), (288, 64, 288, 64, 64, 0, 64, 19600, 1),
    (288, 128, 288, 128, 96, 0, 96, 19600, 1), (288, 224, 288, 224, 64, 0, 64, 19600, 1),
    (128, 0, 128, 0, 128, 0, 128, 4624, 1), (160, 0, 160, 0, 160, 0, 160, 4624, 1), (192, 0, 192, 0, 192, 0, 192, 4624, 1),
    (384, 0, 384, 0, 384, 0, 384, 4624, 1), (448, 0, 448, 0, 448, 0, 448, 4624, 1), (512, 0, 512, 0, 512, 0, 512, 4624, 1),
    (576, 0, 576, 0, 576, 0, 576, 4624, 1), (768, 0, 768, 0, 384, 0, 384, 4624, 1),
    (768, 192, 768, 192, 192, 0, 192, 4624, 1), (768, 384, 768, 384, 192, 0, 192, 4624, 1),
    (768, 384, 768, 384, 96, 0, 96, 4624, 1), (768, 576, 768, 576, 192, 0, 192, 4624, 1),
    (256, 0, 256, 0, 256, 0, 256, 4624, 0),                      # the region-feature head (no ReLU)
    (384, 0, 384, 0, 384, 0, 384, 1024, 1), (1152, 0, 1152, 0, 1152, 0, 1152, 1024, 1),
    (1280, 0, 1280, 0, 320, 0, 320, 1024, 1), (1280, 320, 1280, 320, 192, 0, 192, 1024, 1),
    (2048, 320, 2048, 320, 384, 0, 384, 1024, 1), (2048, 704, 2048, 704, 384, 0, 384, 1024, 1),
    (2048, 1088, 2048, 1088, 384, 0, 384, 1024, 1), (2048, 1472, 2048, 1472, 384, 0, 384, 1024, 1),
    (2048, 1856, 2048, 1856, 192, 0, 192, 1024, 1),
]

CASES = {
    # words_loss of the generator step (17 x 17 regions, 18 word slots) and of the R-precision pool of 100
    WP_FWD: [(16, 16, 256, 18, 289, "ragged"), (100, 100, 256, 18, 289, "ragged")],
    WP_BWD: [(16, 16, 256, 18, 289, "ragged")],
    # sent_loss
    COS_FWD: [(16, 16, 256, "rand"), (100, 100, 256, "rand")],
    COS_BWD: [(16, 16, 256, "rand")],
    # the step: no class ids; the pool: the same-class mask, all zero when every class id differs (COCO)
    CE: [(16, None, "arange", False), (100, "zero", "arange", False)],
    CE_BWD: [(256, True, True)],
    # the encoder's input resize 256^2 -> 299^2, its global pool of Mixed_7c, its ReLU epilogues
    BL_BWD: [(16, 256, 256, 8, 299, 299)],
    GAP_BWD: [(16, 64, 2048)],
    RELU_SLICE: _RELU_STEP,
}

EDGE_CASES = {
    WP_FWD: [
        *[(3, 5, 256, T, 289, "ragged") for T in (1, 19, 20, 21, 32)],    # the <20> / <32> templates and their seam
        *[(2, 3, 256, 18, S, "ragged") for S in (1, 31, 160, 161, 320)],  # one / two regions per thread
        (2, 3, 255, 18, 289, "ragged"),      # odd ndf: the last channel pass has no partner channel
        (2, 3, 8, 32, 289, "ragged"),
        (3, 5, 256, 18, 289, "zero"),
        (2, 3, 255, 32, 320, "zero"),
    ],
    WP_BWD: [
        *[(3, 5, 256, T, 289, "ragged") for T in (1, 19, 20, 21, 32)],
        *[(2, 3, 256, 18, S, "ragged") for S in (1, 31, 160, 161, 320)],
        (2, 3, 255, 18, 289, "ragged"),
        (2, 3, 8, 32, 289, "ragged"),
        (3, 5, 256, 18, 289, "zero"),        # 5 captions per image: the atomics sum over several pairs
        (2, 3, 255, 32, 320, "zero"),
    ],
    COS_FWD: [(5, 3, 256, "rand"), (3, 7, 255, "zero"), (1, 1, 8, "rand")],
    COS_BWD: [(5, 3, 256, "rand"), (3, 7, 255, "zero"), (1, 1, 8, "rand")],
    CE: [
        (1, None, "arange", False), (2, None, "arange", False), (127, None, "perm", True),
        (128, None, "arange", True), (128, "class", "perm", False), (16, "zero", "perm", True),
        (16, "class", "arange", True), (100, "class", "arange", False),
    ],
    CE_BWD: [(256, False, True), (256, True, False), (10000, True, True)],
    BL_BWD: [
        (2, 1, 1, 8, 7, 5),                  # IH = IW = 1: every output reads the one input pixel
        (2, 5, 6, 8, 1, 1),                  # OH = OW = 1: the output reads input (0, 0) only
        (2, 17, 17, 8, 17, 17),              # identity
        (2, 299, 299, 8, 17, 17),            # downsampling: rows without a contribution
        (2, 200, 150, 8, 299, 173),          # non-square
        (2, 64, 64, 8, 127, 127),            # r = 63 / 126 = 0.5: r * o lands on integers
        (2, 9, 5, 8, 25, 17),                # r = 1 / 3, 1 / 4
        (16, 200, 200, 8, 299, 299),         # the encoder at 200^2
    ],
    GAP_BWD: [(3, 1, 2048), (2, 5, 8)],
    RELU_SLICE: [
        (64, 16, 64, 32, 48, 8, 16, 1000, 1),   # different slices of y, g and out; out lanes outside stay untouched
        (64, 16, 64, 32, 48, 8, 16, 1000, 0),
        (8, 0, 8, 0, 8, 0, 8, 3, 1),
    ],
}

# argument lists that must be refused with cudaErrorInvalidValue before anything is launched
REFUSED = [
    (WP_FWD, (2, 2, 256, 33, 289)), (WP_FWD, (2, 2, 256, 18, 321)),
    (WP_BWD, (2, 2, 256, 33, 289)), (WP_BWD, (2, 2, 256, 18, 321)),
    (CE, (129,)), (CE, (0,)),
]


def _key(entry, row):
    """The fields of a row that a library call fixes (og_ce_pair: whether a mask is passed, not what it holds)"""
    if entry == CE:
        return (row[0], row[1] is not None)
    if entry in (WP_FWD, WP_BWD, COS_FWD, COS_BWD):
        return tuple(row[:-1])
    return tuple(row)


def damsm_needs(work):
    """The set of (entry, key) pairs the DAMSM and encoder-gather calls of a recorded workload (tests/dry.py) need,
    keys as ``_key`` gives them for a row."""
    needs = set()
    for name, a in work.calls:
        if name == WP_FWD:           # words, ctx, lens, B, NC, ndf, T, S, gamma1, gamma2, eps, wc, attn, sim
            needs.add((name, tuple(a[3:8])))
        elif name == WP_BWD:         # words, ctx, lens, wc, attn, g_sim, B, NC, ndf, T, S, gamma1, gamma2, eps, g_ctx
            needs.add((name, tuple(a[6:11])))
        elif name == COS_FWD:        # a, b, Ba, Bb, D, eps, out
            needs.add((name, tuple(a[2:5])))
        elif name == COS_BWD:        # a, b, g, Ba, Bb, D, eps, ga
            needs.add((name, tuple(a[3:6])))
        elif name == CE:             # sim, mask, labels, B, gamma3, loss0, loss1, G0, G1, correct
            needs.add((name, (a[3], bool(a[1]))))
        elif name == CE_BWD:         # G0, G1, g0, g1, n, gsim
            needs.add((name, (a[4], bool(a[2]), bool(a[3]))))
        elif name == BL_BWD:         # g, N, IH, IW, C, OH, OW, gx
            needs.add((name, tuple(a[1:7])))
        elif name == GAP_BWD:        # g, N, P, C, gx
            needs.add((name, tuple(a[1:4])))
        elif name == RELU_SLICE:     # y, ldy, yoff, g, ldg, goff, out, ldo, ooff, nch, P, relu
            needs.add((name, tuple(a[1:3]) + tuple(a[4:6]) + tuple(a[7:12])))
    return needs


def uncovered(needs):
    """The needs no CASES row covers."""
    return sorted((n for n in needs if not any(_key(n[0], r) == n[1] for r in CASES[n[0]])), key=str)


def stale(needs):
    """The CASES rows no need matches."""
    return [(e, r) for e in ENTRIES for r in CASES[e] if (e, _key(e, r)) not in needs]
