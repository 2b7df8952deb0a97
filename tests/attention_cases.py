"""Shapes of the attention and mask-paint kernels (csrc/attention.cu, csrc/attention_tc.cu), shared by
tests/test_gpu_attention.py (which runs every row against a float64 restatement) and tests/test_census.py
(which checks that the networks issue no shape missing here).

One table of rows per C entry point:
  og_att_general_fwd / og_att_general_bwd   (B, Q, idf, cs, L, mask)
      Q = H*W queries, idf real channels of the NHWC rows of stride cs, L words; mask: a caption mask is passed (for
      the backward: the probabilities it reads were computed under one)
  og_bu_att_fwd / og_bu_att_bwd             (B, E, R, L, idf, norm)      E GloVe dims, R roi slots, norm: cosine
  og_paint_max_fwd / og_paint_max_bwd       (B, num, R, Rtot, P, stride, off)
      num channels painted at lane offset off of NHWC rows of `stride` lanes, R of the Rtot mask slots used
  og_words_proj / og_words_proj_bwd         (B, idf, cdf, L)

CASES holds the rows the networks issue (one batch-16 Step-B step, eval-mode G_NET at batch 1 and 16), kept at the size
they run.  EDGE_CASES holds rows that pin the dispatch branches and code paths the networks do not reach.  A field of an
EDGE_CASES row may be a string naming a batch size that depends on the device's SM count (see batch_for).
"""
FWD, BWD = "og_att_general_fwd", "og_att_general_bwd"
BU_FWD, BU_BWD = "og_bu_att_fwd", "og_bu_att_bwd"
PAINT_FWD, PAINT_BWD = "og_paint_max_fwd", "og_paint_max_bwd"
PROJ, PROJ_BWD = "og_words_proj", "og_words_proj_bwd"
ENTRIES = (FWD, BWD, BU_FWD, BU_BWD, PAINT_FWD, PAINT_BWD, PROJ, PROJ_BWD)

CASES = {
    # ATT_NET of the three generator stages: 64x64 and 128x128 maps, 18-word captions
    FWD: [(B, Q, 48, 48, 18, True) for B in (1, 16) for Q in (4096, 16384)],
    BWD: [(16, Q, 48, 48, 18, True) for Q in (4096, 16384)],
    # BT_ATT_NET: 10 roi slots
    BU_FWD: [(B, 50, 10, 18, 48, True) for B in (1, 16)],
    BU_BWD: [(16, 50, 10, 18, 48, True)],
    # pprocess_bt_attns: 18 / 48 / 50 channels (padded to 24 / 48 / 56 lanes) at 32x32, 64x64, 128x128
    PAINT_FWD: [(B, num, 10, 10, P, stride, 0) for B in (1, 16) for num, stride in ((18, 24), (48, 48), (50, 56))
                for P in (1024, 4096, 16384)],
    PAINT_BWD: [(16, 48, 10, 10, P, 48, 0) for P in (1024, 4096, 16384)],
    PROJ: [(B, 48, 256, 18) for B in (1, 16)],
    PROJ_BWD: [(16, 48, 256, 18)],
}

# batch sizes that set the tensor-core kernels' CTA count per image (nslots) against the Q / 128 query tiles; resolved
# on the device by batch_for
NSLOTS_EQ, NSLOTS_DIV, NSLOTS_NDIV, BWD_ONE_SLOT = "nslots=ntiles", "nslots|ntiles", "nslots!|ntiles", "bwd nslots=1"
AT_FWD_CTAS, AT_BWD_CTAS = 3, 2          # CTAs per SM of the forward / backward tensor-core kernels (attention_tc.cu)

EDGE_CASES = {
    FWD: [
        # tensor cores, <20> template: every caption length up to 20, ragged masks on odd batches (mask row wraps)
        *[(3, 4096, 48, 48, L, True) for L in (1, 2, 7, 12, 17, 18, 19, 20)],
        # <32> template
        *[(3, 4096, 48, 48, L, True) for L in (21, 25, 32)],
        (10, 4096 + 128, 48, 48, 18, True),    # Q = 4096 + 128: 33 tiles
        (100, 4096, 48, 48, 18, True),         # nslots = 3 (132 SMs): mstep = 384 mod 100 != 0
        (128, 4096, 48, 48, 13, True),         # the largest batch the mask bit table holds
        (7, 4096, 48, 48, 18, False),          # no mask
        (NSLOTS_EQ, 4096, 48, 48, 18, True),
        (NSLOTS_DIV, 4096, 48, 48, 18, True),
        (NSLOTS_NDIV, 4096, 48, 48, 18, True),
        # SIMT
        (3, 3968, 48, 48, 18, True),           # Q % 128 == 0 below the Q >= 4096 gate: <20>
        (3, 4160, 48, 48, 18, True),           # Q % 128 != 0: <20> above the gate
        (129, 4096, 48, 48, 18, True),         # B > 128: <20>
        (2, 4096, 32, 32, 18, True),           # C = 32: <20>
        (3, 4160, 48, 48, 32, True),           # <LMAX> above the gate
        (3, 1000, 48, 48, 21, True),           # <LMAX>
        (3, 1000, 48, 48, 32, True),
        (2, 4096, 72, 80, 18, True),           # idf > 64, cs != idf: <20>, pad lanes
        (2, 1000, 72, 80, 18, True),           # idf > 64 on <20> below the gate
    ],
    BWD: [
        *[(3, 4096, 48, 48, L, True) for L in (1, 7, 18, 20, 21, 32)],
        (10, 4096 + 128, 48, 48, 18, True),
        (100, 4096, 48, 48, 18, True),
        (BWD_ONE_SLOT, 4096, 48, 48, 18, True),   # nslots == 1: g_src stored without the workspace planes
        (3, 3968, 48, 48, 18, True),           # SIMT bwd20
        (3, 100, 48, 48, 18, True),            # ... one CTA per image: g_src stored without the workspace planes
        (3, 4160, 48, 48, 18, True),           # Q % 128 != 0: bwd20 above the Q >= 4096 gate
        (3, 1000, 48, 48, 18, False),
        (3, 1000, 48, 48, 21, True),           # the general kernel: L > 20
        (3, 1000, 48, 48, 32, True),
        (2, 128, 48, 48, 21, True),            # ... one CTA per image
        (2, 1000, 72, 80, 18, True),           # ... idf > 64
        (2, 4096, 72, 80, 12, True),           # ... above the gate
    ],
    BU_FWD: [(B, 50, R, L, 48, norm) for B, R, L in ((3, 10, 18), (3, 1, 7), (4, 1, 18), (16, 10, 12))
             for norm in (True, False)],
    BU_BWD: [(3, 50, 10, 18, 48, None), (3, 50, 1, 7, 48, None)],
    PAINT_FWD: [
        (2, 18, 0, 10, 1024, 24, 0),                  # R = 0: the memset path
        (2, 18, 1, 10, 1000, 24, 0),                  # R = 1, P not a multiple of the pixel tile
        (3, 13, 4, 6, 777, 20, 4),                    # num % 4 != 0 at an offset: pad lanes [17, 20) zeroed
        (2, 13, 4, 6, 777, 20, 3),                    # off % 4 != 0: the scalar kernel
        (2, 48, 70, 70, 300, 48, 0),                  # shared memory of the vectorised kernel > 48 KB: scalar
        (2, 48, 128, 128, 300, 48, 0),                # ... and of the scalar kernel too (57 KB)
        (2, 18, 0, 10, 300, 24, 3),                   # R = 0 at an odd offset
    ],
    PAINT_BWD: [
        (2, 18, 10, 10, 64, 24, 0),                   # one block: no split sum
        (2, 13, 1, 6, 777, 20, 3),                    # R = 1, odd offset and stride
        (3, 48, 10, 10, 4096, 56, 4),
        (2, 18, 0, 10, 1024, 24, 0),                  # R = 0: zeros
    ],
    PROJ: [(3, 48, 256, 1), (3, 48, 256, 32), (2, 72, 100, 13)],
    PROJ_BWD: [(3, 48, 256, 1), (3, 48, 256, 32), (2, 72, 100, 13)],
}


def batch_for(tag, Q, sms):
    """The batch size a tag of an EDGE_CASES row stands for on a device with `sms` SMs.  The forward launches
    nslots = min(3 sms / B, Q / 128) CTAs per image, the backward max(1, min(2 sms / B, Q / 128))."""
    if not isinstance(tag, str):
        return tag
    ntiles = Q // 128
    fwd = lambda B: min(AT_FWD_CTAS * sms // B, ntiles)   # noqa: E731
    if tag == NSLOTS_EQ:
        want = lambda n: n == ntiles                      # noqa: E731
    elif tag == NSLOTS_DIV:
        want = lambda n: 1 < n < ntiles and ntiles % n == 0   # noqa: E731
    elif tag == NSLOTS_NDIV:
        want = lambda n: 1 < n < ntiles and ntiles % n != 0   # noqa: E731
    elif tag == BWD_ONE_SLOT:
        return AT_BWD_CTAS * sms + 1
    else:
        raise ValueError(tag)
    # the largest such batch whose mask-row step nslots * 128 mod B is not 0 (the kernel's incremental advance)
    return max(B for B in range(2, 129) if want(fwd(B)) and fwd(B) * 128 % B)


def matches(need, row):
    return all(n is None or n == r for n, r in zip(need, row))


def att_needs(work):
    """The set of (entry, pattern) pairs the attention, paint and word-projection calls of a recorded workload
    (tests/dry.py) need: patterns shaped like a row of that entry's table, None where the call does not fix the
    field."""
    needs = set()
    for name, a in work.calls:
        if name == FWD:          # h, src, mask, B, Q, idf, cs, L, wc, attn
            needs.add((name, (a[3], a[4], a[5], a[6], a[7], bool(a[2]))))
        elif name == BWD:        # h, src, attn, g_wc, B, Q, idf, cs, L, g_h, g_src
            needs.add((name, (a[4], a[5], a[6], a[7], a[8], None)))
        elif name == BU_FWD:     # labels, glove, src, mask, B, E, R, L, idf, norm, eps, wc, attn
            needs.add((name, (a[4], a[5], a[6], a[7], a[8], bool(a[9]))))
        elif name == BU_BWD:     # attn, g_wc, B, R, L, idf, g_src
            needs.add((name, (a[2], None, a[3], a[4], a[5], None)))
        elif name == PAINT_FWD:  # f, m, B, num, R, Rtot, P, out, stride, off
            needs.add((name, (a[2], a[3], a[4], a[5], a[6], a[8], a[9])))
        elif name == PAINT_BWD:  # f, m, g, gstride, goff, B, num, R, Rtot, P, g_f
            needs.add((name, (a[5], a[6], a[7], a[8], a[9], a[3], a[4])))
        elif name == PROJ:       # words, W, B, idf, cdf, L, src
            needs.add((name, (a[2], a[3], a[4], a[5])))
        elif name == PROJ_BWD:   # words, W, gsrc, B, idf, cdf, L, gW, accumulate, gwords
            needs.add((name, (a[3], a[4], a[5], a[6])))
    return needs


def uncovered(needs):
    """The needs no CASES row covers."""
    return sorted((n for n in needs if not any(matches(n[1], r) for r in CASES[n[0]])), key=str)


def stale(needs):
    """The CASES rows no need matches."""
    return [(e, r) for e in ENTRIES for r in CASES[e] if not any(n[0] == e and matches(n[1], r) for n in needs)]
