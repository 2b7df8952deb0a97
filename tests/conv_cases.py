"""Shapes of the convolutions (csrc/conv_tc.cu, conv_simt.cu, wgmma.cuh), shared by tests/test_gpu_conv.py (which runs
every row against float64 on both engines) and tests/test_census.py (which checks that the networks issue no shape
missing here, that no row is stale, and that each row's path is the one the GPU takes).

A CASES / EDGE_CASES row is (N, H, W, Cin, Cout, k, stride, pad, mode, act, bias, split, path):
  N, H, W, Cin  the input (N, H, W, cpad(Cin)) NHWC;  Cout, k  the OIHW weight (Cout, Cin, k, k)
  stride, pad   as nn.Conv2d;  mode  lib.PAD_ZERO / PAD_REFLECT / UPSAMPLE2X (nearest 2x upsample, then the conv)
  act           lib.ACT_NONE / ACT_LRELU / ACT_TANH / ACT_SIGMOID, applied in the epilogue
  bias          a bias is added in the epilogue;  split  GLU halves: Cout = 2 split, each half padded to cpad(split)
  path          the path the f16x3 engine takes (ops.conv_path): "s1" / "s2" (tensor cores), "narrow" (8 padded output
                channels on small maps: og_conv2d_narrow_*), "simt" (og_conv2d_simt / og_conv2d_wgrad_simt)
An ENC_CASES row is (dir, N, H, W, Cin, Cout, kh, kw, stride, padh, padw, relu, bias, yoff, Cy, path): one call of
ops.enc_conv_fwd (dir "fwd": output channels [yoff, yoff + Cout) of a Cy-channel destination) or ops.enc_conv_dgrad
(dir "dgrad": yoff 0, Cy = cpad(Cin), the input gradient); path "tc" or "simt" (ops.conv_path).
Rows are kept at the size the networks run them (no batch is cut), so a shape the networks issue must be in the table
as it stands.
"""
from objgan_b200.lib import ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, PAD_REFLECT, PAD_ZERO, UPSAMPLE2X

Z, R, U = PAD_ZERO, PAD_REFLECT, UPSAMPLE2X

# every distinct shape of one batch-16 StepBTrainer.step (DAMSM image encoder attached) and of an eval-mode G_NET
# forward at batch 1 and 16
CASES = [
    # Step B, batch 16 (the roi heads run on 15 / 16 / 48 / 49 / 160 rows)
    (15, 4, 4, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (15, 8, 8, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (15, 16, 16, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (16, 4, 4, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (16, 8, 8, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (16, 16, 16, 768, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (48, 4, 4, 384, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (49, 4, 4, 384, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, 'narrow'),
    (15, 8, 8, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (15, 16, 16, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (16, 4, 4, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (16, 8, 8, 192, 192, 3, 1, 1, U, ACT_NONE, False, 96, 's1'),
    (16, 8, 8, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (16, 16, 16, 96, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (16, 16, 16, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (16, 32, 32, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (16, 32, 32, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (16, 32, 32, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (16, 64, 64, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (16, 64, 64, 80, 12, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 64, 64, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 64, 64, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (16, 64, 64, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (16, 64, 64, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (16, 128, 128, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (16, 128, 128, 80, 12, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 128, 128, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 128, 128, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (16, 128, 128, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (16, 128, 128, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (16, 256, 256, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (16, 256, 256, 80, 12, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 256, 256, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (16, 512, 512, 80, 12, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (48, 4, 4, 482, 384, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (49, 4, 4, 482, 384, 3, 1, 1, Z, ACT_NONE, False, 0, 's1'),
    (160, 5, 5, 384, 384, 4, 1, 1, Z, ACT_LRELU, True, 0, 's1'),
    (160, 5, 5, 768, 384, 4, 1, 1, Z, ACT_LRELU, True, 0, 's1'),
    (16, 8, 8, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 16, 16, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 16, 16, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 32, 32, 96, 192, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 32, 32, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 32, 32, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 64, 64, 3, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 64, 64, 15, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 64, 64, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 64, 64, 96, 192, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 64, 64, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 64, 64, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 128, 128, 3, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 128, 128, 15, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 128, 128, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 128, 128, 96, 192, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 128, 128, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 256, 256, 3, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 256, 256, 15, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 256, 256, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (16, 256, 256, 96, 192, 4, 2, 1, Z, ACT_NONE, False, 0, 's2'),
    (16, 512, 512, 15, 96, 4, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (15, 4, 4, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, 'simt'),
    (16, 1, 1, 200, 24576, 1, 1, 0, Z, ACT_NONE, False, 12288, 'simt'),
    (16, 1, 1, 256, 400, 1, 1, 0, Z, ACT_NONE, True, 200, 'simt'),
    (16, 1, 1, 2048, 256, 1, 1, 0, Z, ACT_NONE, True, 0, 'simt'),
    # eval-mode G_NET at batch 1 (batch 16 issues no shape the step does not)
    (1, 8, 8, 192, 192, 3, 1, 1, U, ACT_NONE, False, 96, 's1'),
    (1, 16, 16, 96, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (1, 32, 32, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (1, 32, 32, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (1, 32, 32, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (1, 64, 64, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (1, 64, 64, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (1, 64, 64, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (1, 64, 64, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (1, 64, 64, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (1, 128, 128, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (1, 128, 128, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (1, 128, 128, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, 's1'),
    (1, 128, 128, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, 's1'),
    (1, 128, 128, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, 's1'),
    (1, 256, 256, 48, 3, 3, 1, 1, Z, ACT_TANH, False, 0, 's1'),
    (1, 256, 256, 80, 24, 3, 1, 1, R, ACT_NONE, True, 0, 's1'),
    (1, 64, 64, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (1, 128, 128, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (1, 256, 256, 24, 48, 3, 2, 1, Z, ACT_LRELU, False, 0, 's2'),
    (1, 1, 1, 200, 24576, 1, 1, 0, Z, ACT_NONE, False, 12288, 'simt'),
    (1, 1, 1, 256, 400, 1, 1, 0, Z, ACT_NONE, True, 200, 'simt'),
    # INCEPTION_V3's classifier
    (16, 1, 1, 2048, 1000, 1, 1, 0, Z, ACT_NONE, True, 0, 'simt'),
]

# rows that pin code paths the networks do not reach on their own
EDGE_CASES = [
    # SIMT (og_conv2d_simt): TN = 2 / 4 / 8 (<= 32, <= 64, > 64 padded output channels), split-K (no bias, no
    # activation, few tiles) and the single-pass epilogue
    (2, 6, 6, 40, 24, 3, 1, 1, Z, ACT_NONE, False, 0, "simt"),
    (2, 6, 6, 40, 20, 3, 1, 1, Z, ACT_LRELU, True, 0, "simt"),
    (3, 5, 7, 64, 48, 3, 1, 1, Z, ACT_NONE, False, 0, "simt"),
    (3, 5, 7, 64, 44, 3, 1, 1, Z, ACT_TANH, True, 0, "simt"),
    (2, 8, 8, 256, 96, 3, 1, 1, Z, ACT_NONE, False, 0, "simt"),
    (2, 8, 8, 64, 72, 3, 1, 1, Z, ACT_SIGMOID, True, 0, "simt"),
    # SIMT reflection and upsample addressing on maps under TC_MIN_PIXELS, GLU halves through the upsample
    (2, 7, 9, 24, 40, 3, 1, 1, R, ACT_NONE, False, 0, "simt"),
    (1, 6, 5, 32, 16, 3, 1, 1, U, ACT_NONE, False, 8, "simt"),
    (2, 3, 4, 48, 40, 3, 1, 1, U, ACT_NONE, False, 20, "simt"),
    # SIMT stride 2: the input gradient is a stride-2 TRANSPOSED convolution; odd maps never take the tc phases
    (2, 10, 10, 16, 32, 4, 2, 1, Z, ACT_LRELU, True, 0, "simt"),
    (4, 33, 33, 24, 48, 3, 2, 1, Z, ACT_NONE, False, 0, "simt"),
    # narrow: short-reduction forward (k k C / 4 < 512), tanh and sigmoid epilogues, wgrad with one pixel slice and
    # with many
    (4, 8, 8, 24, 1, 4, 2, 0, Z, ACT_SIGMOID, True, 0, "narrow"),
    (2, 8, 8, 16, 3, 3, 1, 1, Z, ACT_TANH, True, 0, "narrow"),
    (1, 6, 6, 16, 1, 4, 2, 0, Z, ACT_NONE, False, 0, "narrow"),
    (8, 34, 34, 8, 2, 4, 2, 0, Z, ACT_LRELU, True, 0, "narrow"),
    # tensor cores: split reduction at exactly TC_MIN_PIXELS, stacked [w_hi | w_lo] tiles at <= 16 and 17..32
    # output channels, every activation of the epilogue with a bias
    (1, 16, 16, 256, 64, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (2, 32, 32, 64, 16, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (2, 32, 32, 64, 30, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (2, 16, 16, 32, 40, 3, 1, 1, R, ACT_TANH, True, 0, "s1"),
    (2, 16, 16, 32, 40, 3, 1, 1, Z, ACT_SIGMOID, True, 0, "s1"),
    (2, 16, 16, 32, 40, 3, 1, 1, Z, ACT_LRELU, True, 0, "s1"),
    (4, 32, 32, 16, 64, 4, 2, 1, Z, ACT_SIGMOID, True, 0, "s2"),
    (4, 32, 32, 16, 24, 3, 2, 1, Z, ACT_TANH, True, 0, "s2"),
    # hand-picked tensor-core geometry: ragged tiles, several N tiles, batches that do not fill the last pixel tile or
    # wgrad image group (N % cn != 0), reflection halos on narrow maps, 3 / 15 channel sources and destinations
    (2, 64, 64, 194, 388, 3, 1, 1, R, ACT_NONE, False, 194, "s1"),
    (4, 32, 64, 194, 194, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (2, 64, 64, 194, 96, 3, 1, 1, U, ACT_NONE, False, 48, "s1"),
    (36, 16, 16, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (2, 80, 72, 64, 48, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (5, 48, 48, 40, 24, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (8, 16, 16, 1024, 768, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (4, 64, 64, 96, 192, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (8, 32, 32, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (32, 16, 16, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (2, 64, 64, 48, 3, 3, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (4, 64, 64, 3, 96, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (2, 64, 64, 80, 24, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (32, 8, 8, 768, 1536, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (4, 16, 16, 40, 24, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (4, 64, 64, 24, 48, 3, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (130, 5, 5, 384, 384, 4, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (70, 5, 5, 384, 384, 4, 1, 1, Z, ACT_NONE, False, 0, "s1"),
    (13, 16, 16, 192, 384, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (19, 8, 8, 384, 768, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
    (3, 8, 8, 96, 48, 3, 1, 1, U, ACT_NONE, False, 24, "s1"),
    (2, 128, 128, 80, 12, 3, 1, 1, R, ACT_NONE, False, 0, "s1"),
    (2, 128, 128, 15, 96, 4, 2, 1, Z, ACT_NONE, False, 0, "s2"),
]

# every EncConv call of CNN_ENCODER's forward and input gradient on the step's 256x256 images at batch 16, and of the
# INCEPTION_V3 and INCEPTION_V3_FID forwards at batch 16
ENC_CASES = [
    ('dgrad', 16, 299, 299, 3, 32, 3, 3, 2, 0, 0, True, True, 0, 8, 'tc'),
    ('dgrad', 16, 149, 149, 32, 32, 3, 3, 1, 0, 0, True, True, 0, 32, 'tc'),
    ('dgrad', 16, 147, 147, 32, 64, 3, 3, 1, 1, 1, True, True, 0, 32, 'tc'),
    ('dgrad', 16, 73, 73, 64, 80, 1, 1, 1, 0, 0, True, True, 0, 64, 'tc'),
    ('dgrad', 16, 73, 73, 80, 192, 3, 3, 1, 0, 0, True, True, 0, 80, 'tc'),
    ('dgrad', 16, 35, 35, 48, 64, 5, 5, 1, 2, 2, True, True, 0, 48, 'tc'),
    ('dgrad', 16, 35, 35, 64, 96, 3, 3, 1, 1, 1, True, True, 0, 64, 'tc'),
    ('dgrad', 16, 35, 35, 96, 96, 3, 3, 1, 1, 1, True, True, 0, 96, 'tc'),
    ('dgrad', 16, 35, 35, 96, 96, 3, 3, 2, 0, 0, True, True, 0, 96, 'tc'),
    ('dgrad', 16, 35, 35, 192, 32, 1, 1, 1, 0, 0, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 35, 35, 192, 176, 1, 1, 1, 0, 0, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 35, 35, 256, 64, 1, 1, 1, 0, 0, True, True, 0, 256, 'tc'),
    ('dgrad', 16, 35, 35, 256, 176, 1, 1, 1, 0, 0, True, True, 0, 256, 'tc'),
    ('dgrad', 16, 35, 35, 288, 64, 1, 1, 1, 0, 0, True, True, 0, 288, 'tc'),
    ('dgrad', 16, 35, 35, 288, 176, 1, 1, 1, 0, 0, True, True, 0, 288, 'tc'),
    ('dgrad', 16, 35, 35, 288, 384, 3, 3, 2, 0, 0, True, True, 0, 288, 'tc'),
    ('dgrad', 16, 17, 17, 128, 128, 1, 7, 1, 0, 3, True, True, 0, 128, 'tc'),
    ('dgrad', 16, 17, 17, 128, 128, 7, 1, 1, 3, 0, True, True, 0, 128, 'tc'),
    ('dgrad', 16, 17, 17, 128, 192, 1, 7, 1, 0, 3, True, True, 0, 128, 'tc'),
    ('dgrad', 16, 17, 17, 128, 192, 7, 1, 1, 3, 0, True, True, 0, 128, 'tc'),
    ('dgrad', 16, 17, 17, 160, 160, 1, 7, 1, 0, 3, True, True, 0, 160, 'tc'),
    ('dgrad', 16, 17, 17, 160, 160, 7, 1, 1, 3, 0, True, True, 0, 160, 'tc'),
    ('dgrad', 16, 17, 17, 160, 192, 1, 7, 1, 0, 3, True, True, 0, 160, 'tc'),
    ('dgrad', 16, 17, 17, 160, 192, 7, 1, 1, 3, 0, True, True, 0, 160, 'tc'),
    ('dgrad', 16, 17, 17, 192, 192, 1, 7, 1, 0, 3, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 17, 17, 192, 192, 3, 3, 2, 0, 0, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 17, 17, 192, 192, 7, 1, 1, 3, 0, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 17, 17, 192, 320, 3, 3, 2, 0, 0, True, True, 0, 192, 'tc'),
    ('dgrad', 16, 17, 17, 768, 192, 1, 1, 1, 0, 0, True, True, 0, 768, 'tc'),
    ('dgrad', 16, 17, 17, 768, 256, 1, 1, 1, 0, 0, False, False, 0, 768, 'tc'),
    ('dgrad', 16, 17, 17, 768, 384, 1, 1, 1, 0, 0, True, True, 0, 768, 'tc'),
    ('dgrad', 16, 17, 17, 768, 448, 1, 1, 1, 0, 0, True, True, 0, 768, 'tc'),
    ('dgrad', 16, 17, 17, 768, 512, 1, 1, 1, 0, 0, True, True, 0, 768, 'tc'),
    ('dgrad', 16, 17, 17, 768, 576, 1, 1, 1, 0, 0, True, True, 0, 768, 'tc'),
    ('dgrad', 16, 8, 8, 384, 384, 1, 3, 1, 0, 1, True, True, 0, 384, 'tc'),
    ('dgrad', 16, 8, 8, 384, 384, 3, 1, 1, 1, 0, True, True, 0, 384, 'tc'),
    ('dgrad', 16, 8, 8, 448, 384, 3, 3, 1, 1, 1, True, True, 0, 448, 'tc'),
    ('dgrad', 16, 8, 8, 1280, 192, 1, 1, 1, 0, 0, True, True, 0, 1280, 'tc'),
    ('dgrad', 16, 8, 8, 1280, 1152, 1, 1, 1, 0, 0, True, True, 0, 1280, 'tc'),
    ('dgrad', 16, 8, 8, 2048, 192, 1, 1, 1, 0, 0, True, True, 0, 2048, 'tc'),
    ('dgrad', 16, 8, 8, 2048, 1152, 1, 1, 1, 0, 0, True, True, 0, 2048, 'tc'),
    ('fwd', 16, 299, 299, 3, 32, 3, 3, 2, 0, 0, True, True, 0, 32, 'tc'),
    ('fwd', 16, 149, 149, 32, 32, 3, 3, 1, 0, 0, True, True, 0, 32, 'tc'),
    ('fwd', 16, 147, 147, 32, 64, 3, 3, 1, 1, 1, True, True, 0, 64, 'tc'),
    ('fwd', 16, 73, 73, 64, 80, 1, 1, 1, 0, 0, True, True, 0, 80, 'tc'),
    ('fwd', 16, 73, 73, 80, 192, 3, 3, 1, 0, 0, True, True, 0, 192, 'tc'),
    ('fwd', 16, 35, 35, 48, 64, 5, 5, 1, 2, 2, True, True, 64, 256, 'tc'),
    ('fwd', 16, 35, 35, 48, 64, 5, 5, 1, 2, 2, True, True, 64, 288, 'tc'),
    ('fwd', 16, 35, 35, 64, 96, 3, 3, 1, 1, 1, True, True, 0, 96, 'tc'),
    ('fwd', 16, 35, 35, 96, 96, 3, 3, 1, 1, 1, True, True, 128, 256, 'tc'),
    ('fwd', 16, 35, 35, 96, 96, 3, 3, 1, 1, 1, True, True, 128, 288, 'tc'),
    ('fwd', 16, 35, 35, 96, 96, 3, 3, 2, 0, 0, True, True, 384, 768, 'tc'),
    ('fwd', 16, 35, 35, 192, 32, 1, 1, 1, 0, 0, True, True, 224, 256, 'tc'),
    ('fwd', 16, 35, 35, 192, 176, 1, 1, 1, 0, 0, True, True, 0, 176, 'tc'),
    ('fwd', 16, 35, 35, 256, 64, 1, 1, 1, 0, 0, True, True, 224, 288, 'tc'),
    ('fwd', 16, 35, 35, 256, 176, 1, 1, 1, 0, 0, True, True, 0, 176, 'tc'),
    ('fwd', 16, 35, 35, 288, 64, 1, 1, 1, 0, 0, True, True, 0, 64, 'tc'),
    ('fwd', 16, 35, 35, 288, 64, 1, 1, 1, 0, 0, True, True, 224, 288, 'tc'),
    ('fwd', 16, 35, 35, 288, 176, 1, 1, 1, 0, 0, True, True, 0, 176, 'tc'),
    ('fwd', 16, 35, 35, 288, 384, 3, 3, 2, 0, 0, True, True, 0, 768, 'tc'),
    ('fwd', 16, 17, 17, 128, 128, 1, 7, 1, 0, 3, True, True, 0, 128, 'tc'),
    ('fwd', 16, 17, 17, 128, 128, 7, 1, 1, 3, 0, True, True, 0, 128, 'tc'),
    ('fwd', 16, 17, 17, 128, 192, 1, 7, 1, 0, 3, True, True, 384, 768, 'tc'),
    ('fwd', 16, 17, 17, 128, 192, 7, 1, 1, 3, 0, True, True, 192, 768, 'tc'),
    ('fwd', 16, 17, 17, 160, 160, 1, 7, 1, 0, 3, True, True, 0, 160, 'tc'),
    ('fwd', 16, 17, 17, 160, 160, 7, 1, 1, 3, 0, True, True, 0, 160, 'tc'),
    ('fwd', 16, 17, 17, 160, 192, 1, 7, 1, 0, 3, True, True, 384, 768, 'tc'),
    ('fwd', 16, 17, 17, 160, 192, 7, 1, 1, 3, 0, True, True, 192, 768, 'tc'),
    ('fwd', 16, 17, 17, 192, 192, 1, 7, 1, 0, 3, True, True, 0, 192, 'tc'),
    ('fwd', 16, 17, 17, 192, 192, 1, 7, 1, 0, 3, True, True, 384, 768, 'tc'),
    ('fwd', 16, 17, 17, 192, 192, 3, 3, 2, 0, 0, True, True, 320, 1280, 'tc'),
    ('fwd', 16, 17, 17, 192, 192, 7, 1, 1, 3, 0, True, True, 0, 192, 'tc'),
    ('fwd', 16, 17, 17, 192, 192, 7, 1, 1, 3, 0, True, True, 192, 768, 'tc'),
    ('fwd', 16, 17, 17, 192, 320, 3, 3, 2, 0, 0, True, True, 0, 1280, 'tc'),
    ('fwd', 16, 17, 17, 768, 192, 1, 1, 1, 0, 0, True, True, 576, 768, 'tc'),
    ('fwd', 16, 17, 17, 768, 256, 1, 1, 1, 0, 0, False, False, 0, 256, 'tc'),
    ('fwd', 16, 17, 17, 768, 384, 1, 1, 1, 0, 0, True, True, 0, 384, 'tc'),
    ('fwd', 16, 17, 17, 768, 448, 1, 1, 1, 0, 0, True, True, 0, 448, 'tc'),
    ('fwd', 16, 17, 17, 768, 512, 1, 1, 1, 0, 0, True, True, 0, 512, 'tc'),
    ('fwd', 16, 17, 17, 768, 576, 1, 1, 1, 0, 0, True, True, 0, 576, 'tc'),
    ('fwd', 16, 8, 8, 384, 384, 1, 3, 1, 0, 1, True, True, 320, 2048, 'tc'),
    ('fwd', 16, 8, 8, 384, 384, 1, 3, 1, 0, 1, True, True, 1088, 2048, 'tc'),
    ('fwd', 16, 8, 8, 384, 384, 3, 1, 1, 1, 0, True, True, 704, 2048, 'tc'),
    ('fwd', 16, 8, 8, 384, 384, 3, 1, 1, 1, 0, True, True, 1472, 2048, 'tc'),
    ('fwd', 16, 8, 8, 448, 384, 3, 3, 1, 1, 1, True, True, 0, 384, 'tc'),
    ('fwd', 16, 8, 8, 1280, 192, 1, 1, 1, 0, 0, True, True, 1856, 2048, 'tc'),
    ('fwd', 16, 8, 8, 1280, 1152, 1, 1, 1, 0, 0, True, True, 0, 1152, 'tc'),
    ('fwd', 16, 8, 8, 2048, 192, 1, 1, 1, 0, 0, True, True, 1856, 2048, 'tc'),
    ('fwd', 16, 8, 8, 2048, 1152, 1, 1, 1, 0, 0, True, True, 0, 1152, 'tc'),
]


def path_of(N, H, W, Cin, Cout, k, stride, pad, mode, split):
    """The path the f16x3 engine takes for this layer (ops.conv_path)."""
    from objgan_b200 import ops
    from objgan_b200.ops import cpad
    kp = 2 * cpad(split) if split else cpad(Cout)
    return ops.conv_path(N, H, W, k, k, stride, pad, pad, mode, kp, "f16x3")


def enc_path(N, H, W, kh, kw, stride, padh, padw):
    """ops.conv_path of an encoder layer (the general form, which has no narrow path: kp is not read) under the f16x3
    engine, as "tc" or "simt"."""
    from objgan_b200 import ops
    path = ops.conv_path(N, H, W, kh, kw, stride, padh, padw, PAD_ZERO, 0, "f16x3", general=True)
    return "simt" if path == "simt" else "tc"


def conv_needs(work):
    """The set of rows the convolutions of a recorded workload (tests/dry.py) need: CASES-shaped tuples for
    ops.conv2d, ENC_CASES-shaped tuples for ops.enc_conv_fwd / enc_conv_dgrad."""
    return ({r + (path_of(*r[:9], r[11]),) for r in work.convs} |
            {r + (enc_path(*r[1:4], *r[6:11]),) for r in work.encs})


def uncovered(needs):
    """The needs no row of CASES / ENC_CASES covers."""
    rows = set(CASES) | set(ENC_CASES)
    return sorted((n for n in needs if n not in rows), key=str)


def stale(needs):
    """The rows of CASES / ENC_CASES no need asks for."""
    return [r for r in CASES + ENC_CASES if r not in needs]
