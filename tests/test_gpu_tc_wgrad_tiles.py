"""GPU test of the weight-gradient kernel's tiling (conv_tc.cu): the ci tile is fitted to the layer (200 channels run
as 2 x 104 columns, starting mid-slab), each stage is one wgmma over the tile's whole ci extent, a co slab past the
layer's rows issues nothing, and up to 104 columns two taps share one CTA and its G tile.  None of that may change
a result: an element's k-sum has the same stages, partial sums and order at any tile width or position, so the
gradients of sub-layers are compared bitwise with the corresponding block of the wide layer's."""
import pytest
import torch

from objgan_b200 import model, ops
from objgan_b200.lib import PAD_REFLECT

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (co_lo, co_cnt, ci_lo, ci_cnt) blocks of a 400 x 200 layer.  Row counts 400, 200, 96, 64, 40 cover 4 / 2 / 1 co
# tiles with and without an idle second slab; column counts 200, 104, 64, 48, 24 take ci widths 104, 104, 64, 48, 32
# at slab-aligned and unaligned starts; 112 and 128 columns take 112 and 128.  Each runs with one tap per CTA and, up
# to 104 columns, with two taps sharing a CTA and its G tile (OG_WGRAD_PAIR).
BLOCKS = [(4, 200, 0, 200), (100, 96, 8, 104), (92, 64, 96, 104), (60, 48, 100, 48), (0, 400, 72, 64),
          (100, 40, 100, 24), (64, 64, 0, 112), (36, 72, 72, 128)]


def _wgrad(w, x, gy):
    """OIHW weight gradient of a reflection-padded 3x3 Conv2dP holding w, at the NCHW input x and output gradient gy."""
    m = model.Conv2dP(w.shape[1], w.shape[0], 3, 1, 1, mode=PAD_REFLECT).to(DEV)
    with torch.no_grad():
        m.weight.copy_(w)
    y = m(ops.to_nhwc(x.to(DEV)))
    y.backward(ops.to_nhwc(gy.to(DEV)))
    torch.cuda.synchronize()
    return m.weight.grad.detach().cpu().clone()


def test_wgrad_tile_width_does_not_change_results(monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", "f16x3")
    torch.manual_seed(23)
    cin, cout, n, h = 200, 400, 1, 24
    # one image of 24 x 24 = 9 pixel chunks of 8 x 8: too few to split the pixel reduction (at least 8 chunks per
    # split), so every layer below sums its chunks in the same single pass (the split count follows the number of
    # tiles, and a different count regroups the sum)
    w = torch.randn(cout, cin, 3, 3) * 0.05
    x = torch.randn(n, cin, h, h)
    gy = torch.randn(n, cout, h, h)
    # the operand scales come from max|x| and max|g|: every block holds both maxima (channel 100 of each)
    x[0, 100, 5, 7] = 4 * x.abs().max()
    gy[0, 100, 9, 3] = 4 * gy.abs().max()
    wide = _wgrad(w, x, gy)
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1), mode="reflect").double()
    ref = torch.einsum("nohw,nchw->oc", gy.double(), xp[:, :, 1:1 + h, 1:1 + h])  # centre tap only
    assert (wide[:, :, 1, 1].double() - ref).abs().max() <= 1e-4 * ref.abs().max()
    for pair in ("0", "1"):
        monkeypatch.setenv("OG_WGRAD_PAIR", pair)
        assert torch.equal(_wgrad(w, x, gy), wide), pair
        for co_lo, co_n, ci_lo, ci_n in BLOCKS:
            narrow = _wgrad(w[co_lo:co_lo + co_n, ci_lo:ci_lo + ci_n], x[:, ci_lo:ci_lo + ci_n],
                            gy[:, co_lo:co_lo + co_n])
            assert torch.equal(narrow, wide[co_lo:co_lo + co_n, ci_lo:ci_lo + ci_n]), (pair, co_lo, co_n, ci_lo, ci_n)


def test_wgrad_pairing_does_not_change_results_with_split_pixels(monkeypatch):
    """The res-block conv1 shape at batch 4, 64 x 64: the pixel reduction is split over CTAs and the nine taps share
    CTAs in pairs (the last one alone); bitwise equal to one tap per CTA."""
    monkeypatch.setattr(ops, "CONV_ENGINE", "f16x3")
    torch.manual_seed(29)
    w = torch.randn(400, 200, 3, 3) * 0.05
    x, gy = torch.randn(4, 200, 64, 64), torch.randn(4, 400, 64, 64)
    monkeypatch.setenv("OG_WGRAD_PAIR", "0")
    single = _wgrad(w, x, gy)
    monkeypatch.setenv("OG_WGRAD_PAIR", "1")
    assert torch.equal(_wgrad(w, x, gy), single)
