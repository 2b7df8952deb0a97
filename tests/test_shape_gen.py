"""Shape generator for box-conditioned sampling (CPU): the oracle's SHP_G_NET forward and form_hmaps
(oracle/shape_oracle.py) against the reference's own code, the box-map builder against hand-worked cases, the state_dict
layout, and the library calls the shape path issues (DRY_RUN: host logic only).

The reference side is stored in tests/golden/reference/shp_g_net_forward_B{1,3}.npz, form_hmaps_gen.npz and
shp_g_net_layout.json.  Re-record with the reference importable (tests/refimport.py):

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_shape_gen.py
"""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import reference_fixtures as fixtures
import refimport
from objgan_b200 import lib, model, ops, synth
from objgan_b200.sampler import GSampler, strip_module_prefix
from oracle import shape_oracle as S

OUT_CAP = 4096          # stored elements per SHP_G_NET output
HM_CAP = 8192           # stored elements per form_hmaps output
SHP_CASES = {1: [6], 3: [7, 2, 5]}   # num_rois per image; 2 rois at Rmax = 7: 2 + 7 <= 10, an all-empty backward sequence


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fixtures
# ---------------------------------------------------------------------------------------------------------------------
_sd = {}


def shp_sd():
    """state_dict of objgan_b200's SHP_G_NET(80) after weights_init under torch.manual_seed(0)."""
    if "sd" not in _sd:
        torch.manual_seed(0)
        net = model.SHP_G_NET(80)
        net.apply(model.weights_init)
        _sd["sd"] = {k: v.clone() for k, v in net.state_dict().items()}
    return {k: v.clone() for k, v in _sd["sd"].items()}


def layout_inputs(B, seed, num_rois):
    """A seeded layout: rois0 / fm_rois (B, 10, 6) float64 [x, y, w, h, cls, 0] at 64 / 32 pixels (every third box on
    half-integer coordinates), roi_cls (B, 10) int64, num_rois (B,), noise_shp (B, 10, 320)."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(B, 10, 2, generator=g).double() * 48.0
    wh = 4.0 + torch.rand(B, 10, 2, generator=g).double() * 24.0
    half = (torch.arange(10) % 3 == 0).view(1, 10, 1)
    xy = torch.where(half, torch.floor(xy) + 0.5, xy)
    wh = torch.where(half, torch.floor(wh), wh)
    cls = torch.randint(0, 80, (B, 10), generator=g)
    nr = torch.tensor(num_rois, dtype=torch.int64)
    valid = (torch.arange(10).view(1, 10) < nr.view(B, 1)).unsqueeze(-1)
    rois0 = torch.cat([xy, wh, cls.double().unsqueeze(-1), torch.zeros(B, 10, 1, dtype=torch.float64)], 2) * valid
    fm = rois0.clone()
    fm[..., :4] /= 2.0
    noise = torch.randn(B, 10, 320, generator=g)
    return dict(rois0=rois0, fm_rois=fm, roi_cls=rois0[..., 4].to(torch.int64), num_rois=nr, noise_shp=noise,
                rmax=int(nr.max()))


def shp_inputs(B):
    return layout_inputs(B, 500 + B, SHP_CASES[B])


def shp_fixture(B):
    def produce():
        ref = refimport.load()
        inp = shp_inputs(B)
        fwd, bwd, fmaps = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], inp["rmax"], 80)
        net = ref.model.SHP_G_NET(80)
        net.load_state_dict(shp_sd(), strict=True)
        net.eval()
        cuda = torch.Tensor.cuda
        torch.Tensor.cuda = lambda self, *a, **k: self         # CLSTMCell moves its zero state with .cuda()
        try:
            with torch.no_grad():
                out = net(inp["noise_shp"][:, :inp["rmax"]], fwd, bwd, fmaps)
        finally:
            torch.Tensor.cuda = cuda
        return {"in__rois0": inp["rois0"], "in__fm_rois": inp["fm_rois"], "in__num_rois": inp["num_rois"],
                "in__noise_shp": inp["noise_shp"], "out": out, "out_absmax": out.abs().max()}
    return fixtures.recorded(f"shp_g_net_forward_B{B}", produce, cap=OUT_CAP)


HM_NUM_ROIS = [4, 2]


def hmap_inputs():
    """Raw masks (2, 5, 64, 64) for form_hmaps: image 0 has a constant slot below 0.6 (slot 1, class 7), a constant slot
    above it (slot 2, class 9), class 5 twice (slots 0 and 3) and an unused slot 4; image 1 has class 3 twice and three
    unused slots.  Every other slot spans >= 0.5 over its map.  The constants are 0.25 and 1.0, which the bilinear
    resize reproduces exactly (any other value picks up rounding noise there, and the normalisation stretches that
    noise to [0, 1] -- in the reference too)."""
    g = torch.Generator().manual_seed(77)
    raw = 0.05 + 0.9 * torch.rand(2, 5, 64, 64, generator=g)
    raw[0, 1] = 0.25
    raw[0, 2] = 1.0
    cls = torch.tensor([[5, 7, 9, 5, 11, 0, 0, 0, 0, 0], [3, 3, 12, 13, 14, 0, 0, 0, 0, 0]], dtype=torch.int64)
    rois0 = torch.zeros(2, 10, 6, dtype=torch.float64)
    rois0[..., 4] = cls.double()
    return dict(raw=raw, roi_cls=cls, rois0=rois0, num_rois=torch.tensor(HM_NUM_ROIS, dtype=torch.int64))


def _hm_outputs(hm, bt, fm):
    out = {f"hmaps{i}": h for i, h in enumerate(hm)}
    out.update({f"bt_masks{i}": m for i, m in enumerate(bt)})
    out["fm_bt_masks"] = fm
    out["x_const_lo"] = bt[0][0, 1]             # constant 0.25: set to 0
    out["x_const_hi"] = bt[0][0, 2]             # constant 1.0: left as it is
    out["x_hm_const"] = hm[0][0, [7, 9]]        # their class channels
    out["x_pad0"] = bt[0][0, 4]                 # unused slots: raw
    out["x_pad1"] = bt[0][1, 2:4]
    out["x_fm_pad1"] = fm[1, 2:5]
    return out


def hmap_fixture():
    def produce():
        ref = refimport.load()
        inp = hmap_inputs()
        with torch.no_grad():
            hm, bt, fm = ref.utils.form_hmaps(inp["raw"].clone(), inp["num_rois"], inp["rois0"], (64, 128, 256), 80)
        return _hm_outputs(hm, bt, fm)
    return fixtures.recorded("form_hmaps_gen", produce, cap=HM_CAP)


def _layout(state_dict):
    return hashlib.sha256(json.dumps([[k, list(v.shape), str(v.dtype)] for k, v in state_dict.items()]).encode()).hexdigest()


def shp_layout():
    """{"state": sha256 of (key, shape, dtype) in order, "keys": [[key, shape]]} of the reference's SHP_G_NET(80)."""
    path = os.path.join(fixtures.GOLD, "shp_g_net_layout.json")
    if fixtures.RECORD:
        sd = refimport.load().model.SHP_G_NET(80).state_dict()
        json.dump({"state": _layout(sd), "keys": [[k, list(v.shape)] for k, v in sd.items()]}, open(path, "w"), indent=0)
    return json.load(open(path))


def _close(a, b, tol, cap):
    """a (full tensor) against the stored sample b, within tol of max|b|."""
    a = torch.from_numpy(fixtures.sample(a, cap)).reshape(-1)
    b = torch.as_tensor(b).float().reshape(-1)
    assert a.numel() == b.numel() and torch.isfinite(a).all()
    err = (a - b).abs().max().item()
    assert err <= tol * max(b.abs().max().item(), 1e-12), err


# ---------------------------------------------------------------------------------------------------------------------
# oracle vs reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
def test_shp_g_net_oracle_matches_reference(B):
    want = shp_fixture(B)
    inp = shp_inputs(B)
    for k in ("rois0", "fm_rois", "noise_shp"):      # the seeded inputs are the recorded ones
        assert torch.equal(inp[k].float(), want["in__" + k]), k
    fwd, bwd, fmaps = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], inp["rmax"], 80)
    with torch.no_grad():
        out = S.shp_g_net_forward(shp_sd(), inp["noise_shp"][:, :inp["rmax"]], fwd, bwd, fmaps)
    assert out.shape == (B, inp["rmax"], 1, 64, 64)
    _close(out, want["out"], 1e-5, OUT_CAP)
    assert abs(out.abs().max().item() - float(want["out_absmax"])) <= 1e-5


def test_backward_sequence_reversal():
    """bwd[b, t] = fwd slot 9 - t: the image with 2 rois at Rmax = 7 sees only empty maps backwards; the others see
    their last rois in reverse order."""
    inp = shp_inputs(3)
    fwd, bwd, _ = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], 10, 80)
    f7, b7, fm7 = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], 7, 80)
    for b in range(3):
        for t in range(10):
            assert torch.equal(bwd[b, t], fwd[b, 9 - t])
        assert torch.equal(b7[b], bwd[b, :7]) and torch.equal(f7[b], fwd[b, :7])
    assert b7[1].abs().sum() == 0 and f7[1, :2].abs().sum() > 0
    assert b7[0, 3:].abs().sum() > 0 and b7[0, :3].abs().sum() == 0       # 7 rois: backward slots 3..6 = rois 6..3


def test_form_hmaps_oracle_matches_reference():
    want = hmap_fixture()
    inp = hmap_inputs()
    hm, bt, fm = S.form_hmaps(inp["raw"].clone(), inp["num_rois"], inp["roi_cls"], (64, 128, 256), 80)
    got = _hm_outputs(hm, bt, fm)
    for k, v in got.items():
        if k.startswith("x_"):                      # the constant-map branches and the unused slots: exactly
            assert torch.equal(v.reshape(-1), want[k].reshape(-1)), k
        else:
            _close(v, want[k], 1e-6, HM_CAP)
    # the branches at 256^2: 0.25 -> 0, 1.0 kept (the resize to 64^2 that follows leaves 1.0 within an ulp)
    assert got["x_const_lo"].abs().max() == 0 and (got["x_const_hi"] - 1.0).abs().max() <= 1e-7
    assert got["x_hm_const"][0].abs().max() == 0 and (got["x_hm_const"][1] - 1.0).abs().max() <= 1e-7
    for k in ("x_pad0", "x_pad1", "x_fm_pad1"):     # unused slots: raw values in [0.05, 0.95], not stretched to [0, 1]
        assert got[k].min() > 0.04 and got[k].max() < 0.96, k


# ---------------------------------------------------------------------------------------------------------------------
# box maps: hand-worked cases
# ---------------------------------------------------------------------------------------------------------------------
def _box(rows, cols, size):
    m = torch.zeros(size, size)
    if rows and cols:
        m[rows[0]:rows[1], cols[0]:cols[1]] = 1
    return m


def test_bbox_maps_hand_worked():
    rows = [  # x, y, w, h (64 px), cls, fm (x, y, w, h at 32 px) -> expected [y0, y1), [x0, x1) at 64 and at 16
        ((10.5, 3.5, 2.0, 2.0), 4, (5.0, 5.0, 4.0, 3.0), ((4, 6), (10, 12)), ((2, 4), (2, 4))),    # half-to-even
        ((60.0, 61.2, 10.0, 10.0), 7, (29.0, 30.0, 10.0, 10.0), ((61, 63), (60, 63)), ((15, 15), (14, 15))),  # edge
        ((0.49, 0.5, 0.02, 1.0), 79, (0.25, 1.0, 0.5, 3.0), ((0, 2), (0, 1)), ((0, 2), (0, 0))),   # 0.5 -> 0, 1.5 -> 2
        ((11.5, 20.0, 1.0, 5.0), 0, (3.0, 1.0, 1.0, 0.9), ((20, 25), (12, 12)), ((0, 1), (2, 2))),  # 11.5 -> 12: empty
    ]
    B, boxes = 1, 10
    rois0 = torch.zeros(B, boxes, 6, dtype=torch.float64)
    fm = torch.zeros(B, boxes, 6, dtype=torch.float64)
    for r, (box, c, fbox, _, _) in enumerate(rows):
        rois0[0, r, :4] = torch.tensor(box, dtype=torch.float64)
        rois0[0, r, 4] = c
        fm[0, r, :4] = torch.tensor(fbox, dtype=torch.float64)
    rois0[0, 4, :5] = torch.tensor([5.0, 5.0, 9.0, 9.0, 3.0])      # slot 4 is past num_rois: ignored
    nr = torch.tensor([4])
    fwd, bwd, fmaps = S.bbox_maps(rois0, fm, nr, 6, 80)
    assert fwd.shape == (1, 6, 80, 64, 64) and fmaps.shape == (1, 6, 16, 16)
    for r, (_, c, _, (ys, xs), (fys, fxs)) in enumerate(rows):
        want = torch.zeros(80, 64, 64)
        want[c] = _box(ys, xs, 64)
        assert torch.equal(fwd[0, r], want), r
        assert torch.equal(fmaps[0, r], _box(fys, fxs, 16)), r
    assert fwd[0, 4:].abs().sum() == 0 and fmaps[0, 4:].abs().sum() == 0
    assert fwd[0, :, :, 63, :].abs().sum() == 0 and fwd[0, :, :, :, 63].abs().sum() == 0   # never set
    assert bwd.abs().sum() == 0                     # slots 9..4 backwards: all past num_rois
    _, bwd8, _ = S.bbox_maps(rois0, fm, torch.tensor([4]), 8, 80)
    assert torch.equal(bwd8[0, 6], fwd[0, 3]) and torch.equal(bwd8[0, 7], fwd[0, 2])


# ---------------------------------------------------------------------------------------------------------------------
# module API
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def dry():
    lib.DRY_RUN = True
    model.FAST_INIT = True
    yield
    lib.DRY_RUN = False
    model.FAST_INIT = False


def test_shp_g_net_state_dict_matches_reference(dry):
    ref = shp_layout()
    net = model.SHP_G_NET(80)
    sd = net.state_dict()
    assert _layout(sd) == ref["state"]
    assert [[k, list(v.shape)] for k, v in sd.items()] == ref["keys"]
    other = {k: torch.randn(v.shape) for k, v in sd.items()}
    net.load_state_dict(strip_module_prefix({"module." + k: v for k, v in other.items()}), strict=True)
    assert all(torch.equal(net.state_dict()[k], v) for k, v in other.items())
    net.load_state_dict(strip_module_prefix(other), strict=True)
    with pytest.raises(RuntimeError):
        net.load_state_dict(strip_module_prefix({"module." + k: v for k, v in list(other.items())[1:]}), strict=True)


def test_snapshot_loads_with_and_without_module_prefix(dry, tmp_path):
    g = model.G_NET(80)
    torch.save(g.state_dict(), tmp_path / "netG.pth")
    shp = {k: torch.randn(v.shape) for k, v in model.SHP_G_NET(80).state_dict().items()}
    torch.save({"module." + k: v for k, v in shp.items()}, tmp_path / "shape_gen.pth")
    torch.save(shp, tmp_path / "shape_gen_bare.pth")
    for name in ("shape_gen.pth", "shape_gen_bare.pth"):
        s = GSampler.from_snapshot(str(tmp_path / "netG.pth"), device="cpu", shape_snapshot=str(tmp_path / name))
        got = s.netShpG.state_dict()
        assert all(torch.equal(got[k], v) for k, v in shp.items()), name
        assert not any(p.requires_grad for p in s.netShpG.parameters())
    assert GSampler.from_snapshot(str(tmp_path / "netG.pth"), device="cpu").netShpG is None


def test_inference_only(dry):
    net = model.SHP_G_NET(80)
    args = (torch.randn(1, 2, 320), torch.zeros(1, 2, 80, 64, 64), torch.zeros(1, 2, 80, 64, 64), torch.zeros(1, 2, 16, 16))
    with pytest.raises(RuntimeError, match="inference only"):
        net(*args)
    with torch.no_grad():
        assert net(*args).shape == (1, 2, 1, 64, 64)
    with pytest.raises(RuntimeError, match="inference only"):
        ops.form_gen_hmaps(torch.rand(1, 2, 64, 64, requires_grad=True), torch.zeros(1, 10, dtype=torch.int64),
                           torch.tensor([2]))


def _trace(monkeypatch, fn):
    calls = []
    real = ops._call

    def rec(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(ops, "_call", rec)
    try:
        fn()
    finally:
        monkeypatch.setattr(ops, "_call", real)
    return calls


@pytest.mark.parametrize("R", [1, 4])
def test_shape_call_sequence(dry, monkeypatch, R):
    """The recurrence: the x-part of Gates once per direction for all steps, then per step the h-part of both
    directions (not at t = 0, where h = 0) and ONE cell launch for both; no concat pass; one crop."""
    net = model.SHP_G_NET(80)
    B = 2
    maps, fmaps = ops.form_bbox_maps(torch.zeros(B, 10, 6, dtype=torch.float64), torch.zeros(B, 10, 6, dtype=torch.float64),
                                     torch.zeros(B, 10, dtype=torch.int64), torch.tensor([R, 1]), R, 80)
    assert maps.shape == (2 * B * R, 64, 64, 80) and fmaps.shape == (B, R, 16, 16)
    z = torch.randn(B, R, 320)
    with torch.no_grad():
        net.forward_nhwc(z, maps, fmaps)                  # first pass packs the weights
        calls = _trace(monkeypatch, lambda: net.forward_nhwc(z, maps, fmaps))
    conv = "og_conv2d_simt"
    want = [conv, "og_norm_stats", "og_norm_apply", conv, "og_norm_stats", "og_norm_apply",     # downsample1, 2
            conv, conv, "og_broadcast_channels"]                                                # gates_x fwd, bwd; z
    for t in range(R):
        want += ([] if t == 0 else [conv, conv]) + ["og_clstm_cell"]
    want += [conv, "og_norm_stats", "og_norm_apply", "og_mul_pixels",                          # jointConv, crop
             conv, "og_norm_stats", "og_norm_apply", conv, "og_norm_stats", "og_norm_apply", conv, "og_add",
             conv, "og_norm_stats", "og_norm_apply", conv, "og_norm_stats", "og_norm_apply",    # upsample1, 2
             "og_conv2d_narrow_fwd" if B * R * 4096 <= 65536 else conv]
    assert calls == want


def test_sampler_generated_shape_path(dry, monkeypatch):
    g, shp = model.G_NET(80), model.SHP_G_NET(80)
    s = GSampler(g, shp)
    batch = synth.compact(synth.make_inputs(2, seed=5, parity=True))
    for k in ("bt_masks", "fm_bt_masks"):
        batch.pop(k)
    calls = _trace(monkeypatch, lambda: s.sample_eager(batch))
    count = lambda name: sum(1 for c in calls if c == name)
    rmax = batch["glb_max_num_roi"]
    assert count("og_form_bbox_maps") == 1 and count("og_gen_hmaps") == 1 and count("og_clstm_cell") == rmax
    assert count("og_form_hmaps") == 0 and count("og_form_clabels_feat") == 1
    assert calls.index("og_gen_hmaps") < calls.index("og_form_clabels_feat")
    sh = s.sample_shapes(batch)
    assert sh["raw_masks"].shape == (2, rmax, 64, 64) and sh["fm_bt_masks"].shape == (2, 10, 32, 32)
    assert [tuple(h.shape) for h in sh["hmaps"]] == [(2, 80, 64, 64), (2, 80, 128, 128), (2, 80, 256, 256)]
    assert [tuple(m.shape) for m in sh["bt_masks"]] == [(2, 10, 64, 64), (2, 10, 128, 128), (2, 10, 256, 256)]
    assert GSampler._key(s._prepare(batch))[-1] is True
    with_masks = synth.compact(synth.make_inputs(2, seed=5, parity=True))
    assert GSampler._key(s._prepare(with_masks))[-1] is False
    with pytest.raises(ValueError, match="no shape generator"):
        GSampler(g).sample_eager(batch)
