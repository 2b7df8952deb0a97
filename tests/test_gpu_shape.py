"""GPU tests of box-conditioned sampling: SHP_G_NET, the ConvLSTM cell, the device box maps and form_gen_hmaps against
the CPU oracle (oracle/shape_oracle.py, pinned to the reference by tests/test_shape_gen.py), the whole generated-shape
GSampler.sample against the oracle composition (shape oracle -> form_hmaps -> eval-mode G_NET), and graph replay."""
import pytest
import torch

import oracle_eval
from objgan_b200 import model, ops, synth
from objgan_b200.sampler import GSampler
from oracle import shape_oracle as S
from test_eval_mode import eval_fixture, eval_state_dict
from test_gpu_sample import _flat, _same, close, rel
from test_shape_gen import hmap_inputs, layout_inputs, shp_inputs, shp_sd

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]


def _shp(sd):
    net = model.SHP_G_NET(80)
    net.load_state_dict(sd, strict=True)
    return net.to(DEV).eval()


def _g_eval():
    want = eval_fixture(3)
    g = model.G_NET(80)
    g.load_state_dict(eval_state_dict(want), strict=True)
    return g.to(DEV).eval()


def _dev_maps(inp, rmax):
    return ops.form_bbox_maps(inp["rois0"].to(DEV), inp["fm_rois"].to(DEV), inp["roi_cls"].to(DEV),
                              inp["num_rois"].to(DEV), rmax, 80)


# ---------------------------------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rmax", [7, 10])
def test_bbox_maps_bitwise(rmax):
    inp = layout_inputs(4, 17, [7, 2, 10, 0])
    fwd, bwd, fm = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], rmax, 80)
    maps, fmaps = _dev_maps(inp, rmax)
    B = 4
    got = maps.view(2, B, rmax, 64, 64, 80).permute(0, 1, 2, 5, 3, 4).cpu()
    assert torch.equal(got[0], fwd) and torch.equal(got[1], bwd)
    assert torch.equal(fmaps.cpu(), fm)
    assert fwd.sum() > 0 and bwd[2].sum() > 0 and bwd[3].sum() == 0
    # image 1 has 2 rois: its backward sequence reaches them only when 2 + rmax > 10 (slots 8, 9 = rois 1, 0)
    assert (bwd[1].sum() == 0) == (2 + rmax <= 10)


def test_bbox_maps_hand_worked_bitwise():
    """The hand-worked table of test_shape_gen: half-to-even rounding, the exclusive clamp at 63 / 15."""
    rois0 = torch.zeros(1, 10, 6, dtype=torch.float64)
    fm = torch.zeros(1, 10, 6, dtype=torch.float64)
    rows = [((10.5, 3.5, 2.0, 2.0, 4), (5.0, 5.0, 4.0, 3.0)), ((60.0, 61.2, 10.0, 10.0, 7), (29.0, 30.0, 10.0, 10.0)),
            ((0.49, 0.5, 0.02, 1.0, 79), (0.25, 1.0, 0.5, 3.0)), ((11.5, 20.0, 1.0, 5.0, 0), (3.0, 1.0, 1.0, 0.9))]
    for r, (a, f) in enumerate(rows):
        rois0[0, r, :5] = torch.tensor(a, dtype=torch.float64)
        fm[0, r, :4] = torch.tensor(f, dtype=torch.float64)
    inp = dict(rois0=rois0, fm_rois=fm, roi_cls=rois0[..., 4].long(), num_rois=torch.tensor([4]))
    fwd, bwd, fmo = S.bbox_maps(rois0, fm, inp["num_rois"], 8, 80)
    maps, fmaps = _dev_maps(inp, 8)
    got = maps.view(2, 1, 8, 64, 64, 80).permute(0, 1, 2, 5, 3, 4).cpu()
    assert torch.equal(got[0], fwd) and torch.equal(got[1], bwd) and torch.equal(fmaps.cpu(), fmo)


@pytest.mark.parametrize("first", [True, False])
def test_clstm_cell(first):
    torch.manual_seed(5)
    B, R, H, Ch, Cj = 2, 3, 16, 160, 640
    t = 0 if first else 1
    gx = [torch.randn(B * R, H, H, 4 * Ch) * 2 for _ in range(2)]
    gh = None if first else [torch.randn(B, H, H, 4 * Ch) * 2 for _ in range(2)]
    c0 = [torch.randn(B, H, H, Ch) for _ in range(2)]
    joint = torch.full((B * R, H, H, Cj), 7.0)
    d = lambda ts: tuple(x.to(DEV) for x in ts)
    c_dev = d(c0)
    joint_dev = joint.to(DEV)
    hf, hb = ops.clstm_cell(d(gx), d(gh) if gh else None, c_dev, joint_dev, t)
    for k, h_dev in enumerate((hf, hb)):
        gates = gx[k].view(B, R, H, H, 4 * Ch)[:, t] + (gh[k] if gh else 0)
        prev = torch.zeros_like(c0[k]) if first else c0[k]
        h, c = S.lstm_gates(gates.permute(0, 3, 1, 2), prev.permute(0, 3, 1, 2))
        h, c = h.permute(0, 2, 3, 1), c.permute(0, 2, 3, 1)
        assert (h_dev.cpu() - h).abs().max() <= 1e-6 and (c_dev[k].cpu() - c).abs().max() <= 1e-6 * max(1, c.abs().max())
        slot = t if k == 0 else R - 1 - t
        jd = joint_dev.cpu().view(B, R, H, H, Cj)
        assert torch.equal(jd[:, slot, ..., k * Ch:(k + 1) * Ch], h_dev.cpu())
    jd = joint_dev.cpu().view(B, R, H, H, Cj)
    assert (jd[..., 2 * Ch:] == 7.0).all()                        # the z lanes are not touched
    untouched = [s for s in range(R) if s not in (t, R - 1 - t)]
    assert all((jd[:, s] == 7.0).all() for s in untouched)


# ---------------------------------------------------------------------------------------------------------------------
# SHP_G_NET and form_gen_hmaps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B", [1, 3])
def test_shp_g_net_forward(B, engine, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    sd = shp_sd()
    inp = shp_inputs(B)
    r = inp["rmax"]
    fwd, bwd, fm = S.bbox_maps(inp["rois0"], inp["fm_rois"], inp["num_rois"], r, 80)
    z = inp["noise_shp"][:, :r]
    with torch.no_grad():
        ref = S.shp_g_net_forward(sd, z, fwd, bwd, fm)
        net = _shp(sd)
        out = net(z.to(DEV), fwd.to(DEV), bwd.to(DEV), fm.to(DEV))          # public NCHW form
        maps, fmaps = _dev_maps(inp, r)
        out2 = ops.to_nchw(net.forward_nhwc(z.contiguous().to(DEV), maps, fmaps), 1).view(B, r, 1, 64, 64)
    close(out, ref, 1e-3, "SHP_G_NET")
    assert torch.equal(out, out2)
    print(f"B={B} {engine}: rel err {rel(out, ref):.2e}")


def _ranges(raw256, num_rois):
    return [(raw256[b, t].max() - raw256[b, t].min()).item() for b in range(raw256.shape[0])
            for t in range(int(num_rois[b]))]


def test_form_gen_hmaps():
    inp = hmap_inputs()
    raw = inp["raw"]
    up = torch.nn.functional.interpolate(raw, size=(256, 256), mode="bilinear", align_corners=True)
    rg = _ranges(up, inp["num_rois"])
    assert all(x >= 0.05 or x == 0 for x in rg), rg         # bounded amplification (constant slots are exact)
    hm, bt, fm = S.form_hmaps(raw.clone(), inp["num_rois"], inp["roi_cls"])
    with torch.no_grad():
        dh, dbt, dfm = ops.form_gen_hmaps(raw.to(DEV), inp["roi_cls"].to(DEV), inp["num_rois"].to(DEV))
    for a, b in zip(dh, hm):
        close(a, b, 1e-5, "hmaps")
    for a, b in zip(dbt, bt):
        assert a.shape[1] == 10 and a[:, 5:].abs().max() == 0
        close(a[:, :5], b, 1e-5, "bt_masks")
    close(dfm[:, :5], fm, 1e-5, "fm_bt_masks")
    assert dbt[2][0, 1].abs().max() == 0 and (dbt[2][0, 2] == 1.0).all()     # the two constant-map branches
    again = ops.form_gen_hmaps(raw.to(DEV), inp["roi_cls"].to(DEV), inp["num_rois"].to(DEV))
    assert all(torch.equal(a, b) for a, b in zip([*dh, *dbt, dfm], [*again[0], *again[1], again[2]]))


# ---------------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------------
def gen_batch(B, seed, **kw):
    """A compact batch without masks (the layout only), with its shape noise."""
    x = synth.compact(synth.make_inputs(B, seed=seed, **kw))
    for k in ("bt_masks", "fm_bt_masks"):
        x.pop(k)
    x["noise_shp"] = torch.randn(B, 10, 320, generator=torch.Generator().manual_seed(seed))
    return x


def oracle_sample(sd_g, sd_s, x):
    """shape oracle -> form_hmaps -> eval-mode G_NET oracle."""
    r = int(x["glb_max_num_roi"])
    fwd, bwd, fm = S.bbox_maps(x["rois"][0], x["fm_rois"], x["num_rois"], r, 80)
    raw = S.shp_g_net_forward(sd_s, x["noise_shp"][:, :r], fwd, bwd, fm)
    hm, bt, fmb = S.form_hmaps(raw[:, :, 0], x["num_rois"], x["roi_cls"])
    inp = synth.make_inputs(x["z"].shape[0], seed=x["_seed"], parity=True)
    inp.update(hmaps=hm, bt_masks=bt, fm_bt_masks=fmb, z=x["z"], eps=x["eps"])
    return oracle_eval.g_net_forward_eval(sd_g, inp), raw


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_generated_vs_oracle(engine, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    g = _g_eval()
    sd_g = {k: v.detach().cpu().clone() for k, v in g.state_dict().items()}
    sd_s = shp_sd()
    s = GSampler(g, _shp(sd_s))
    x = gen_batch(3, 33, parity=True)
    x["_seed"] = 33
    with torch.no_grad():
        ref, raw = oracle_sample(sd_g, sd_s, x)
    up = torch.nn.functional.interpolate(raw[:, :, 0], size=(256, 256), mode="bilinear", align_corners=True)
    print("roi mask ranges at 256^2:", [round(v, 3) for v in _ranges(up, x["num_rois"])])
    shapes = s.sample_shapes(x)
    close(shapes["raw_masks"], raw[:, :, 0], 1e-3, "raw masks")
    got = s.sample(x)
    for i, (a, b) in enumerate(zip(_flat(got), _flat(ref))):
        close(a, b, 1e-3, f"output {i}")


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_graph_replay_mixed(engine, monkeypatch):
    """Generated-shape and ground-truth-mask batches of several shapes, interleaved: every replay equals the eager pass
    bit for bit, and the two kinds of batch never share a graph."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    s = GSampler(_g_eval(), _shp(shp_sd()))
    ga, ga2, gb = gen_batch(2, 61, parity=True), gen_batch(2, 62, parity=True), gen_batch(3, 63, parity=True)
    assert ga["glb_max_num_roi"] == ga2["glb_max_num_roi"]
    gt = synth.make_inputs(2, seed=61, parity=True)                 # same key apart from the flag
    first = [s.sample(b) for b in (ga, gt, gb)]                    # eager warm-up + capture of three keys
    assert len(s._graphs) == 3
    for _ in range(2):
        for b, f in zip((ga, gt, gb), first):
            assert _same(s.sample(b), f, 1e-6, what="replay") is True
        assert _same(s.sample(ga2), s.sample_eager(ga2), 1e-6, what="replay, other inputs") is True
    assert len(s._graphs) == 3
    assert not torch.equal(s.sample(ga)[0][0], s.sample(ga2)[0][0])
    drawn = [s.sample({k: v for k, v in ga.items() if k not in ("noise_shp", "z", "eps")}) for _ in range(2)]
    assert not torch.equal(drawn[0][0][0], drawn[1][0][0])          # fresh noise every call when the batch has none


def test_sampler_from_snapshot_shape(tmp_path):
    g = _g_eval()
    sd_s = shp_sd()
    torch.save({k: v.cpu() for k, v in g.state_dict().items()}, tmp_path / "netG.pth")
    torch.save({"module." + k: v for k, v in sd_s.items()}, tmp_path / "shape_gen.pth")
    s = GSampler.from_snapshot(str(tmp_path / "netG.pth"), device=DEV, shape_snapshot=str(tmp_path / "shape_gen.pth"))
    want = GSampler(g, _shp(sd_s))
    x = gen_batch(2, 71, parity=True)
    _same(s.sample(x), want.sample(x), 1e-6, what="from_snapshot")
    _same(s.sample(x), want.sample_eager(x), 1e-6, what="from_snapshot, replayed")
    with pytest.raises(ValueError, match="no shape generator"):
        GSampler(g).sample(x)


def test_sampler_generated_full_size():
    s = GSampler(_g_eval(), _shp(shp_sd()))
    x = gen_batch(16, 91)                                            # B = 16, 10 rois each
    assert x["glb_max_num_roi"] == 10
    s.sample(x)
    got = s.sample(x)
    assert all(torch.isfinite(t).all() for t in _flat(got))
    _same(got, s.sample_eager(x), 1e-6, what="B=16 generated")
    sh = s.sample_shapes(x)
    assert sh["raw_masks"].shape == (16, 10, 64, 64) and torch.isfinite(sh["raw_masks"]).all()
