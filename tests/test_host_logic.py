"""CPU tests of the host-side logic in a dry run (tests/dry.py: the host code takes the GPU's dispatch on CPU tensors,
every library call is checked against the header and counted instead of launched, outputs are uninitialised).  Checks
shapes, autograd wiring, flat-bucket plumbing and state_dict compatibility."""
import torch

import refimport
from dry import dry  # noqa: F401
from objgan_b200 import lib, model, synth, trainer
from objgan_b200.config import cfg


def test_step_a_wiring(dry):
    t = trainer.StepATrainer(device="cpu", seed=0)
    inp = synth.make_inputs(2, parity=True)
    n0 = lib.get().launches
    out = t.step(inp)
    assert lib.get().launches - n0 > 300
    assert [tuple(f.shape) for f in out["fake_imgs"]] == [(2, 3, 64, 64), (2, 3, 128, 128), (2, 3, 256, 256)]
    assert t.bG.step == 1 and all(b.step == 1 for b in t.bD)
    # every parameter is a view of its bucket and received a gradient view
    for b in [t.bG, *t.bD]:
        for p, o in zip(b.params, b.offsets):
            assert p.data.data_ptr() == b.flat[o:].data_ptr()
            assert p.grad.data_ptr() == b.grad[o:].data_ptr()


def test_module_signatures(dry):
    g = model.G_NET(80)
    inp = synth.make_inputs(2, parity=True)
    fake, btc, att, btatt, mu, logvar = g(inp["z"], inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"],
                                          inp["slabels_feat"], inp["mask"], inp["hmaps"], inp["rois"], inp["fm_rois"],
                                          inp["num_rois"], inp["bt_masks"], inp["fm_bt_masks"], inp["glb_max_num_roi"])
    assert mu.shape == (2, 100) and logvar.shape == (2, 100)
    assert [tuple(a.shape) for a in att] == [(2, 18, 64, 64), (2, 18, 128, 128)]
    assert [tuple(a.shape) for a in btatt] == [(2, 18, 64, 64), (2, 18, 128, 128)]
    assert [tuple(a.shape) for a in btc] == [(2, inp["glb_max_num_roi"], 48)] * 2
    d = model.PAT_D_NET128()
    f = d(fake[1])
    assert f.size(0) == 2 and tuple(f.size()) == (2, 768, 8, 8)
    assert tuple(d.COND_DNET(f, inp["sent_emb"]).shape) == (2, 1, 3, 3)
    assert tuple(d.UNCOND_DNET(f[:1]).shape) == (1, 1, 3, 3)
    # standalone drop-in modules on NCHW tensors
    a = model.ATT_NET(48, 256)
    a.applyMask(inp["mask"])
    wc, am = a(torch.randn(2, 48, 16, 16), inp["words_embs"])
    assert tuple(wc.shape) == (2, 48, 16, 16) and tuple(am.shape) == (2, 18, 16, 16)
    out = model.pprocess_bt_attns(torch.randn(2, 48, 5, 1), 16, 16, torch.rand(2, 5, 16, 16))
    assert tuple(out.shape) == (2, 48, 16, 16)
    r = model.RoIAlignAvg(5, 5, 1.0 / 16)(torch.randn(2, 16, 32, 32), torch.zeros(20, 5))
    assert tuple(r.shape) == (20, 16, 5, 5)


NETS = [("G_NET", (80,)), ("PAT_D_NET64", ()), ("PAT_D_NET128", ()), ("PAT_D_NET256", ()), ("SHP_D_NET64", (80,)),
        ("SHP_D_NET128", (80,)), ("SHP_D_NET256", (80,)), ("OBJ_SS_D_NET", (80,)), ("OBJ_LS_D_NET", (80,))]


def _layout(state_dict):
    """sha256 of a state_dict's layout: every (key, shape, dtype) in order."""
    import hashlib
    import json
    return hashlib.sha256(json.dumps([[k, list(v.shape), str(v.dtype)] for k, v in state_dict.items()]).encode()).hexdigest()


def _names(module):
    import hashlib
    return hashlib.sha256(" ".join(n for n, _ in module.named_parameters()).encode()).hexdigest()


def _reference_layouts():
    """{net: {"state": _layout, "params": _names}} of the reference's nine networks, stored in
    tests/golden/reference/state_dict_layouts.json (recorded from the reference's own modules, see
    tests/reference_fixtures.py)."""
    import json
    import os
    import reference_fixtures as fixtures
    path = os.path.join(fixtures.GOLD, "state_dict_layouts.json")
    if fixtures.RECORD:
        ref = refimport.load()
        out = {}
        for name, args in NETS:
            r = getattr(ref.model, name)(*args)
            out[name] = {"state": _layout(r.state_dict()), "params": _names(r)}
        os.makedirs(fixtures.GOLD, exist_ok=True)
        json.dump(out, open(path, "w"), indent=0)
    return json.load(open(path))


def test_state_dict_keys_match_reference():
    """Every network's state_dict (order, shapes, dtypes) and parameter list equal the reference's."""
    ref = _reference_layouts()
    for name, args in NETS:
        m = getattr(model, name)(*args)
        assert _layout(m.state_dict()) == ref[name]["state"], name
        assert _names(m) == ref[name]["params"], name


def test_state_dict_keys_golden():
    """Same check against the key list committed under tests/golden (works without the reference)."""
    import json
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "state_dict_keys.json")
    gold = json.load(open(path))
    for name, cls in (("G_NET", lambda: model.G_NET(80)), ("PAT_D_NET64", model.PAT_D_NET64)):
        sd = cls().state_dict()
        assert [[k, list(v.shape)] for k, v in sd.items()] == gold[name]


def test_obj_and_damsm_loss_wiring(dry):
    """objD_loss / shpD_loss / words_loss / sent_loss run end to end through autograd with every library call checked
    against the header's argument count (DRY_RUN: no arithmetic, values are meaningless)."""
    import random
    import numpy as np
    from objgan_b200 import losses
    inp = synth.make_inputs(3, seed=8, parity=True)
    real, seg, fm, nr = inp["imgs"][2], inp["hmaps"][2], inp["fm_rois"].clone(), inp["num_rois"]
    fm[..., 2:4] *= torch.tensor([1.0, 3.0, 0.2]).view(3, 1, 1)
    fake = torch.tanh(torch.randn_like(real))
    net = model.OBJ_SS_D_NET(80)
    random.seed(3)
    err = losses.objD_loss(net, real, fake, seg, inp["clabels_emb"], torch.randn(3, 10, cfg.GAN.GF_DIM), fm, nr)
    assert torch.is_tensor(err) and err.dim() == 0
    err.backward()
    assert net.roi_code[0].weight.grad is not None
    B, nef = 4, 256
    img = torch.randn(B, nef, 17, 17, requires_grad=True)
    labels = torch.arange(B)
    w0, w1, maps, acc = losses.words_loss(img, torch.randn(B, nef, 18), labels, torch.tensor([18, 7, 12, 3]),
                                          np.array([1, 2, 1, 5]), B)
    (w0 + w1).backward()
    assert img.grad.shape == img.shape and len(maps) == B and tuple(maps[1].shape) == (1, 7, 17, 17)
    cnn = torch.randn(B, nef, requires_grad=True)
    s0, s1, sacc = losses.sent_loss(cnn, torch.randn(B, nef), labels, None, B)
    (s0 + s1).backward()
    assert cnn.grad.shape == cnn.shape


def test_g_loss_wiring(dry):
    """The full G_loss runs through every discriminator family and the DAMSM terms and back-propagates to the fake images
    and the generator's bt_c_code (DRY_RUN: argument counts and autograd wiring only)."""
    import numpy as np
    from objgan_b200 import losses
    inp = synth.make_inputs(2, seed=5, parity=True)
    pat = [model.PAT_D_NET64(), model.PAT_D_NET128(), model.PAT_D_NET256()]
    shp = [model.SHP_D_NET64(80), model.SHP_D_NET128(80), model.SHP_D_NET256(80)]
    fk = [torch.tanh(torch.randn_like(im)).requires_grad_(True) for im in inp["imgs"]]
    bt = torch.randn(2, 10, cfg.GAN.GF_DIM, requires_grad=True)

    class Enc(torch.nn.Module):
        def forward(self, x):
            r = torch.nn.functional.adaptive_avg_pool2d(x, 17).repeat(1, 86, 1, 1)[:, :256]
            return r, r.mean((2, 3))

    fm = inp["fm_rois"].clone()
    fm[..., 2:4] *= torch.tensor([3.0, 0.6]).view(2, 1, 1)
    total, logs = losses.G_loss(pat, shp, model.OBJ_SS_D_NET(80), model.OBJ_LS_D_NET(80), Enc(), fk, inp["hmaps"],
                                inp["words_embs"], inp["sent_emb"], inp["clabels_emb"], bt, torch.arange(2),
                                inp["cap_lens"], np.array([4, 9]), inp["rois"][0], fm, inp["num_rois"])
    assert "pat_g_loss2" in logs and "shp_g_loss0" in logs and "w_loss" in logs
    total.backward()
    assert all(f.grad is not None and f.grad.shape == f.shape for f in fk)
    assert ("objss_g_loss" not in logs and "objls_g_loss" not in logs) or bt.grad is not None


def test_step_b_wiring(dry):
    """The complete step (all nine optimisers) on the CPU in DRY_RUN: every bucket steps once, every parameter of every
    network is a view of its bucket with a gradient view, and the library call arities hold on every path."""
    t = trainer.StepBTrainer(device="cpu", seed=0)
    inp = synth.make_inputs(2, parity=True)
    import random
    random.seed(1)
    out = t.step(inp)
    assert out["errG"].dim() == 0 and "pat_g_loss0" in out["logs"] and "shp_g_loss2" in out["logs"]
    assert t.bG.step == 1 and all(b.step == 1 for b in [*t.bD, *t.bShp])
    assert all(b.step in (0, 1) for b in t.bObj)       # an object discriminator only steps when it saw rois of its scale
    for b in [t.bG, *t._d_buckets()]:
        for p, o in zip(b.params, b.offsets):
            assert p.data.data_ptr() == b.flat[o:].data_ptr() and p.grad.data_ptr() == b.grad[o:].data_ptr()


def test_checkpoint_files_round_trip(dry, tmp_path):
    """f4: the reference's snapshot file set (ref: trainer.py:251-273) written by StepBTrainer.save_model loads back
    (strict) into a fresh trainer with identical tensors, and matches the layout the reference's own modules load with
    load_state_dict(strict=True), which is what its build_models does (152-194)."""
    t = trainer.StepBTrainer(device="cpu", seed=0)
    with torch.no_grad():
        for b in [t.bG, *t._d_buckets()]:
            b.flat.copy_(torch.randn(b.flat.shape))
        t.bG.avg.copy_(t.bG.flat * 0.5)
    files = t.save_model(str(tmp_path), 7)
    assert files == sorted(["netG_epoch_7.pth", "netPatD0.pth", "netPatD1.pth", "netPatD2.pth", "netShpD0.pth",
                            "netShpD1.pth", "netShpD2.pth", "netObjSSD.pth", "netObjLSD.pth"])
    u = trainer.StepBTrainer(device="cpu", seed=1)
    assert u.load_model(str(tmp_path / "netG_epoch_7.pth")) == 8
    for (ka, a), (kb, b) in zip(u.netG.state_dict().items(), t.bG.ema_state_dict().items()):
        assert ka == kb and torch.equal(a, b), ka                         # the generator file holds the EMA weights
    assert torch.equal(u.bG.avg, u.bG.flat)
    for na, nb in zip([*u.netsPatD, *u.netsShpD, u.netObjSSD, u.netObjLSD],
                      [*t.netsPatD, *t.netsShpD, t.netObjSSD, t.netObjLSD]):
        for (ka, a), (kb, b) in zip(na.state_dict().items(), nb.state_dict().items()):
            assert ka == kb and torch.equal(a, b), ka
    for b in [u.bG, *u._d_buckets()]:                                      # parameters are bucket views again
        for p, o in zip(b.params, b.offsets):
            assert p.data.data_ptr() == b.flat[o:].data_ptr()
    # the reference's build_models loads these files with load_state_dict(strict=True) (trainer.py:155-191): same
    # keys, shapes and dtypes as its modules
    ref = _reference_layouts()
    for name, net in [("netG_epoch_7.pth", "G_NET"), ("netPatD0.pth", "PAT_D_NET64"), ("netPatD1.pth", "PAT_D_NET128"),
                      ("netPatD2.pth", "PAT_D_NET256"), ("netShpD0.pth", "SHP_D_NET64"), ("netShpD1.pth", "SHP_D_NET128"),
                      ("netShpD2.pth", "SHP_D_NET256"), ("netObjSSD.pth", "OBJ_SS_D_NET"), ("netObjLSD.pth", "OBJ_LS_D_NET")]:
        sd = torch.load(str(tmp_path / name), map_location=lambda storage, loc: storage)
        assert _layout(sd) == ref[net]["state"], name


def test_res_chain_tells_each_block_its_consumer(dry):
    """Producer-side operand split (og_norm_apply_split): every residual block of the generator knows which operand layout
    the convolution after it wants -- the next block's reflection-padded conv (halo 1) or the upsample conv that ends
    the chain (plain copies, halo 0) -- and the C ABI declares the two launchers the fused pass needs."""
    from objgan_b200 import lib as L
    g = model.G_NET(80)
    for main in (g.h_net1_main, g.h_net2_main, g.h_net3_main):
        pads = [b.next_pad for b in main.residual]
        assert pads == [1] * (len(pads) - 1) + [0], pads
    protos = L.get().protos
    assert "og_norm_bound" in protos and "og_norm_apply_split" in protos
    assert len(protos["og_norm_apply_split"]) == 19          # 18 arguments + the stream
