"""The library's CNN_ENCODER inside training and evaluation on the GPU: losses.G_loss and one StepBTrainer.step with the
DAMSM terms against the oracle with the oracle's encoder (oracle/image_encoder_oracle.py), on both engines;
RPrecision at the evaluator's pool of 100 (words_pairs over 10,000 pairs) against the reference's recorded accuracies;
GSampler.encode_image + RPrecision over 100 generated samples against the oracle.  (File name sorts last: the step
tests build every network of the complete step.)"""
import os
import random
import sys

import numpy as np
import pytest
import torch

from objgan_b200 import losses, model, ops, synth, trainer
from objgan_b200.sampler import GSampler, _new_g
from oracle import image_encoder_oracle as E
from oracle import objgan_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))


def _encoder():
    net = model.CNN_ENCODER(256)
    sd = E.test_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd)
    return net.to(DEV), sd


def _rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _cpu_sd(m):
    return {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("engine", ["simt", "f16x3"])
def test_g_loss_with_library_encoder(engine, monkeypatch):
    """losses.G_loss with model.CNN_ENCODER equals oracle.g_loss with the oracle's encoder: the total, the DAMSM terms
    (x DAMSM_LAMBDA = 100) and the gradient reaching the 256x256 fake image, where the encoder's input gradient adds
    to the discriminators'."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    nets, inp, fakes, raw_bt, rois0, fm, class_ids = make_golden.g_loss_case()
    sds = dict(pat=[_cpu_sd(n) for n in nets["pat"]], shp=[_cpu_sd(n) for n in nets["shp"]], ss=_cpu_sd(nets["ss"]),
               ls=_cpu_sd(nets["ls"]))
    for n in nets["pat"] + nets["shp"] + [nets["ss"], nets["ls"]]:
        n.to(DEV)
    enc, esd = _encoder()
    fo = [f.clone().requires_grad_(True) for f in fakes]
    want, wterms = O.g_loss(sds["pat"], sds["shp"], sds["ss"], sds["ls"], lambda x: E.cnn_encoder_forward(esd, x), fo,
                            inp["hmaps"], inp["words_embs"], inp["sent_emb"], inp["clabels_emb"], raw_bt,
                            torch.arange(2), [int(v) for v in inp["cap_lens"]], class_ids, rois0, fm,
                            [int(v) for v in inp["num_rois"]])
    want.backward()
    fk = [f.to(DEV).requires_grad_(True) for f in fakes]
    total, logs = losses.G_loss(nets["pat"], nets["shp"], nets["ss"], nets["ls"], enc, fk,
                                [h.to(DEV) for h in inp["hmaps"]], inp["words_embs"].to(DEV), inp["sent_emb"].to(DEV),
                                inp["clabels_emb"].to(DEV), raw_bt.to(DEV), torch.arange(2, device=DEV),
                                inp["cap_lens"], class_ids, rois0, fm, inp["num_rois"])
    for k in ("w_loss", "s_loss"):
        v = float(wterms[k])
        assert abs(float(logs[k]) - v) <= 1e-3 * max(1.0, abs(v)), (k, float(logs[k]), v)
    assert abs(float(total) - float(want)) <= 1e-3 * max(1.0, abs(float(want))), (float(total), float(want))
    total.backward()
    err = _rel_l2(fk[2].grad.cpu(), fo[2].grad)
    print(f"{engine}: fake256 gradient relative L2 {err:.3e}")
    assert err <= 1e-2, err


def _check_weights(net, sd_oracle, what=""):
    """As tests/test_gpu_zz_step_b.py: the first Adam step is sign descent, so compare the fraction of entries that
    agree to 0.1 * lr and the worst deviation."""
    lr = 2e-4
    for k, p in net.named_parameters():
        a, b = p.detach().cpu(), sd_oracle[k]
        d = (a - b).abs()
        assert torch.isfinite(a).all(), (what, k)
        assert d.max().item() <= 2 * lr + 5e-5, (what, k, d.max().item())
        if k.endswith(("shp_code.1.bias", "conv3x3.1.bias")):
            continue        # bias ahead of InstanceNorm: exact gradient is zero, the step direction is noise
        assert (d <= 0.1 * lr).float().mean().item() >= 0.97, (what, k)


@pytest.mark.parametrize("engine", ["simt", "f16x3"])
def test_step_b_with_damsm(engine, monkeypatch):
    """One StepBTrainer.step with image_encoder = model.CNN_ENCODER against oracle.step_b(image_encoder = the oracle's
    encoder): every loss including w_loss / s_loss, and the generator's weights and EMA after its Adam step."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    enc, esd = _encoder()
    t = trainer.StepBTrainer(device=DEV, seed=3, image_encoder=enc)
    st = O.StepBState(_cpu_sd(t.netG), [_cpu_sd(d) for d in t.netsPatD], [_cpu_sd(d) for d in t.netsShpD],
                      _cpu_sd(t.netObjSSD), _cpu_sd(t.netObjLSD))
    inp = synth.make_inputs(3, seed=4, parity=True)
    random.seed(5)
    want = O.step_b(st, inp, image_encoder=lambda x: E.cnn_encoder_forward(esd, x))
    random.seed(5)
    got = t.step(t.to_device(inp))
    ltol = 2e-3 if engine == "simt" else 5e-3
    for k in ("errG", "kl"):
        assert abs(float(got[k]) - want[k]) <= ltol * max(1.0, abs(want[k])), (k, float(got[k]), want[k])
    assert {"w_loss", "s_loss"} <= set(want["terms"])
    for k, v in want["terms"].items():
        assert abs(float(got["logs"][k]) - v) <= ltol * max(1.0, abs(v)), (k, float(got["logs"][k]), v)
    _check_weights(t.netG, st.g, what="G")
    ema = t.bG.ema_state_dict()
    for k in st.g_keys:
        assert (ema[k].cpu() - st.g_avg[k]).abs().max().item() <= 1e-3 * (2 * 2e-4 + 5e-5) + 1e-7, k


def test_rprecision_pool100_matches_reference():
    """Seven batches of 16 fill the pool of 100 (cut from 112), the eighth scores it: words_pairs runs 100 x 100 pairs
    in one launch; the accuracies equal the reference's words_loss / sent_loss on the same pool."""
    sys.path.insert(0, HERE)
    from test_image_encoder import pool_case, rprecision_fixture
    ref = rprecision_fixture()
    region, code, words, sent, lens, cls = pool_case()
    extra = pool_case(seed=7, n=28)             # the 12 samples past the pool, and the dropped eighth batch
    cat = [torch.cat([a, b], 0) if torch.is_tensor(a) else np.concatenate([a, b]) for a, b in
           zip((region, code, words, sent, lens, cls), extra)]
    rp = losses.RPrecision(100)
    for i in range(8):
        sl = slice(16 * i, 16 * i + 16)
        rp.add(cat[0][sl].to(DEV), cat[1][sl].to(DEV), cat[2][sl].to(DEV), cat[3][sl].to(DEV), cat[4][sl],
               cat[5][sl])
    assert len(rp.w_accuracy) == 1
    aw, sw, as_, ss = rp.result()
    assert aw == float(ref["w_accuracy"]) and as_ == float(ref["s_accuracy"]), (aw, as_, ref)
    assert sw == 0.0 and ss == 0.0


def test_sampler_encode_image_rprecision():
    """GSampler.encode_image + RPrecision over 100 generated samples (eight batches of 16; the eighth scores the pool)
    against the oracle's encoder (float64) and losses on the same images.  An argmax decided by less than the fp32
    rounding of the features may go either way, so one of the 200 decisions of each accuracy may differ."""
    enc, esd = _encoder()
    sd64 = {k: (v.double() if v.is_floating_point() else v).to(DEV) for k, v in esd.items()}
    s = GSampler(_new_g(80, DEV), image_encoder=enc)
    rp = losses.RPrecision(100)
    pool = {k: [] for k in ("region", "code", "words", "sent", "lens")}
    for i in range(8):
        batch = synth.make_inputs(16, seed=300 + i, parity=True)
        fake_imgs = s.sample(batch)[0]
        region, code = s.encode_image(fake_imgs)
        dev_words, dev_sent = batch["words_embs"].to(DEV), batch["sent_emb"].to(DEV)
        rp.add(region, code, dev_words, dev_sent, batch["cap_lens"])
        if i < 7:
            with torch.no_grad():
                rf, rc = E.cnn_encoder_forward(sd64, fake_imgs[-1].double())
            for k, v in (("region", rf), ("code", rc), ("words", batch["words_embs"]), ("sent", batch["sent_emb"]),
                         ("lens", batch["cap_lens"])):
                pool[k].append(v.float().cpu() if v.is_floating_point() else v.cpu())
    p = {k: torch.cat(v, 0)[:100] for k, v in pool.items()}
    labels = torch.arange(100)
    w = O.words_loss(p["region"], p["words"], labels, p["lens"].tolist(), None, 100)[3]
    sacc = O.sent_loss(p["code"], p["sent"], labels, None, 100)[2]
    aw, _, as_, _ = rp.result()
    assert len(rp.w_accuracy) == 1
    assert abs(aw - float(w)) <= 0.5 and abs(as_ - float(sacc)) <= 0.5, (aw, float(w), as_, float(sacc))
