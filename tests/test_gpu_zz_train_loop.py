"""The training loop (trainer.condGANTrainer) on the GPU: one step from an unsorted reference-format batch against the
oracle (the text stage, the sort and prepare_cat_emb restated on the CPU, feeding oracle.step_b with the oracle's
image encoder) on both engines; the text stage the loop runs against the same stage run beforehand; the epoch's
Inception score against INCEPTION_V3 over the returned images; and two epochs end to end with a reload of the written
snapshot set.  (File name sorts last: every test builds all the networks of the complete step.)"""
import os
import random

import numpy as np
import pytest
import torch

import inception_oracle as I
from objgan_b200 import losses, model, ops, synth, trainer
from objgan_b200.config import cfg
from oracle import image_encoder_oracle as E
from oracle import objgan_oracle as O
from oracle import text_oracle as T
from test_gpu_zz_step_b import _check_weights, _cpu_sd

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_WORDS = 150


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """text_encoder100.pth / image_encoder100.pth (the image encoder with the oracle tests' weights) and the Inception
    weights with the scoring tests' spread of logits."""
    d = tmp_path_factory.mktemp("pretrained")
    torch.manual_seed(0)
    text_sd = model.RNN_ENCODER(N_WORDS, nhidden=256).state_dict()
    torch.save(text_sd, d / "text_encoder100.pth")
    img_sd = E.test_state_dict(model.CNN_ENCODER(256).state_dict(), seed=0)
    torch.save(img_sd, d / "image_encoder100.pth")
    inc = I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0)
    return str(d / "text_encoder100.pth"), inc, text_sd, img_sd


@pytest.fixture()
def loop_cfg(monkeypatch, files):
    for k, v in dict(MAX_EPOCH=2, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=1, BATCH_SIZE=3, FLAG=True, NET_E=files[0],
                     NET_G="").items():
        monkeypatch.setitem(cfg.TRAIN, k, v)
    return files


def _loop(out_dir, files, loader, seed=3):
    t = trainer.condGANTrainer(str(out_dir), loader, synth.reference_dataset(n_words=N_WORDS),
                               inception_weights=files[1], device=DEV)
    torch.manual_seed(seed)
    t.setup()
    return t


def _oracle_inputs(data, ds, text_sd, z, eps):
    """The reference's prepare_data + text stage + prepare_cat_emb + form_clabels_feat on the CPU."""
    imgs, caps, gcaps, lens, hmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks, class_ids, _ = data
    b = lens.shape[0]
    order = torch.sort(lens, dim=0, descending=True, stable=True).indices
    lens = lens[order]
    caps, gcaps = caps[order].view(b, -1), gcaps[order].view(b, -1)
    max_len = int(lens.max())
    words, sent = T.rnn_encoder_forward(text_sd, caps, lens, max_len)
    glove = ds.glove_embed.weight.detach().float()
    glove_words, mask = T.text_inputs(caps, gcaps, glove, max_len)
    clabels = T.prepare_cat_emb(glove, ds.cat_labels, ds.cat_label_lens, ds.sorted_cat_label_indices)
    rois = [r[order] for r in rois]
    nr = num_rois[order]
    rmax = int(nr.max())
    cls = rois[0][..., 4].long()
    sl = torch.zeros(b, rmax, clabels.shape[1])
    for i in range(b):
        sl[i, :int(nr[i])] = clabels[cls[i, :int(nr[i])]]
    inp = dict(z=z.cpu(), eps=eps.cpu(), sent_emb=sent, words_embs=words, glove_words_embs=glove_words,
               clabels_emb=clabels, slabels_feat=sl.transpose(1, 2).unsqueeze(3).contiguous(), cap_lens=lens, mask=mask,
               num_rois=nr, rois=rois, fm_rois=fm_rois[order], bt_masks=[m[order].float() for m in bt_masks],
               fm_bt_masks=fm_bt_masks[order].float(), hmaps=[h[order].float() for h in hmaps],
               imgs=[x[order] for x in imgs], glb_max_num_roi=rmax)
    return inp, class_ids[order].numpy()


@pytest.mark.parametrize("engine", ["simt", "f16x3"])
def test_loop_step_vs_oracle(engine, loop_cfg, tmp_path, monkeypatch):
    """One step of the loop from an unsorted caption batch (B = 3, lengths in [5, 18]) with injected z and eps against
    oracle.step_b, with test_step_b_parity's tolerances: every loss, the fake images, the weights of the nine networks
    and the generator's EMA."""
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    data = synth.reference_batch(3, seed=31, lens=[9, 16, 5], n_words=N_WORDS)
    t = _loop(tmp_path, loop_cfg, [data])
    net = t.net
    st = O.StepBState(_cpu_sd(net.netG), [_cpu_sd(d) for d in net.netsPatD], [_cpu_sd(d) for d in net.netsShpD],
                      _cpu_sd(net.netObjSSD), _cpu_sd(net.netObjLSD))
    g = torch.Generator().manual_seed(32)
    z, eps = torch.randn(3, cfg.GAN.Z_DIM, generator=g), torch.randn(3, cfg.GAN.CONDITION_DIM, generator=g)
    inp, class_ids = _oracle_inputs(data, synth.reference_dataset(n_words=N_WORDS), loop_cfg[2], z, eps)
    esd = loop_cfg[3]
    random.seed(5)
    want = O.step_b(st, inp, image_encoder=lambda x: E.cnn_encoder_forward(esd, x), class_ids=class_ids)
    random.seed(5)
    got = t.train_step(data, z=z.to(DEV), eps=eps.to(DEV))
    assert (got["class_ids"] == class_ids).all()
    ltol = 2e-3 if engine == "simt" else 5e-3
    for k in ("errPatD0", "errPatD1", "errPatD2", "errShpD0", "errShpD1", "errShpD2", "errObjSSD", "errObjLSD",
              "errG", "kl"):
        if want[k] is None:
            assert got[k] is None, k
        else:
            assert abs(float(got[k]) - want[k]) <= ltol * max(1.0, abs(want[k])), (k, float(got[k]), want[k])
    assert {"w_loss", "s_loss"} <= set(want["terms"])
    for k, v in want["terms"].items():
        assert abs(float(got["logs"][k]) - v) <= ltol * max(1.0, abs(v)), (k, float(got["logs"][k]), v)
    for i in range(3):
        a, b = got["fake_imgs"][i].cpu(), want["fake"][i]
        assert (a - b).abs().max().item() <= 1e-3 * b.abs().max().item(), i
    for i, d in enumerate(net.netsPatD):
        _check_weights(d, st.ds[i], what=f"PatD{i}")
    for i, d in enumerate(net.netsShpD):
        _check_weights(d, st.extra[i], what=f"ShpD{i}")
    for j, (d, k) in enumerate(((net.netObjSSD, "errObjSSD"), (net.netObjLSD, "errObjLSD"))):
        _check_weights(d, st.extra[3 + j], what=k)
        assert net.bObj[j].step == st.x_step[3 + j]
    _check_weights(net.netG, st.g, what="G")
    ema = net.bG.ema_state_dict()
    for k in st.g_keys:
        assert (ema[k].cpu() - st.g_avg[k]).abs().max().item() <= 1e-3 * (2 * 2e-4 + 5e-5) + 1e-7, k


def test_loop_text_stage_bitwise(loop_cfg, tmp_path, monkeypatch):
    """The inputs the loop hands to StepBTrainer.step are bitwise the text stage run beforehand on the same batch, and
    the step's forward results (fake images, first discriminator loss) are bitwise those of StepBTrainer.step fed with
    them by hand from the same initial weights; the rest of the step (whose object path adds with fp32 atomics) agrees
    within test_step_b_parity's bounds."""
    data = synth.reference_batch(3, seed=41, lens=[12, 6, 17], n_words=N_WORDS)
    a = _loop(tmp_path / "a", loop_cfg, [data], seed=9)
    b = _loop(tmp_path / "b", loop_cfg, [data], seed=9)
    g = torch.Generator().manual_seed(42)
    z, eps = torch.randn(3, 100, generator=g).to(DEV), torch.randn(3, 100, generator=g).to(DEV)
    # by hand on b: intake, copies, text stage, then the step
    batch, class_ids, _ = trainer.prepare_reference_batch(data)
    dev = b.net.to_device(dict(batch, clabels_emb=b.clabels_emb))
    with torch.no_grad():
        text = trainer.text_stage(b.text_encoder, b.glove, dev["captions"], dev["cap_lens"], dev["glove_captions"],
                                  batch["max_len"])
    dev.update(text, z=z, eps=eps)
    random.seed(5)
    want = b.net.step(dev, class_ids)
    seen = {}
    real = trainer.StepBTrainer.step
    monkeypatch.setattr(trainer.StepBTrainer, "step", lambda self, inp, *x: (seen.update(inp), real(self, inp, *x))[1])
    random.seed(5)
    got = a.train_step(data, z=z, eps=eps)
    for k, v in text.items():
        assert torch.equal(seen[k], v), k
    for k in ("hmaps", "bt_masks", "imgs"):
        assert all(torch.equal(x, y) for x, y in zip(seen[k], dev[k])), k
    assert torch.equal(seen["slabels_feat"], dev["slabels_feat"])
    for x, y in zip(got["fake_imgs"], want["fake_imgs"]):
        assert torch.equal(x, y)
    assert torch.equal(got["errPatD0"], want["errPatD0"])
    for k in ("errG", "kl", "errShpD2"):
        assert abs(float(got[k]) - float(want[k])) <= 1e-3 * max(1.0, abs(float(want[k]))), k
    for x, y in ((a.net.netG, b.net.netG), *zip(a.net.netsPatD, b.net.netsPatD)):
        _check_weights(x, _cpu_sd(y), what="a vs b")


def test_epoch_inception_score(loop_cfg, tmp_path):
    """The per-epoch score is bitwise an InceptionScore over INCEPTION_V3(fake_imgs[-1]) of each step's images."""
    loader = [synth.reference_batch(3, seed=50 + i, n_words=N_WORDS) for i in range(4)]
    t = _loop(tmp_path, loop_cfg, loader)
    score = losses.InceptionScore(min(10, cfg.TRAIN.BATCH_SIZE))
    want = losses.InceptionScore(min(10, cfg.TRAIN.BATCH_SIZE))
    for data in loader:
        out = t.train_step(data, score)
        want.add(t.inception(out["fake_imgs"][-1]))
    assert score.result() == want.result()
    assert all(np.isfinite(score.result()))
    t.write_score(0, score)
    lines = (tmp_path / "Score" / "scores_0.txt").read_text().split("\n")
    assert lines == ["mean, std, mean_conf, std_conf ", "%f, %f, %f, %f" % want.result()]


def test_train_two_epochs_end_to_end(loop_cfg, tmp_path, monkeypatch):
    """2 epochs x 2 batches at B = 2 through train(): every loss of every step finite, the reference's file set
    written, and StepBTrainer.load_model reloads it."""
    monkeypatch.setitem(cfg.TRAIN, "BATCH_SIZE", 2)
    loader = [synth.reference_batch(2, seed=60 + i, n_words=N_WORDS) for i in range(2)]
    t = trainer.condGANTrainer(str(tmp_path), loader, synth.reference_dataset(n_words=N_WORDS),
                               inception_weights=loop_cfg[1], device=DEV)
    seen = []
    real = trainer.condGANTrainer.host_losses
    monkeypatch.setattr(trainer.condGANTrainer, "host_losses", staticmethod(lambda out: seen.append(real(out)) or
                                                                            seen[-1]))
    t.train()
    assert len(seen) == 4 + 2          # PRINT_INTERVAL 1: every step, and each epoch's end
    for h in seen:
        vals = [v for k, v in h.items() if k != "logs" and v is not None] + list(h["logs"].values())
        assert np.isfinite(vals).all(), h
    assert t.net.bG.step == 4
    for e in (0, 1):
        lines = (tmp_path / "Score" / f"scores_{e}.txt").read_text().split("\n")
        assert lines[0] == "mean, std, mean_conf, std_conf " and np.isfinite([float(v) for v in lines[1].split(",")]).all()
    assert {f"netG_epoch_{e}.pth" for e in (0, 1, 2)} <= set(os.listdir(tmp_path / "Model"))
    r = trainer.StepBTrainer(device=DEV)
    assert r.load_model(str(tmp_path / "Model" / "netG_epoch_1.pth")) == 2
    for k, v in t.net.netsPatD[2].state_dict().items():
        assert torch.equal(r.netsPatD[2].state_dict()[k], v), k
    g = torch.load(tmp_path / "Model" / "netG_epoch_2.pth")
    assert all(torch.isfinite(v).all() for v in g.values() if v.is_floating_point())
