"""CPU tests of the training loop (trainer.condGANTrainer) and its batch intake (trainer.prepare_reference_batch): the
caption-length sort, the dtype conversions and the dropped heat maps of the intake; the order of the library calls in
one step; the reference's snapshot and score files, and resuming; and, in a gloo world of two, that only rank 0 writes
and that the Inception predictions are gathered once per epoch.  No kernel runs (a dry run)."""
import os
import re
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dry import dry, record  # noqa: F401
from objgan_b200 import lib, model, synth, trainer
from objgan_b200.config import cfg

N_WORDS = 120


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """The DAMSM encoder snapshots (NET_E) and a torchvision-layout Inception file, written once."""
    d = tmp_path_factory.mktemp("pretrained")
    fast, model.FAST_INIT = model.FAST_INIT, True
    try:
        net_e = synth.reference_encoders(str(d), n_words=N_WORDS)
        inc = str(d / "inception_v3_google.pth")
        torch.save(model._Inception3().state_dict(), inc)
    finally:
        model.FAST_INIT = fast
    return net_e, inc


@pytest.fixture()
def loop_cfg(monkeypatch, files):
    for k, v in dict(MAX_EPOCH=2, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=2, BATCH_SIZE=2, FLAG=True, NET_E=files[0],
                     NET_G="").items():
        monkeypatch.setitem(cfg.TRAIN, k, v)
    return files


def _perm_check(data, batch, class_ids, keys, order):
    imgs, caps, gcaps, lens, hmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks, cids, ks = data
    b = lens.shape[0]
    for i in range(3):
        assert torch.equal(batch["imgs"][i], imgs[i][order])
        assert torch.equal(batch["rois"][i], rois[i][order]) and batch["rois"][i].dtype == torch.float64
        assert batch["bt_masks"][i].dtype == torch.float32
        assert torch.equal(batch["bt_masks"][i], bt_masks[i][order].float())
    assert torch.equal(batch["captions"], caps[order].view(b, -1))
    assert torch.equal(batch["glove_captions"], gcaps[order].view(b, -1))
    assert torch.equal(batch["cap_lens"], lens[order])
    assert torch.equal(batch["fm_rois"], fm_rois[order])
    assert torch.equal(batch["num_rois"], num_rois[order])
    assert batch["fm_bt_masks"].dtype == torch.float32
    assert torch.equal(batch["fm_bt_masks"], fm_bt_masks[order].float())
    assert torch.equal(batch["roi_cls"], rois[0][order][..., 4].to(torch.int64))
    assert (class_ids == cids[order].numpy()).all()
    assert keys == [ks[i] for i in order.tolist()]
    assert "hmaps" not in batch and batch["hmap_clamp"] == 0.0
    assert batch["max_len"] == int(lens.max()) and batch["glb_max_num_roi"] == int(num_rois.max())
    hb = batch["host_boxes"]
    assert all(torch.equal(a, b) for a, b in zip(hb["rois"], batch["rois"]))
    assert torch.equal(hb["fm_rois"], batch["fm_rois"]) and torch.equal(hb["num_rois"], batch["num_rois"])


def test_intake_distinct_lengths():
    data = synth.reference_batch(5, seed=11, lens=[7, 12, 5, 18, 9])
    batch, class_ids, keys = trainer.prepare_reference_batch(data)
    order = torch.sort(data[3], 0, True).indices
    assert order.tolist() == [3, 1, 4, 0, 2]
    _perm_check(data, batch, class_ids, keys, order)


def test_intake_ties_keep_loader_order():
    data = synth.reference_batch(6, seed=12, lens=[9, 12, 9, 12, 5, 9])
    batch, class_ids, keys = trainer.prepare_reference_batch(data)
    order = torch.sort(data[3], dim=0, descending=True, stable=True).indices
    assert order.tolist() == [1, 3, 0, 2, 5, 4]
    _perm_check(data, batch, class_ids, keys, order)


def _trainer(tmp_path, files, batches=2, b=2, seed=20):
    loader = [synth.reference_batch(b, seed=seed + i, n_words=N_WORDS) for i in range(batches)]
    return trainer.condGANTrainer(str(tmp_path), loader, synth.reference_dataset(n_words=N_WORDS),
                                  inception_weights=files[1], device="cpu")


def test_step_call_sequence(dry, loop_cfg, tmp_path, monkeypatch):
    """Intake -> heat maps -> text stage -> the complete step -> INCEPTION_V3, in that order, and nothing read back."""
    t = _trainer(tmp_path, loop_cfg)
    t.setup()
    data = t.data_loader[0]
    t.train_step(data)                        # first step: the text encoder's derived weight copies are built
    events = []
    real_step, real_inc = trainer.StepBTrainer.step, model.INCEPTION_V3.forward
    monkeypatch.setattr(trainer.StepBTrainer, "step",
                        lambda self, *a, **k: (events.append(("<step>", ())), real_step(self, *a, **k))[1])
    monkeypatch.setattr(model.INCEPTION_V3, "forward",
                        lambda self, x: (events.append(("<inception>", ())), real_inc(self, x))[1])
    reads, out = [], []
    monkeypatch.setattr(trainer.condGANTrainer, "host_losses", staticmethod(lambda out: reads.append(1)))
    events = [name for name, _ in record(lambda: out.append(t.train_step(data)), events)]
    out = out[0]
    s, i = events.index("<step>"), events.index("<inception>")
    text = [e for e in events[:s] if e in ("og_gather_rows", "og_conv2d_simt", "og_lstm_bidir", "og_text_inputs")]
    assert text == ["og_gather_rows", "og_conv2d_simt", "og_lstm_bidir", "og_text_inputs"]
    first_text = events.index("og_gather_rows")
    assert set(events[:first_text]) <= {"og_form_hmaps", "og_form_clabels_feat"} and "og_form_hmaps" in events[:s]
    assert events[events.index("og_text_inputs") + 1] == "<step>"
    assert s < i and len(events[s + 1:i]) > 300 and len(events[i + 1:]) > 50
    assert not reads
    assert [tuple(f.shape) for f in out["fake_imgs"]] == [(2, 3, 64, 64), (2, 3, 128, 128), (2, 3, 256, 256)]
    assert tuple(out["predictions"].shape) == (2, 1000)


SCORE_LINE = re.compile(r"^[-+\w.]+, [-+\w.]+, [-+\w.]+, [-+\w.]+$")
MODEL_FILES = {"netPatD0.pth", "netPatD1.pth", "netPatD2.pth", "netShpD0.pth", "netShpD1.pth", "netShpD2.pth",
               "netObjSSD.pth", "netObjLSD.pth"}


def test_files_and_resume(dry, loop_cfg, tmp_path, monkeypatch, capsys):
    import numpy as np
    reads = []
    real = trainer.condGANTrainer.host_losses
    monkeypatch.setattr(trainer.condGANTrainer, "host_losses", staticmethod(lambda out: (reads.append(1), real(out))[1]))
    t = _trainer(tmp_path, loop_cfg)
    with np.errstate(all="ignore"):
        t.train()
    # 2 epochs x 2 batches: print steps 2 and 4, and each epoch's end
    assert len(reads) == 4
    log = capsys.readouterr().out
    assert log.count("errPatD0: ") == 2 and log.count("Loss_PatD: ") == 2 and log.count("inception_score: ") == 4
    got = set(os.listdir(tmp_path / "Model"))
    assert got == MODEL_FILES | {"netG_epoch_0.pth", "netG_epoch_1.pth", "netG_epoch_2.pth"}
    assert sorted(os.listdir(tmp_path / "Score")) == ["scores_0.txt", "scores_1.txt"]
    assert os.path.isdir(tmp_path / "Image")
    for e in (0, 1):
        lines = (tmp_path / "Score" / f"scores_{e}.txt").read_text().split("\n")
        assert lines[0] == "mean, std, mean_conf, std_conf " and len(lines) == 2 and SCORE_LINE.match(lines[1])
    g = torch.load(tmp_path / "Model" / "netG_epoch_1.pth")
    assert set(g) == set(t.net.netG.state_dict())
    # resume: NET_G names the epoch-1 generator, the discriminators come from the same directory
    monkeypatch.setitem(cfg.TRAIN, "NET_G", str(tmp_path / "Model" / "netG_epoch_1.pth"))
    monkeypatch.setitem(cfg.TRAIN, "MAX_EPOCH", 3)
    out2 = tmp_path / "resumed"
    t2 = _trainer(out2, loop_cfg)
    with np.errstate(all="ignore"):
        t2.train()
    assert sorted(os.listdir(out2 / "Score")) == ["scores_2.txt"]
    assert {f for f in os.listdir(out2 / "Model") if f.startswith("netG")} == {"netG_epoch_2.pth", "netG_epoch_3.pth"}
    assert t2.net.bG.step == 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, files, outdirs, res):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import numpy as np
    lib.DRY_RUN = True
    model.FAST_INIT = True
    cfg.TRAIN.update(MAX_EPOCH=2, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=100, BATCH_SIZE=2, NET_E=files[0], NET_G="")
    torch.manual_seed(300 + rank)
    gathers = []
    real = dist.all_gather

    def counted(tensors, t, *a, **k):
        if t.dim() == 2:
            gathers.append(tuple(t.shape))
        return real(tensors, t, *a, **k)
    dist.all_gather = counted
    loader = [synth.reference_batch(2, seed=40 + 10 * rank + i, n_words=N_WORDS) for i in range(2)]
    t = trainer.condGANTrainer(outdirs[rank], loader, synth.reference_dataset(n_words=N_WORDS),
                               inception_weights=files[1], device="cpu")
    with np.errstate(all="ignore"):
        t.train()
    res[rank] = (t.world, t.rank, gathers, t.net.bG.step)
    dist.destroy_process_group()


def test_data_parallel_gloo(tmp_path, files):
    world = 2
    outdirs = [str(tmp_path / f"rank{r}") for r in range(world)]
    mgr = mp.Manager()
    res = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), files, outdirs, res), nprocs=world, join=True)
    for r in range(world):
        w, rank, gathers, steps = res[r]
        assert w == world and rank == r and steps == 4
        assert gathers == [(4, 1000), (4, 1000)]          # the predictions: one gather per epoch
    assert sorted(os.listdir(os.path.join(outdirs[0], "Score"))) == ["scores_0.txt", "scores_1.txt"]
    assert "netG_epoch_2.pth" in os.listdir(os.path.join(outdirs[0], "Model"))
    assert not os.path.exists(outdirs[1])
