"""CPU tests of the snapshot PNGs in the two loops, without a GPU (a dry run: no kernel runs, the canvases hold
whatever memory they were given): the trainer's epoch-numbered file set in Image/ through train(), on display steps
only, one og_snapshot_canvas call and one device -> host read per PNG, the writer drained before train() returns, its
errors surfaced without replacing the loop's own, the warning without a font, and in a gloo world of two only rank 0
rendering; the evaluator's file set per mode and SAVE_OPTIONS, drained before evaluate() returns, and nothing written
without a font."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from PIL import ImageFont

from dry import dry, record  # noqa: F401
from objgan_b200 import evaluator, lib, model, ops, snapshots, synth, trainer
from objgan_b200.config import cfg
from objgan_b200.sampler import GSampler

N_WORDS = 120
DIMS = 64
FONT = ImageFont.load_default(size=50)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("pretrained")
    fast, model.FAST_INIT = model.FAST_INIT, True
    try:
        net_e = synth.reference_encoders(str(d), n_words=N_WORDS)
        torch.save(model.G_NET(80).state_dict(), d / "netG_epoch_120.pth")
        torch.save(model.SHP_G_NET(80).state_dict(), d / "shape_gen.pth")
        inc = str(d / "inception_v3_google.pth")
        torch.save(model._Inception3().state_dict(), inc)
    finally:
        model.FAST_INIT = fast
    return dict(net_e=net_e, net_g=str(d / "netG_epoch_120.pth"), shp=str(d / "shape_gen.pth"), inc=inc)


@pytest.fixture()
def cfg_restore(monkeypatch):
    for k in list(cfg.TRAIN):
        monkeypatch.setitem(cfg.TRAIN, k, cfg.TRAIN[k])
    for k in list(cfg.TEST):
        monkeypatch.setitem(cfg.TEST, k, cfg.TEST[k])
    monkeypatch.setitem(cfg, "DATA_DIR", "/nonexistent")


def _dataset():
    ds = synth.reference_dataset(n_words=N_WORDS)
    ds.ixtoword = {i: "w%d" % i for i in range(N_WORDS)}
    return ds


def _trainer(out, files, font, batches=2):
    cfg.TRAIN.update(MAX_EPOCH=2, SNAPSHOT_INTERVAL=1, PRINT_INTERVAL=100, BATCH_SIZE=2, FLAG=True,
                     NET_E=files["net_e"], NET_G="", DISPLAY_INTERVAL=3)
    loader = [synth.reference_batch(2, seed=20 + i, n_words=N_WORDS) for i in range(batches)]
    return trainer.condGANTrainer(str(out), loader, _dataset(), inception_weights=files["inc"], device="cpu",
                                  font=font)


def _count(monkeypatch, fn):
    """Runs ``fn()`` and returns (its result, its og_snapshot_canvas calls, canvas reads and writer closes)."""
    n = dict(read=0, close=0)
    real_read, real_close = snapshots._to_host, snapshots.PngWriter.close

    def read(t):
        n["read"] += 1
        return real_read(t)

    def close(self, *a, **k):
        n["close"] += 1
        return real_close(self, *a, **k)
    monkeypatch.setattr(snapshots, "_to_host", read)
    monkeypatch.setattr(snapshots.PngWriter, "close", close)
    out = []
    n["canvas"] = sum(name == "og_snapshot_canvas" for name, _ in record(lambda: out.append(fn())))
    return out[0], n


# ------------------------------------------------------------------------------------------------------ trainer
def test_trainer_files_on_display_steps(dry, cfg_restore, files, tmp_path, monkeypatch):
    """2 epochs x 2 steps, DISPLAY_INTERVAL 3: one display, at step 3 (epoch 1), five PNGs named by the epoch."""
    t = _trainer(tmp_path, files, FONT)
    displays = []
    real = trainer.condGANTrainer.save_img_results
    monkeypatch.setattr(trainer.condGANTrainer, "save_img_results",
                        lambda self, epoch, w: (displays.append(epoch), real(self, epoch, w))[1])
    with np.errstate(all="ignore"):
        _, n = _count(monkeypatch, t.train)
    assert displays == [1]
    assert sorted(os.listdir(tmp_path / "Image")) == sorted(
        ["G_average_1_0.png", "G_average_1_1.png", "bt_G_average_1_0.png", "bt_G_average_1_1.png",
         "D_average_1.png"])
    assert n == dict(canvas=5, read=5, close=1)              # one canvas and one read per PNG; drained once
    assert t.fixed_noise.shape == (2, cfg.GAN.Z_DIM)


def test_trainer_without_font_warns_once_and_writes_nothing(dry, cfg_restore, files, tmp_path, monkeypatch):
    t = _trainer(tmp_path, files, None)
    cfg.TRAIN.DISPLAY_INTERVAL = 1
    t.display_interval = 1
    with np.errstate(all="ignore"), pytest.warns(UserWarning, match="attention-map PNGs") as rec:
        _, n = _count(monkeypatch, t.train)
    assert len([w for w in rec if "attention-map" in str(w.message)]) == 1
    assert os.listdir(tmp_path / "Image") == [] and n["canvas"] == 0 and n["read"] == 0
    assert t.fixed_noise is None


def test_trainer_writer_error_surfaces(dry, cfg_restore, files, tmp_path, monkeypatch):
    monkeypatch.setattr(snapshots.Canvas, "pixels", lambda self: (_ for _ in ()).throw(OSError("disk full")))
    t = _trainer(tmp_path, files, FONT)
    with np.errstate(all="ignore"), pytest.raises(RuntimeError, match="snapshot PNG"):
        t.train()


def test_trainer_loop_error_is_not_replaced(dry, cfg_restore, files, tmp_path, monkeypatch):
    """A failing step after a failed PNG: the step's exception leaves train(), not the writer's."""
    monkeypatch.setattr(snapshots.Canvas, "pixels", lambda self: (_ for _ in ()).throw(OSError("disk full")))
    t = _trainer(tmp_path, files, FONT, batches=2)
    real, calls = trainer.condGANTrainer.train_step, []

    def step(self, *a, **k):
        calls.append(1)
        if len(calls) == 4:
            raise KeyError("the step failed")
        return real(self, *a, **k)
    monkeypatch.setattr(trainer.condGANTrainer, "train_step", step)
    with np.errstate(all="ignore"), pytest.raises(KeyError, match="the step failed"):
        t.train()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, files, outdirs, res):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lib.DRY_RUN = True
    model.FAST_INIT = True
    cfg.DATA_DIR = "/nonexistent"
    torch.manual_seed(300 + rank)
    t = _trainer(outdirs[rank], files, FONT)
    with np.errstate(all="ignore"):
        calls = record(t.train)
    res[rank] = (t.rank, sum(name == "og_snapshot_canvas" for name, _ in calls), t.fixed_noise is not None)
    dist.destroy_process_group()


def test_trainer_only_rank0_renders_gloo(tmp_path, files):
    world = 2
    outdirs = [str(tmp_path / f"rank{r}") for r in range(world)]
    mgr = mp.Manager()
    res = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), files, outdirs, res), nprocs=world, join=True)
    assert res[0] == (0, 5, True) and res[1] == (1, 0, True)    # both draw fixed_noise; rank 0 alone renders
    assert len(os.listdir(os.path.join(outdirs[0], "Image"))) == 5
    assert not os.path.exists(outdirs[1])


# ---------------------------------------------------------------------------------------------------- evaluator
def _seeded_scores(tag):
    def score_images(self, fake_imgs):
        b = fake_imgs[-1].shape[0]
        g = torch.Generator().manual_seed(tag)
        p = torch.rand(b, 1000, generator=g) + 0.01
        return p / p.sum(1, keepdim=True), torch.randn(b, DIMS, generator=g)
    return score_images


def _moments_cpu(x, k, s1, s2, init):
    x = x.detach().double()
    if init:
        k.copy_(x[0])
        s1.zero_()
        s2.zero_()
    d = x - k
    s1 += d.sum(0)
    s2 += d.T @ d


def _evaluate(out, files, mode, options, font, monkeypatch):
    monkeypatch.setattr(ops, "moments_f64", _moments_cpu)
    monkeypatch.setattr(GSampler, "score_images", _seeded_scores(mode))
    cfg.TRAIN.update(BATCH_SIZE=2, DISPLAY_INTERVAL=2, NET_E=files["net_e"], NET_G=files["net_g"])
    cfg.TEST.update(USE_GT_BOX_SEG=mode, NET_SHP_G=files["shp"], RP_POOL_SIZE=4, FID_DIMS=DIMS, USE_TF=0,
                    TEST_IMG_NUM=1000000, SAVE_OPTIONS=options)
    loader = [synth.reference_test_batch(2, seed=20 + i, mode=mode, full_maps=False, n_words=N_WORDS, fid_dims=DIMS)
              for i in range(4)]
    ds = synth.reference_test_dataset(n_words=N_WORDS)
    ds.ixtoword = {i: "w%d" % i for i in range(N_WORDS)}
    e = evaluator.condGANEvaluator(str(out), loader, ds, inception_weights=files["inc"], device="cpu", font=font)
    with np.errstate(all="ignore"):
        e.evaluate("test", [64, 128, 256])
    return sorted(os.listdir(out / "Snapshot"))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_evaluator_snapshot_files(dry, cfg_restore, files, tmp_path, mode, monkeypatch):
    """SNAPSHOT, DISPLAY_INTERVAL 2 over 4 batches: displays at 0 and 2.  G_ / bt_G_ per stage; ShapeG_ in modes 1
    and 2; ShapeD_ in mode 1.  One canvas and one read per PNG, drained before evaluate() returns."""
    got, n = _count(monkeypatch, lambda: _evaluate(tmp_path, files, mode, "SNAPSHOT", FONT, monkeypatch))
    want = []
    for it in (0, 2):
        want += ["G_%d_0.png" % it, "G_%d_1.png" % it, "bt_G_%d_0.png" % it, "bt_G_%d_1.png" % it]
        want += ["ShapeG_%d.png" % it] if mode > 0 else []
        want += ["ShapeD_%d.png" % it] if mode == 1 else []
    assert got == sorted(want)
    assert n["canvas"] == n["read"] == len(want) and n["close"] == 1


@pytest.mark.parametrize("mode", [1, 2])
def test_evaluator_shape_files_in_image_mode(dry, cfg_restore, files, tmp_path, mode, monkeypatch):
    got = _evaluate(tmp_path, files, mode, "IMAGE", FONT, monkeypatch)
    want = ["ShapeG_0.png", "ShapeG_2.png"] + (["ShapeD_0.png", "ShapeD_2.png"] if mode == 1 else [])
    assert got == sorted(want)


@pytest.mark.parametrize("mode", [1, 2])
def test_evaluator_without_font_writes_no_png(dry, cfg_restore, files, tmp_path, mode, monkeypatch):
    with pytest.warns(UserWarning, match="attention-map PNGs"):
        got, n = _count(monkeypatch, lambda: _evaluate(tmp_path, files, mode, "SNAPSHOT", None, monkeypatch))
    assert got == [] and n["canvas"] == 0
