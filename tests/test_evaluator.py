"""CPU tests of the evaluation loop (evaluator.condGANEvaluator) and its batch intake
(trainer.prepare_reference_test_batch): the caption-length sort of all three cfg.TEST.USE_GT_BOX_SEG modes and the
tensors it never reads; the order of the library calls of one batch; the score file, TEST_IMG_NUM, the saved images
and the refusals; dump_fid_acts' file; _Moments.merge; and, in a gloo world of two, the scores over both ranks written
by rank 0 alone.  No kernel runs (lib.DRY_RUN): where a test needs real numbers, the scoring networks' outputs are
seeded and og_moments_f64 is restated on the CPU."""
import os
import pickle
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dry import dry, record  # noqa: F401
from objgan_b200 import evaluator, lib, losses, model, ops, synth, trainer
from objgan_b200.config import cfg
from objgan_b200.sampler import GSampler

N_WORDS = 120
DIMS = 64


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """NET_E, a generator and a shape generator snapshot, and a torchvision-layout Inception file."""
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


def _set_cfg(files, mode, **test):
    cfg.TRAIN.update(BATCH_SIZE=2, DISPLAY_INTERVAL=2, NET_E=files["net_e"], NET_G=files["net_g"])
    cfg.TEST.update(dict(USE_GT_BOX_SEG=mode, NET_SHP_G=files["shp"], RP_POOL_SIZE=4, FID_DIMS=DIMS, USE_TF=0,
                         TEST_IMG_NUM=1000000, SAVE_OPTIONS="IMAGE"), **test)


@pytest.fixture()
def eval_cfg(monkeypatch, files):
    for k in ("BATCH_SIZE", "DISPLAY_INTERVAL", "NET_E", "NET_G"):
        monkeypatch.setitem(cfg.TRAIN, k, cfg.TRAIN[k])
    for k in list(cfg.TEST):
        monkeypatch.setitem(cfg.TEST, k, cfg.TEST[k])
    return files


def _moments_cpu(x, k, s1, s2, init):
    """og_moments_f64 restated (full s2)."""
    x = x.detach().double()
    if init:
        k.copy_(x[0])
        s1.zero_()
        s2.zero_()
    d = x - k
    s1 += d.sum(0)
    s2 += d.T @ d


def _seeded_scores(tag):
    """GSampler.score_images replaced by seeded outputs: (predictions (B, 1000) rows summing to 1, activations)."""
    count = [0]

    def score_images(self, fake_imgs):
        b = fake_imgs[-1].shape[0]
        g = torch.Generator().manual_seed(1000 * tag + count[0])
        count[0] += 1
        p = torch.rand(b, 1000, generator=g) + 0.01
        return p / p.sum(1, keepdim=True), torch.randn(b, DIMS, generator=g)
    return score_images


def _evaluator(out_dir, files, loader, mode=2, **test):
    _set_cfg(files, mode, **test)
    return evaluator.condGANEvaluator(str(out_dir), loader, synth.reference_test_dataset(n_words=N_WORDS),
                                      inception_weights=files["inc"], device="cpu")


def _loader(mode, n, b=2, seed=20):
    return [synth.reference_test_batch(b, seed=seed + i, mode=mode, full_maps=False, n_words=N_WORDS, fid_dims=DIMS)
            for i in range(n)]


# ---------------------------------------------------------------------------------------------------------------------
# intake
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_intake(mode):
    data = synth.reference_test_batch(6, seed=12, mode=mode, lens=[9, 12, 9, 12, 5, 9], n_words=N_WORDS,
                                      fid_dims=DIMS)
    assert len(data) == (14 if mode == 2 else 17)
    batch, acts, class_ids, keys, sent_ids = trainer.prepare_reference_test_batch(data, mode)
    r = 9 if mode < 2 else 8                                 # rois, fm_rois, num_rois follow the box maps
    lens, rois, fm_rois, num_rois = data[4], data[r], data[r + 1], data[r + 2]
    order = torch.sort(lens, dim=0, descending=True, stable=True).indices
    assert order.tolist() == [1, 3, 0, 2, 5, 4]                          # ties keep the loader's order
    assert torch.equal(acts, data[1][order]) and acts.dtype == torch.float64
    assert (class_ids == data[-3][order].numpy()).all()
    assert keys == [data[-2][i] for i in order.tolist()] and sent_ids == data[-1][order].tolist()
    assert torch.equal(batch["captions"], data[2][order].view(6, -1))
    assert torch.equal(batch["glove_captions"], data[3][order].view(6, -1))
    assert torch.equal(batch["cap_lens"], lens[order]) and batch["max_len"] == 12
    for i in range(3):
        assert batch["rois"][i].dtype == torch.float64 and torch.equal(batch["rois"][i], rois[i][order])
    assert torch.equal(batch["fm_rois"], fm_rois[order]) and batch["fm_rois"].dtype == torch.float64
    assert torch.equal(batch["num_rois"], num_rois[order]) and batch["glb_max_num_roi"] == int(num_rois.max())
    assert torch.equal(batch["roi_cls"], rois[0][order][..., 4].long())
    assert not {"imgs", "hmaps", "bbox_maps_fwd", "bbox_maps_bwd", "bbox_fmaps"} & set(batch)
    if mode == 0:
        bt, fm = data[12], data[13]
        assert all(m.dtype == torch.float32 and torch.equal(m, x[order].float()) for m, x in zip(batch["bt_masks"], bt))
        assert batch["fm_bt_masks"].dtype == torch.float32 and torch.equal(batch["fm_bt_masks"], fm[order].float())
        assert batch["hmap_clamp"] == 0.0
    else:
        assert "bt_masks" not in batch and "fm_bt_masks" not in batch


def test_intake_never_reads_maps_or_images():
    """The images, heat maps and box maps of the tuple are objects whose every use raises."""
    class Untouchable:
        def __getattr__(self, name):
            raise AssertionError(f"read: {name}")

        def __getitem__(self, i):
            raise AssertionError("indexed")
    for mode in (0, 1, 2):
        data = list(synth.reference_test_batch(3, seed=5, mode=mode, full_maps=False, n_words=N_WORDS, fid_dims=DIMS))
        skip = [0, 5, 6, 7] if mode == 2 else [0, 5, 6, 7, 8]
        for i in skip:
            data[i] = Untouchable()
        trainer.prepare_reference_test_batch(tuple(data), mode)


def test_intake_wrong_tuple_length():
    with pytest.raises(ValueError, match="17-field"):
        trainer.prepare_reference_test_batch(synth.reference_test_batch(2, seed=1, mode=2, full_maps=False), 0)
    with pytest.raises(ValueError, match="14-field"):
        trainer.prepare_reference_test_batch(synth.reference_test_batch(2, seed=1, mode=1, full_maps=False), 2)


def test_test_batch_box_maps_are_the_loaders():
    """The float64 box maps of the synthetic tuple are the load.py rasterisation the device rebuilds them with."""
    from oracle import shape_oracle as S
    data = synth.reference_test_batch(2, seed=3, mode=2, n_words=N_WORDS, fid_dims=DIMS)
    fwd, bwd, fm = data[5:8]
    assert fwd.dtype == torch.float64 and fwd.shape == (2, 10, 80, 64, 64) and fm.shape == (2, 10, 16, 16)
    want = S.bbox_maps(data[8][0], data[9], data[10], 10, 80)
    assert torch.equal(fwd.float(), want[0]) and torch.equal(bwd.float(), want[1]) and torch.equal(fm.float(), want[2])
    assert fwd.sum() > 0


# ---------------------------------------------------------------------------------------------------------------------
# one batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_batch_call_sequence(mode, dry, eval_cfg, tmp_path, monkeypatch):
    e = _evaluator(tmp_path, eval_cfg, _loader(mode, 2), mode)
    e.build_models()
    rp, is_, fid = losses.RPrecision(4), losses.InceptionScore(2), losses.FrechetDistance(DIMS)
    e.evaluate_batch(e.data_loader[0], rp, is_, fid)          # first batch: derived weight copies built
    events = []
    for cls, meth, tag in ((model.SHP_G_NET, "forward_nhwc", "<shp_g>"), (model.G_NET, "forward", "<g>"),
                           (model.CNN_ENCODER, "forward", "<cnn>"), (model.INCEPTION_V3, "forward", "<inception>"),
                           (model.INCEPTION_V3_FID, "activations", "<inception_fid>")):
        real = getattr(cls, meth)
        monkeypatch.setattr(cls, meth, (lambda r, t: lambda self, *a, **k: (events.append((t, ())),
                                                                            r(self, *a, **k))[1])(real, tag))
    events = [name for name, _ in record(lambda: e.evaluate_batch(e.data_loader[1], rp, is_, fid), events)]
    marks = ["og_gather_rows", "og_form_bbox_maps", "og_gen_hmaps", "og_form_hmaps", "<shp_g>", "<g>", "<cnn>",
             "<inception>", "<inception_fid>"]
    seq = [x for x in events if x in marks]
    seq = [x for i, x in enumerate(seq) if x != "og_gather_rows" or "og_gather_rows" not in seq[:i]]
    seq = [x for i, x in enumerate(seq) if i == 0 or x != seq[i - 1]]     # og_form_hmaps: one call per scale
    if mode > 0:
        assert seq == ["og_gather_rows", "og_form_bbox_maps", "<shp_g>", "og_gen_hmaps", "<g>", "<cnn>", "<inception>",
                       "<inception_fid>"]
    else:
        assert seq == ["og_form_hmaps", "og_gather_rows", "<g>", "<cnn>", "<inception>", "<inception_fid>"]
    assert "og_images_to_u8" not in events                    # not a display batch


_READS = ("cpu", "tolist", "item", "numpy", "__int__", "__float__", "__index__", "__bool__")


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_batch_host_reads(mode, dry, eval_cfg, tmp_path, monkeypatch):
    """Past the host intake, a batch reads tensors to the host only in the sampler's caption check, and the batch that
    finds the R-precision pool full also in that pool's scoring.  Every way a tensor's values reach Python is counted
    (Tensor.cpu / tolist / item / numpy and the int / float / index / bool conversions) and attributed to the
    function of the library that asked for it."""
    import sys
    loader = _loader(mode, 4)
    e = _evaluator(tmp_path, eval_cfg, loader, mode)          # B = 2, RP_POOL_SIZE = 4: batch 3 scores the pool
    e.build_models()
    rp, is_, fid = losses.RPrecision(4), losses.InceptionScore(2), losses.FrechetDistance(DIMS)
    e.evaluate_batch(loader[0], rp, is_, fid)                 # first batch: derived weight copies built
    staged = iter([trainer.prepare_reference_test_batch(d, mode) for d in loader[1:]])
    monkeypatch.setattr(evaluator, "prepare_reference_test_batch", lambda data, mode=None: next(staged))
    reads = []

    def caller():
        f = sys._getframe(2)
        names = set()
        while f is not None:
            names.add(f.f_code.co_name)
            f = f.f_back
        return "caption check" if "_text_mode" in names else "pool score" if "_score" in names else "other"

    for name in _READS:
        real = getattr(torch.Tensor, name)
        monkeypatch.setattr(torch.Tensor, name, (lambda r, n: lambda self, *a, **k: (reads.append((n, caller())),
                                                                                     r(self, *a, **k))[1])(real, name))
    per_batch = []
    for data in loader[1:]:
        reads.clear()
        e.evaluate_batch(data, rp, is_, fid)
        per_batch.append({c for _, c in reads})
        assert ("tolist", "caption check") in reads
    monkeypatch.undo()
    assert per_batch == [{"caption check"}, {"caption check", "pool score"}, {"caption check"}], per_batch
    assert len(rp.w_accuracy) == 1


# ---------------------------------------------------------------------------------------------------------------------
# files and refusals
# ---------------------------------------------------------------------------------------------------------------------
SCORE_LINE = re.compile(r"^([-+\w.]+, ){8}[-+\w.]+$")


def test_files_interval_and_cap(dry, eval_cfg, tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(ops, "moments_f64", _moments_cpu)
    monkeypatch.setattr(GSampler, "score_images", _seeded_scores(1))
    loader = _loader(2, 6)
    e = _evaluator(tmp_path, eval_cfg, loader, 2, TEST_IMG_NUM=5)
    seen = []
    real = e.evaluate_batch
    e.evaluate_batch = lambda data, *a, **k: (seen.append(data), real(data, *a, **k))[1]
    res = e.evaluate("test", [64, 128, 256])
    assert len(seen) == 5                                     # TEST_IMG_NUM counts batches
    lines = (tmp_path / "Score" / "scores.txt").read_text().split("\n")
    assert lines[0] == "mean, std, mean_conf, std_conf, accu_w, std_w, accu_s, std_s, fid_score "
    assert len(lines) == 2 and SCORE_LINE.match(lines[1])
    assert lines[1] == "%f, %f, %f, %f, %f, %f, %f, %f, %f" % res["scores"]
    assert len(res["w_accuracy"]) == 1                        # batch 3 scores the pool of batches 1-2
    log = capsys.readouterr().out
    assert log.count("inception_score: ") == 2
    # DISPLAY_INTERVAL 2: batches 0, 2 and 4 write <key>_<sent_id>.jpg
    want = set()
    for i in (0, 2, 4):
        _, _, _, keys, sent_ids = trainer.prepare_reference_test_batch(loader[i], 2)
        want |= {f"{k}_{s}.jpg" for k, s in zip(keys, sent_ids)}
    assert set(os.listdir(tmp_path / "Image")) == want
    assert {"Model", "Image", "Snapshot", "Score"} <= set(os.listdir(tmp_path))


def test_no_scored_pool_gives_nan(dry, eval_cfg, tmp_path, monkeypatch):
    monkeypatch.setattr(ops, "moments_f64", _moments_cpu)
    monkeypatch.setattr(GSampler, "score_images", _seeded_scores(2))
    e = _evaluator(tmp_path, eval_cfg, _loader(2, 2), 2, RP_POOL_SIZE=100)
    res = e.evaluate("test", [64, 128, 256])
    assert np.isnan(res["scores"][4:8]).all() and np.isfinite(res["scores"][:4]).all()


def test_refusals(eval_cfg, tmp_path):
    with pytest.raises(ValueError, match="USE_TF"):
        _evaluator(tmp_path, eval_cfg, [], 2, USE_TF=1)
    with pytest.raises(ValueError, match="SAVE_OPTIONS"):
        _evaluator(tmp_path, eval_cfg, [], 2, SAVE_OPTIONS="PNG")
    assert not os.path.exists(tmp_path / "Score")


def test_snapshot_warns_once(dry, eval_cfg, tmp_path, monkeypatch):
    monkeypatch.setattr(ops, "moments_f64", _moments_cpu)
    monkeypatch.setattr(GSampler, "score_images", _seeded_scores(3))
    e = _evaluator(tmp_path, eval_cfg, _loader(2, 4), 2, SAVE_OPTIONS="SNAPSHOT")
    with pytest.warns(UserWarning, match="attention-map PNGs") as rec:
        e.evaluate("test", [64, 128, 256])
    assert len([w for w in rec if "attention-map" in str(w.message)]) == 1
    assert os.listdir(tmp_path / "Image") == []


# ---------------------------------------------------------------------------------------------------------------------
# dump_fid_acts
# ---------------------------------------------------------------------------------------------------------------------
def test_dump_fid_acts(dry, eval_cfg, tmp_path):
    loader = synth.reference_acts_batches(2, 3, seed=9)
    e = _evaluator(tmp_path / "out", eval_cfg, loader, 2)
    e.dump_fid_acts(str(tmp_path), "test")
    path = tmp_path / "test_acts_tf0.pickle"
    raw = path.read_bytes()
    assert raw[:2] == b"\x80\x02"                             # pickle protocol 2
    obj = pickle.loads(raw)
    assert isinstance(obj, list) and len(obj) == 1
    acts = obj[0]
    assert set(acts) == {k for _, keys in loader for k in keys}
    assert all(v.dtype == np.float64 and v.shape == (DIMS,) for v in acts.values())
    got = evaluator.load_acts_data(str(tmp_path), "test")
    assert got.keys() == acts.keys() and all(np.array_equal(got[k], acts[k], equal_nan=True) for k in acts)
    before = path.stat().st_mtime_ns
    e.dump_fid_acts(str(tmp_path), "test")                    # an existing file is left alone
    assert path.read_bytes() == raw and path.stat().st_mtime_ns == before


# ---------------------------------------------------------------------------------------------------------------------
# _Moments.merge
# ---------------------------------------------------------------------------------------------------------------------
def test_moments_merge():
    rng = np.random.default_rng(4)
    d = 70
    rows = rng.normal(size=(31, d)) * 2.5 + 7.0
    tiles = np.arange(d) // 32
    upper = torch.from_numpy(tiles[:, None] <= tiles[None, :])
    parts = []
    for lo, hi, shift in ((0, 3, 0), (3, 22, 5), (22, 31, 17)):
        x = torch.from_numpy(rows[lo:hi])
        k = torch.from_numpy(rows[lo + shift % (hi - lo)].copy())          # each "rank" shifted by another row
        s2 = (x - k).T @ (x - k)
        s2 = torch.where(upper, s2, torch.full_like(s2, float("nan")))    # og_moments_f64 leaves the lower tiles
        parts.append(losses._Moments.from_sums(hi - lo, k, (x - k).sum(0), s2))
    mu, sigma = parts[0].merge(parts[1:]).statistics()
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
    assert rel(mu, rows.mean(0)) <= 1e-12 and rel(sigma, np.cov(rows, rowvar=False)) <= 1e-12
    empty = losses._Moments(d)
    mu2, sigma2 = empty.merge(parts).statistics()
    assert rel(mu2, rows.mean(0)) <= 1e-12 and rel(sigma2, np.cov(rows, rowvar=False)) <= 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# data parallel
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_loader(rank):
    return _loader(2, 3, seed=50 + 10 * rank)


def _worker(rank, world, port, files, outdirs, data_dir, res):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lib.DRY_RUN = True
    model.FAST_INIT = True
    # the real images' activations first, as main.py does before evaluate(): rank 0 writes slowly, and every rank
    # reads the file back as soon as dump_fid_acts returns
    import time
    real_dump = pickle.dump
    if rank == 0:
        evaluator.pickle.dump = lambda *a, **k: (time.sleep(1.0), real_dump(*a, **k))[1]
    acts_loader = synth.reference_acts_batches(2, 2, seed=80 + 10 * rank)
    e = _evaluator(outdirs[rank], files, acts_loader, 2)
    e.dump_fid_acts(data_dir, "test")
    acts = evaluator.load_acts_data(data_dir, "test")
    e.dump_fid_acts(data_dir, "test")                    # the file exists: every rank returns at once
    evaluator.pickle.dump = real_dump
    res[f"acts{rank}"] = None if acts is None else sorted(acts)
    ops.moments_f64 = _moments_cpu
    GSampler.score_images = _seeded_scores(10 + rank)
    seen = {}
    real_fd, real_is = losses.frechet_distance, evaluator.gather_inception_score

    def fd(mu1, s1, mu2, s2):
        seen["fid"] = (mu1, s1, mu2, s2)
        return real_fd(mu1, s1, mu2, s2)

    def gis(*a):
        out = real_is(*a)
        seen["is_rows"] = None if out is None else int(torch.cat(out.predictions).shape[0])
        return out
    losses.frechet_distance = fd
    evaluator.gather_inception_score = gis
    e = _evaluator(outdirs[rank], files, _rank_loader(rank), 2)
    with np.errstate(all="ignore"):
        out = e.evaluate("test", [64, 128, 256])
    res[rank] = (e.world, e.rank, out, seen)
    dist.destroy_process_group()


def test_data_parallel_gloo(tmp_path, files):
    world = 2
    outdirs = [str(tmp_path / f"rank{r}") for r in range(world)]
    mgr = mp.Manager()
    res = mgr.dict()
    data_dir = str(tmp_path / "data")
    os.makedirs(data_dir)
    mp.spawn(_worker, args=(world, _free_port(), files, outdirs, data_dir, res), nprocs=world, join=True)
    for r in range(world):
        assert res[r][:2] == (world, r)
    keys = sorted(k for r in range(world) for _, ks in synth.reference_acts_batches(2, 2, seed=80 + 10 * r) for k in ks)
    assert res["acts0"] == keys and res["acts1"] == keys      # both ranks' shards, readable on both ranks
    assert os.listdir(data_dir) == ["test_acts_tf0.pickle"]
    assert res[1][2] is None and "fid" not in res[1][3]
    out, seen = res[0][2], res[0][3]
    assert seen["is_rows"] == 2 * 3 * 2                       # both ranks' predictions
    assert len(out["w_accuracy"]) == 2 and len(out["s_accuracy"]) == 2   # one pool per rank
    # FID from the merged moments: every rank's real activations and seeded generated ones
    real = np.concatenate([np.concatenate([d[1].numpy() for d in _rank_loader(r)]) for r in range(world)])
    fake = []
    for r in range(world):
        f = _seeded_scores(10 + r)
        fake += [f(None, [torch.zeros(2)])[1].double().numpy() for _ in range(3)]
    fake = np.concatenate(fake)
    mu1, s1, mu2, s2 = seen["fid"]
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
    assert rel(mu1, real.mean(0)) <= 1e-12 and rel(s1, np.cov(real, rowvar=False)) <= 1e-12
    assert rel(mu2, fake.mean(0)) <= 1e-12 and rel(s2, np.cov(fake, rowvar=False)) <= 1e-12
    assert os.listdir(os.path.join(outdirs[0], "Score")) == ["scores.txt"]
    assert not os.path.exists(outdirs[1])
