"""The evaluation loop (evaluator.condGANEvaluator) on the GPU: og_images_to_u8 bitwise against the reference's torch
expression; five batches of every cfg.TEST.USE_GT_BOX_SEG mode on both engines against the oracle composition (the
sort, text_oracle, the loader's own float64 box maps -> shape_oracle -> form_hmaps or the loader's heat maps,
eval-mode G_NET, image_encoder_oracle, inception_oracle, and the reference's R-precision pooling over objgan_oracle's
words_loss / sent_loss); and dump_fid_acts against INCEPTION_V3_FID.activations.  (File name sorts last: every test
builds all the networks of the evaluation.)"""
import os
import pickle

import numpy as np
import pytest
import torch

import inception_oracle as I
import oracle_eval
from objgan_b200 import evaluator, losses, model, ops, synth
from objgan_b200.config import cfg
from oracle import image_encoder_oracle as E
from oracle import objgan_oracle as O
from oracle import shape_oracle as S
from oracle import text_oracle as T
from test_eval_mode import eval_fixture, eval_state_dict
from test_shape_gen import shp_sd

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_WORDS = 150
B, BATCHES, POOL, DIMS = 4, 5, 8, 64


# ---------------------------------------------------------------------------------------------------------------------
# og_images_to_u8
# ---------------------------------------------------------------------------------------------------------------------
def _torch_u8(x):
    return x.add(1).div(2).mul(255).clamp(0, 255).byte().permute(0, 2, 3, 1).contiguous()


def test_images_to_u8_bitwise():
    g = torch.Generator().manual_seed(3)
    k = torch.arange(256, dtype=torch.float32)
    edge = (2 * k / 255 - 1).float()                                  # the byte boundaries (2k/255) - 1
    up = torch.nextafter(edge, torch.tensor(float("inf")))
    down = torch.nextafter(edge, torch.tensor(-float("inf")))
    special = torch.tensor([1.0, -1.0, float("inf"), -float("inf"), 0.0, -0.0])
    vals = torch.cat([edge, up, down, special, torch.rand(2 * 3 * 64 * 64, generator=g) * 2.4 - 1.2])
    n = 3 * 32 * 32
    vals = torch.cat([vals, torch.zeros((-vals.numel()) % n)])
    x = vals.view(-1, 3, 32, 32).to(DEV)
    got = ops.images_to_u8(x)
    want = _torch_u8(x)
    assert got.dtype == torch.uint8 and got.shape == want.shape
    assert torch.equal(got, want)
    # non-square, odd sizes, the 256-pixel images of the evaluator
    for shape in ((3, 3, 7, 5), (2, 3, 256, 256)):
        x = (torch.rand(shape, generator=g) * 2.4 - 1.2).to(DEV)
        assert torch.equal(ops.images_to_u8(x), _torch_u8(x))
    nan = torch.full((1, 3, 4, 4), float("nan"), device=DEV)
    assert (ops.images_to_u8(nan) == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# evaluate against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """netG (eval-mode fixture weights), the shape generator, the DAMSM encoders and the Inception weights."""
    d = tmp_path_factory.mktemp("pretrained")
    g_sd = eval_state_dict(eval_fixture(3))
    torch.save(g_sd, d / "netG_epoch_120.pth")
    s_sd = shp_sd()
    torch.save({"module." + k: v for k, v in s_sd.items()}, d / "shape_gen.pth")
    torch.manual_seed(0)
    text_sd = model.RNN_ENCODER(N_WORDS, nhidden=256).state_dict()
    torch.save(text_sd, d / "text_encoder100.pth")
    img_sd = E.test_state_dict(model.CNN_ENCODER(256).state_dict(), seed=0)
    torch.save(img_sd, d / "image_encoder100.pth")
    inc = I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0)
    return dict(dir=d, g=g_sd, shp=s_sd, text=text_sd, img=img_sd, inc=inc)


def _cfg(monkeypatch, files, mode):
    d = files["dir"]
    for k, v in dict(BATCH_SIZE=B, DISPLAY_INTERVAL=1000, NET_E=str(d / "text_encoder100.pth"),
                     NET_G=str(d / "netG_epoch_120.pth")).items():
        monkeypatch.setitem(cfg.TRAIN, k, v)
    for k, v in dict(USE_GT_BOX_SEG=mode, NET_SHP_G=str(d / "shape_gen.pth"), RP_POOL_SIZE=POOL, FID_DIMS=DIMS,
                     TEST_IMG_NUM=1000000, SAVE_OPTIONS="IMAGE", USE_TF=0).items():
        monkeypatch.setitem(cfg.TEST, k, v)


def _batch(mode, i):
    return synth.reference_test_batch(B, seed=700 + 10 * mode + i, mode=mode, n_words=N_WORDS, fid_dims=DIMS)


def _noise(i):
    g = torch.Generator().manual_seed(900 + i)
    return (torch.randn(B, cfg.GAN.Z_DIM, generator=g), torch.randn(B, cfg.GAN.CONDITION_DIM, generator=g),
            torch.randn(B, cfg.ROI.BOXES_NUM, 4 * 80, generator=g))


def _oracle_batch(files, ds, data, mode, noise):
    """The reference's evaluate() body for one batch on the CPU: prepare_data / prepare_gen_data (the loader's box
    maps sliced to max_num_roi), shapes, text stage, G_NET, then the image encoder and both Inception trunks."""
    if mode == 2:
        _, acts, caps, gcaps, lens, fwd, bwd, fmaps, rois, fm_rois, num_rois, class_ids, _, _ = data
    else:
        _, acts, caps, gcaps, lens, hmaps, fwd, bwd, fmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks, \
            class_ids, _, _ = data
    z, eps, noise_shp = noise
    order = torch.sort(lens, dim=0, descending=True, stable=True).indices
    lens, nr = lens[order], num_rois[order]
    caps, gcaps = caps[order].view(B, -1), gcaps[order].view(B, -1)
    rois = [r[order] for r in rois]
    rmax = int(nr.max())
    cls = rois[0][..., 4].long()
    if mode > 0:
        raw = S.shp_g_net_forward(files["shp"], noise_shp[:, :rmax], fwd[order, :rmax].float(),
                                  bwd[order, :rmax].float(), fmaps[order, :rmax].float())
        hm, bt, fmb = S.form_hmaps(raw[:, :, 0], nr, cls)
    else:
        hm = [h[order].float() for h in hmaps]
        bt, fmb = [m[order].float() for m in bt_masks], fm_bt_masks[order].float()
    max_len = int(lens.max())
    words, sent = T.rnn_encoder_forward(files["text"], caps, lens, max_len)
    glove = ds.glove_embed.weight.detach().float()
    glove_words, mask = T.text_inputs(caps, gcaps, glove, max_len)
    clabels = T.prepare_cat_emb(glove, ds.cat_labels, ds.cat_label_lens, ds.sorted_cat_label_indices)
    sl = torch.zeros(B, rmax, clabels.shape[1])
    for i in range(B):
        sl[i, :int(nr[i])] = clabels[cls[i, :int(nr[i])]]
    inp = dict(z=z, eps=eps, sent_emb=sent, words_embs=words, glove_words_embs=glove_words,
               slabels_feat=sl.transpose(1, 2).unsqueeze(3).contiguous(), mask=mask, hmaps=hm, rois=rois,
               fm_rois=fm_rois[order], num_rois=nr, bt_masks=bt, fm_bt_masks=fmb, glb_max_num_roi=rmax)
    fake = oracle_eval.g_net_forward_eval(files["g"], inp)[0][-1]
    region, code = E.cnn_encoder_forward(files["img"], fake)
    return dict(region=region, code=code, words=words, sent=sent, lens=lens, class_ids=class_ids[order].numpy(),
                pred=I.inception_v3_forward(files["inc"], fake), acts=I.fid_activations(files["inc"], fake, DIMS),
                real=acts[order])


_ORACLE = {}


def _oracle(files, ds, mode):
    """Per-batch oracle outputs of the mode (computed once: the oracle does not depend on the engine)."""
    if mode not in _ORACLE:
        with torch.no_grad():
            _ORACLE[mode] = [_oracle_batch(files, ds, _batch(mode, i), mode, _noise(i)) for i in range(BATCHES)]
    return _ORACLE[mode]


def _oracle_rp(batches):
    """The reference's pooling (evaluator.py:379-419): batches 1-2 fill the pool of 8, batch 3 scores it and is dropped,
    batches 4-5 fill a pool that is never scored.  Returns (word accuracy, sentence accuracy, smallest margin)."""
    pool = batches[:2]
    cat = lambda k: torch.cat([b[k] for b in pool], 0)
    lens = cat("lens")
    ml = int(lens.max())
    words = torch.zeros(POOL, 256, ml)
    acc = 0
    for b in pool:
        words[acc:acc + B, :, :b["words"].shape[2]] = b["words"]
        acc += B
    ids = np.concatenate([b["class_ids"] for b in pool])
    margins = []
    real = O._two_ce

    def record(scores0, labels, bs):
        for s in (scores0, scores0.t()):
            top = s.topk(2, dim=1).values
            margins.append(float((top[:, 0] - top[:, 1]).min()))
        return real(scores0, labels, bs)
    O._two_ce = record
    try:
        labels = torch.arange(POOL)
        w = O.words_loss(cat("region"), words, labels, lens, ids, POOL)[3]
        s = O.sent_loss(cat("code"), cat("sent"), labels, ids, POOL)[2]
    finally:
        O._two_ce = real
    return w, s, min(margins)


def _frob(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("engine", ["simt", "f16x3"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_evaluate_vs_oracle(mode, engine, files, tmp_path, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    _cfg(monkeypatch, files, mode)
    ds = synth.reference_test_dataset(n_words=N_WORDS)
    want = _oracle(files, ds, mode)
    e = evaluator.condGANEvaluator(str(tmp_path), [None] * BATCHES, ds, inception_weights=files["inc"], device=DEV)
    e.build_models()
    rp, is_, fid = losses.RPrecision(POOL), losses.InceptionScore(min(10, B)), losses.FrechetDistance(DIMS)
    scored = []
    for i in range(BATCHES):
        z, eps, noise_shp = (t.to(DEV) for t in _noise(i))
        out = e.evaluate_batch(_batch(mode, i), rp, is_, fid, z=z, eps=eps, noise_shp=noise_shp, gen_iterations=i + 1)
        assert (out["class_ids"] == want[i]["class_ids"]).all()
        scored.append(len(rp.w_accuracy))
    assert scored == [0, 0, 1, 1, 1]                       # batch 3 scores pool 1; pool 2 (batches 4-5) never scored
    res = e.finish(rp, is_, fid)
    # Inception score and confidence
    p = torch.cat([b["pred"] for b in want]).numpy()
    ws = (*losses.inception_score(p, min(10, B)), *losses.negative_log_posterior(p, min(10, B)))
    for a, b in zip(res["scores"][:4], ws):
        assert abs(a - b) <= 1e-4 * abs(b), (res["scores"][:4], ws)
    # FID statistics: the real ones exact up to the fp64 summation order; the generated mean within 1e-5 and their
    # covariance within 3e-5, twice the largest error measured (DESIGN §3.11).  The oracle computes the activations in
    # fp32, and these 20 rows spread by about 1/30 of their mean, so a covariance amplifies the activations' rounding by
    # that factor: mode 0 measures 1.48e-5 on both engines alike, the oracle's own share
    (rmu, rsig), (fmu, fsig) = fid.statistics()
    real = torch.cat([b["real"] for b in want]).numpy()
    fake = torch.cat([b["acts"] for b in want]).double().numpy()
    assert _frob(rmu, real.mean(0)) <= 1e-12 and _frob(rsig, np.cov(real, rowvar=False)) <= 1e-12
    err_mu, err_sigma = _frob(fmu, fake.mean(0)), _frob(fsig, np.cov(fake, rowvar=False))
    print(f"mode {mode} {engine}: generated FID mean {err_mu:.2e}, covariance {err_sigma:.2e}")
    assert err_mu <= 1e-5 and err_sigma <= 3e-5, (err_mu, err_sigma)
    # R-precision: equal decisions, with no near-tie in the oracle
    w_acc, s_acc, margin = _oracle_rp(want)
    assert margin > 1e-4, margin
    assert res["w_accuracy"] == [w_acc] and res["s_accuracy"] == [s_acc]
    lines = (tmp_path / "Score" / "scores.txt").read_text().split("\n")
    assert lines[0] == evaluator.SCORE_HEADER.rstrip("\n") and len(lines[1].split(", ")) == 9
    print(f"mode {mode} {engine}: scores {res['scores']}")


# ---------------------------------------------------------------------------------------------------------------------
# dump_fid_acts
# ---------------------------------------------------------------------------------------------------------------------
def test_dump_fid_acts_bitwise(files, tmp_path, monkeypatch):
    _cfg(monkeypatch, files, 2)
    loader = synth.reference_acts_batches(B, 2, seed=71)
    e = evaluator.condGANEvaluator(str(tmp_path / "out"), loader, synth.reference_test_dataset(n_words=N_WORDS),
                                   inception_weights=files["inc"], device=DEV)
    e.dump_fid_acts(str(tmp_path), "test")
    with open(tmp_path / "test_acts_tf0.pickle", "rb") as f:
        got = pickle.load(f)[0]
    net = model.INCEPTION_V3_FID.from_imagenet(files["inc"], DEV, [model.INCEPTION_V3_FID.BLOCK_INDEX_BY_DIM[DIMS]])
    for imgs, keys in loader:
        with torch.no_grad():
            want = net.activations(imgs[-1].to(DEV)).cpu().numpy()
        for i, k in enumerate(keys):
            assert got[k].dtype == np.float64 and got[k].shape == (DIMS,)
            assert np.array_equal(got[k], want[i].astype(np.float64)), k
    assert evaluator.load_acts_data(str(tmp_path), "test").keys() == got.keys()
