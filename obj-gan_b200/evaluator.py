"""The reference's evaluation loop (ref: image_generation/evaluator.py:30-467, ``condGANEvaluator``, fed by
testDataset.py) on this library: the same constructor, ``dump_fid_acts`` and ``evaluate``, fed by the reference's own
test DataLoader, writing the nine numbers of ``Score/scores.txt``: the Inception score and confidence, the word and
sentence R-precision, and FID.

Each batch runs the host intake (``trainer.prepare_reference_test_batch``), the eager sampler (text encoder, then for
cfg.TEST.USE_GT_BOX_SEG = 1 / 2 the box maps, SHP_G_NET and the generated heat maps, or for 0 the ground-truth heat
maps; then G_NET), the DAMSM image encoder into ``losses.RPrecision``, and both Inception trunks into
``losses.InceptionScore`` and ``losses.FrechetDistance``.  Predictions, activation moments and pooled R-precision
inputs stay on the device; the only per-batch reads are the sampler's caption checks, the scores of a completed
R-precision pool and, on display batches, the image bytes.

Under torchrun (one process per GPU, each with its own shard of the test split) every rank samples and scores its own
batches; at the end the predictions are gathered to rank 0 once, the FID moments are merged there
(``_Moments.merge``), and the per-pool R-precision accuracies of every rank are pooled.  Each rank fills its own
R-precision pools, so the pools hold different images than a single-process run's: the mean over pools estimates the
same quantity, but is not the same number.  Only rank 0 prints and writes files.

On display batches rank 0 writes the reference's snapshot PNGs to ``Snapshot/`` when a caption font is available
(``font=``, or the reference's cfg.DATA_DIR + '/share/Pillow/Tests/fonts/FreeMono.ttf'): with SAVE_OPTIONS =
'SNAPSHOT' the attention maps of each stage (``G_<it>_<i>.png``, ``bt_G_<it>_<i>.png``), and in modes 1 and 2 the
generated shapes (``ShapeG_<it>.png``) and, in mode 1, the ground-truth heat maps (``ShapeD_<it>.png``), composed on
the device (snapshots.py).  The reference's SNAPSHOT call cannot run (it passes parameters build_super_images does
not have); this is what it evidently means: build_super_images per stage with the batch's images and font 50.  The
TensorFlow Inception path (cfg.TEST.USE_TF = 1) is refused."""
from __future__ import annotations

import os
import pickle
import warnings

import numpy as np
import torch
import torch.distributed as dist

from . import losses, model, ops, snapshots
from .config import cfg
from .sampler import GSampler
from .trainer import gather_inception_score, prepare_reference_test_batch

SCORE_HEADER = "mean, std, mean_conf, std_conf, accu_w, std_w, accu_s, std_s, fid_score \n"


def acts_path(data_dir, split):
    """``<data_dir>/<split>_acts_tf0.pickle``: the real images' FID activations (ref: evaluator.py:242, load.py:466)."""
    return os.path.join(data_dir, "%s_acts_tf%d.pickle" % (split, cfg.TEST.USE_TF))


def load_acts_data(data_dir, split):
    """The activations dict that ``dump_fid_acts`` writes (ref: miscc/load.py:465-477), or None without the file."""
    path = acts_path(data_dir, split)
    if not os.path.isfile(path):
        return None
    with open(path, "rb") as f:
        return pickle.load(f)[0]


def _refuse_unsupported():
    if cfg.TEST.USE_TF:
        raise ValueError("cfg.TEST.USE_TF = 1 selects the reference's TensorFlow Inception models, which this library "
                         "does not implement: set cfg.TEST.USE_TF = 0 to score with INCEPTION_V3 / INCEPTION_V3_FID")
    if cfg.TEST.SAVE_OPTIONS not in ("IMAGE", "SNAPSHOT"):
        raise ValueError(f"cfg.TEST.SAVE_OPTIONS must be 'IMAGE' or 'SNAPSHOT', got {cfg.TEST.SAVE_OPTIONS!r}")
    if cfg.TEST.USE_GT_BOX_SEG not in (0, 1, 2):
        raise ValueError(f"cfg.TEST.USE_GT_BOX_SEG must be 0, 1 or 2, got {cfg.TEST.USE_GT_BOX_SEG}")


class condGANEvaluator:
    """Drop-in for the reference's ``condGANEvaluator(output_dir, data_loader, dataset)``.

    ``dataset`` provides what the reference reads from it: ``n_words``, ``cats_index_dict``, ``cat_labels``,
    ``cat_label_lens``, ``sorted_cat_label_indices`` and ``glove_embed``.  ``inception_weights``: torchvision's ImageNet
    file (``inception_v3_google-1a9a5a14.pth``, its path or its loaded state_dict) for both Inception trunks; this
    library reads no network.  The generator is cfg.TRAIN.NET_G, the DAMSM encoders cfg.TRAIN.NET_E (the image
    encoder's path with ``text_encoder`` -> ``image_encoder``), the shape generator cfg.TEST.NET_SHP_G when
    cfg.TEST.USE_GT_BOX_SEG > 0."""

    def __init__(self, output_dir, data_loader, dataset, *, inception_weights, device=None, process_group=None,
                 font=None):
        _refuse_unsupported()
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.model_dir = os.path.join(output_dir, "Model")
        self.image_dir = os.path.join(output_dir, "Image")
        self.snapshot_dir = os.path.join(output_dir, "Snapshot")
        self.score_dir = os.path.join(output_dir, "Score")
        if self.rank == 0:
            for d in (self.model_dir, self.image_dir, self.snapshot_dir, self.score_dir):
                os.makedirs(d, exist_ok=True)
        self.batch_size = cfg.TRAIN.BATCH_SIZE
        self.display_interval = cfg.TRAIN.DISPLAY_INTERVAL
        self.n_words = dataset.n_words
        self.cats_index_dict = dataset.cats_index_dict
        self.cat_labels = dataset.cat_labels
        self.cat_label_lens = dataset.cat_label_lens
        self.sorted_cat_label_indices = dataset.sorted_cat_label_indices
        self.glove_emb = dataset.glove_embed
        self.data_loader = data_loader
        self.num_batches = len(data_loader)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.inception_weights = inception_weights
        self.mode = cfg.TEST.USE_GT_BOX_SEG
        self.sampler = None
        self._warned_snapshot = False
        self.ixtoword = getattr(dataset, "ixtoword", None)
        self.font = snapshots.load_font(font) if self.rank == 0 else None
        self._writer = None

    def build_models(self) -> GSampler:
        """The sampler with every network of the evaluation (ref: evaluator.py:74-86, 88-146): G_NET from
        cfg.TRAIN.NET_G, SHP_G_NET from cfg.TEST.NET_SHP_G (modes 1 / 2), RNN_ENCODER and CNN_ENCODER from
        cfg.TRAIN.NET_E, the label embeddings from the GloVe table, and both Inception trunks (FID at
        cfg.TEST.FID_DIMS)."""
        if not cfg.TRAIN.NET_E:
            raise ValueError("no pretrained text-image encoders: set cfg.TRAIN.NET_E")
        if not cfg.TRAIN.NET_G:
            raise ValueError("no generator snapshot to evaluate: set cfg.TRAIN.NET_G")
        as_i64 = lambda t: torch.as_tensor(t).to(torch.int64)
        self.sampler = GSampler.from_snapshot(
            cfg.TRAIN.NET_G, num_classes=len(self.cats_index_dict), device=self.device,
            shape_snapshot=cfg.TEST.NET_SHP_G if self.mode > 0 else None, text_snapshot=cfg.TRAIN.NET_E,
            glove=self.glove_emb, cat_labels=as_i64(self.cat_labels), cat_label_lens=as_i64(self.cat_label_lens),
            cat_label_order=as_i64(self.sorted_cat_label_indices),
            image_snapshot=cfg.TRAIN.NET_E.replace("text_encoder", "image_encoder"),
            inception_weights=self.inception_weights, fid_dims=cfg.TEST.FID_DIMS)
        return self.sampler

    # ------------------------------------------------------------------ real activations
    def dump_fid_acts(self, data_dir, split):
        """ref: evaluator.py:241-266.  Unless ``<data_dir>/<split>_acts_tf0.pickle`` exists, runs
        INCEPTION_V3_FID.activations over ``imgs[-1]`` of every (imgs, keys) batch of the loader and writes
        ``[{key: float64 (dims,) array}]`` with pickle protocol 2, the file the reference's load_acts_data reads.

        Under torchrun every rank computes the activations of its own shard; rank 0 gathers them and writes the file
        (under a temporary name, renamed when complete), and no rank returns before the file is there, so every rank
        can read it back with ``load_acts_data`` right after.  Whether the file exists is rank 0's decision, so all
        ranks take the same branch."""
        path = acts_path(data_dir, split)
        exists = [os.path.isfile(path)]
        if self.world > 1:
            dist.broadcast_object_list(exists, src=0, group=self.pg)
        if exists[0]:
            return
        fid_net = model.INCEPTION_V3_FID.from_imagenet(
            self.inception_weights, self.device, [model.INCEPTION_V3_FID.BLOCK_INDEX_BY_DIM[cfg.TEST.FID_DIMS]])
        acts_dict = {}
        for count, (imgs, keys) in enumerate(self.data_loader):
            if count % 10 == 0 and self.rank == 0:
                print("%07d / %07d" % (count, self.num_batches))
            with torch.no_grad():
                acts = fid_net.activations(torch.as_tensor(imgs[-1]).to(self.device, torch.float32))
            acts = acts.cpu().numpy().astype(np.float64)         # get_activations' np.empty is float64
            for i, key in enumerate(keys):
                acts_dict[key] = acts[i]
        if self.world > 1:                                       # every rank's shard, written by rank 0
            got = [None] * self.world if self.rank == 0 else None
            dist.gather_object(acts_dict, got, dst=0, group=self.pg)
            if self.rank == 0:
                acts_dict = {k: v for d in got for k, v in d.items()}
        if self.rank == 0:
            tmp = path + ".tmp"
            with open(tmp, "wb") as f:
                pickle.dump([acts_dict], f, protocol=2)
            os.replace(tmp, path)                                # never a half-written file under the final name
            print("Save to: ", path)
        if self.world > 1:
            dist.barrier(group=self.pg)                          # the file is complete before any rank goes on

    # ------------------------------------------------------------------ the loop
    def evaluate_batch(self, data, rp, is_, fid, z=None, eps=None, noise_shp=None, gen_iterations=None) -> dict:
        """One batch of the loop body (ref: evaluator.py:293-436): intake, eager sampling (``z``, the CA_NET ``eps``
        and the shape noise ``noise_shp`` taken when given), the image encoder into ``rp`` (losses.RPrecision), the
        Inception predictions into ``is_`` (losses.InceptionScore) and the generated and real activations into
        ``fid`` (losses.FrechetDistance).  On a display batch (``gen_iterations`` a multiple of DISPLAY_INTERVAL) with
        SAVE_OPTIONS 'IMAGE', rank 0 writes ``Image/<key>_<sent_id>.jpg``.  Returns the fake images and the sorted
        ``class_ids``, ``keys`` and ``sent_ids``."""
        batch, acts, class_ids, keys, sent_ids = prepare_reference_test_batch(data, self.mode)
        s = self.sampler
        inp = dict(batch)
        for k, v in (("z", z), ("eps", eps), ("noise_shp", noise_shp)):
            if v is not None:
                inp[k] = v
        text = {}
        display = gen_iterations is not None and gen_iterations % self.display_interval == 0
        snap = display and self.font is not None
        shapes = {} if snap and self.mode > 0 else None
        with torch.no_grad():
            kw = {} if shapes is None else {"shapes_out": shapes}
            sampled = s.sample_eager(inp, text_out=text, **kw)
            fake_imgs = sampled[0]
            region_features, cnn_code = s.encode_image(fake_imgs)
            rp.add(region_features, cnn_code, text["words_embs"], text["sent_emb"],
                   batch["cap_lens"].to(self.device, non_blocking=True), class_ids)
            pred, fake_acts = s.score_images(fake_imgs)
            is_.add(pred)
            fid.add(fake_acts, acts.to(self.device, non_blocking=True))
        if display:
            if cfg.TEST.SAVE_OPTIONS == "IMAGE":
                self.save_singleimages(fake_imgs[-1], keys, sent_ids)
            elif snap:
                self.save_img_results(fake_imgs, sampled[2], sampled[3], batch["captions"], gen_iterations)
            elif not self._warned_snapshot:
                warnings.warn("cfg.TEST.SAVE_OPTIONS = 'SNAPSHOT': the attention-map PNGs (save_img_results) are not "
                              "produced by this library")
                self._warned_snapshot = True
            if shapes:
                self.save_shape_results(data, batch, shapes["raw_masks"], gen_iterations)
            if self.rank == 0:
                print("%d / %d" % (gen_iterations, self.num_batches))
        return dict(fake_imgs=fake_imgs, class_ids=class_ids, keys=keys, sent_ids=sent_ids)

    def _submit(self, jobs):
        if self._writer is None:
            self._writer = snapshots.PngWriter()
        self._writer.submit(jobs)

    def save_img_results(self, fake_imgs, att_maps, bt_att_maps, captions, gen_iterations):
        """ref: evaluator.py:170-205, as it evidently means: per stage i, build_super_images of fake_imgs[i + 1]
        (lr fake_imgs[i]) with the stage's word and box-word attention maps: ``Snapshot/G_<it>_<i>.png`` and
        ``Snapshot/bt_G_<it>_<i>.png``."""
        if self.rank != 0:
            return
        jobs = []
        for i in range(len(att_maps)):
            for prefix, maps in (("G", att_maps[i]), ("bt_G", bt_att_maps[i])):
                c = snapshots.super_images(fake_imgs[i + 1], captions, self.ixtoword, maps, lr_images=fake_imgs[i],
                                           font=self.font)
                jobs.append((os.path.join(self.snapshot_dir, "%s_%d_%d.png" % (prefix, gen_iterations, i)), c))
        self._submit(jobs)

    def save_shape_results(self, data, batch, raw_masks, gen_iterations):
        """ref: evaluator.py:207-229 and 316-324: ``Snapshot/ShapeG_<it>.png`` from the real 64-pixel images and the
        shape generator's masks and, in mode 1, ``Snapshot/ShapeD_<it>.png`` from the ground-truth heat maps of the
        64 scale, rebuilt on the device from the loader's masks.  The loader's images and masks are read on display
        batches only, in the batch's caption-length order."""
        if self.rank != 0:
            return
        order = torch.sort(torch.as_tensor(data[4]).to(torch.int64).view(-1), dim=0, descending=True,
                           stable=True).indices
        to_dev = lambda t: torch.as_tensor(t)[order].to(self.device, torch.float32)
        imgs0 = to_dev(data[0][0])
        jobs = [(os.path.join(self.snapshot_dir, "ShapeG_%d.png" % gen_iterations),
                 snapshots.super_shape_images(imgs0, raw_masks))]
        if self.mode == 1:
            cls = batch["roi_cls"].to(self.device)
            nr = batch["num_rois"].to(self.device)
            hmaps = ops.form_hmaps(to_dev(data[12][0]).contiguous(), cls, nr, len(self.cats_index_dict), 0.0)
            jobs.append((os.path.join(self.snapshot_dir, "ShapeD_%d.png" % gen_iterations),
                         snapshots.super_shape_images(imgs0, hmaps)))
        self._submit(jobs)

    def save_singleimages(self, images, keys, sent_ids):
        """ref: evaluator.py:231-239: one JPEG per image, the bytes made on the device (ops.images_to_u8)."""
        if self.rank != 0:
            return
        from PIL import Image
        arr = ops.images_to_u8(images).cpu().numpy()
        for i in range(arr.shape[0]):
            Image.fromarray(arr[i]).save("%s/%s_%d.jpg" % (self.image_dir, keys[i], sent_ids[i]))

    def _merged_fid(self, fid):
        """FID statistics over every rank: one gather of (n, k, s1, s2) per moment set, merged on rank 0 (None on
        the others)."""
        if self.world == 1:
            return fid.real, fid.fake
        d = fid.dims
        out = []
        for m in (fid.real, fid.fake):
            buf = torch.zeros(1 + 2 * d + d * d, dtype=torch.float64, device=self.device)
            if m.n > 0:
                buf[0] = m.n
                buf[1:1 + d], buf[1 + d:1 + 2 * d] = m.k, m.s1
                buf[1 + 2 * d:] = m.s2.reshape(-1)
            parts = [torch.empty_like(buf) for _ in range(self.world)]
            dist.all_gather(parts, buf, group=self.pg)
            ms = [losses._Moments.from_sums(int(p[0]), p[1:1 + d], p[1 + d:1 + 2 * d], p[1 + 2 * d:].view(d, d))
                  for p in parts]
            out.append(ms[0].merge(ms[1:]))
        return tuple(out) if self.rank == 0 else None

    def _merged_rp(self, rp):
        """Every rank's per-pool accuracies, rank 0's first (None on the other ranks)."""
        if self.world == 1:
            return rp.w_accuracy, rp.s_accuracy
        got = [None] * self.world
        dist.all_gather_object(got, (rp.w_accuracy, rp.s_accuracy), group=self.pg)
        if self.rank != 0:
            return None
        return [a for w, _ in got for a in w], [a for _, s in got for a in s]

    def evaluate(self, split_dir, hmap_size):
        """ref: evaluator.py:268-467.  Runs the loop over the loader (at most cfg.TEST.TEST_IMG_NUM batches, the
        reference's unit), then writes ``Score/scores.txt`` in the reference's format and prints its two lines.
        ``split_dir`` and ``hmap_size`` are accepted for the reference's signature; the heat-map sizes are the
        generator's.  Returns, on rank 0, a dict with the nine ``scores`` and the per-pool ``w_accuracy`` /
        ``s_accuracy``; None on the other ranks."""
        if self.sampler is None:
            self.build_models()
        num_splits = min(10, self.batch_size)
        rp = losses.RPrecision(cfg.TEST.RP_POOL_SIZE)
        is_ = losses.InceptionScore(num_splits)
        fid = losses.FrechetDistance(cfg.TEST.FID_DIMS)
        gen_iterations = 0
        try:
            for data in self.data_loader:
                self.evaluate_batch(data, rp, is_, fid, gen_iterations=gen_iterations)
                gen_iterations += 1
                if gen_iterations >= cfg.TEST.TEST_IMG_NUM:
                    break
        except BaseException:
            self.close_writer(raise_error=False)
            raise
        return self.finish(rp, is_, fid)

    def close_writer(self, raise_error=True):
        """Waits until every snapshot PNG of the batches so far is written (``finish`` calls it)."""
        if self._writer is not None:
            writer, self._writer = self._writer, None
            writer.close(raise_error)

    def finish(self, rp, is_, fid):
        """The scores over every rank (ref: evaluator.py:443-467), written and printed by rank 0, after the snapshot
        PNGs of ``evaluate_batch`` are written."""
        self.close_writer()
        score = gather_inception_score(is_, self.world, self.rank, self.pg)
        moments = self._merged_fid(fid)
        accs = self._merged_rp(rp)
        if self.rank != 0:
            return None
        with np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)          # no scored pool: nan, as in the reference
            mean, std, mean_conf, std_conf = score.result()
            w, s = np.asarray(accs[0], dtype=np.float64), np.asarray(accs[1], dtype=np.float64)
            accu_w, std_w, accu_s, std_s = np.mean(w), np.std(w), np.mean(s), np.std(s)
        (mu1, sigma1), (mu2, sigma2) = moments[0].statistics(), moments[1].statistics()
        fid_score = float(losses.frechet_distance(mu1, sigma1, mu2, sigma2))
        vals = (mean, std, mean_conf, std_conf, accu_w, std_w, accu_s, std_s, fid_score)
        line = "%f, %f, %f, %f, %f, %f, %f, %f, %f" % vals
        with open(os.path.join(self.score_dir, "scores.txt"), "w") as fp:
            fp.write(SCORE_HEADER)
            fp.write(line)
        print("inception_score: mean, std, mean_conf, std_conf, accu_w, std_w, accu_s, std_s, fid_score")
        print("inception_score: " + line)
        return dict(scores=vals, w_accuracy=list(accs[0]), s_accuracy=list(accs[1]))
