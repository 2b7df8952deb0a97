"""Sampling from a trained generator: the reference's evaluator path (ref: evaluator.py:108-138 builds G_NET, calls
``netG.eval()`` and loads ``netG_epoch_N.pth``; evaluator.py:312 draws the noise) on the sm_90a kernels.

With a shape generator (``SHP_G_NET``, ref: evaluator.py:111-144), a batch that brings boxes but no masks is sampled the
way the reference's default evaluator mode does it (cfg.TEST.USE_GT_BOX_SEG = 1 / 2, evaluator.py:314-332): box maps ->
SHP_G_NET -> form_hmaps -> label embeddings -> G_NET, all on the device and inside the same per-shape CUDA graph.

With a text encoder (``RNN_ENCODER``) and the GloVe table (ref: evaluator.py:90-95, 337-351), a batch that brings
``captions``, ``cap_lens`` and ``glove_captions`` instead of ``words_embs`` is encoded on the device inside the same
graph: token ids -> text encoder + GloVe lookups + padding mask -> (shape generator) -> G_NET.

With a box generator (``BoxGenerator``: PreEncoderRNN + DecoderRNN, ref: box_generation/sample.py, Evaluator.evaluate
and load_gen_insanns), a caption batch that brings no ``rois`` gets its layout on the device first: box captions ->
encoder state -> og_box_decode -> og_box_layout.  The roi count decides the shape of the image graph (Rmax, below), so
the box stage is a CUDA graph of its own, keyed by (B, box caption length); one device -> host read of ``num_rois``
follows it, and then the text + generated-shape graph runs.

``GSampler`` holds its own G_NET in eval mode, so BatchNorm normalises with the running statistics and never updates
them.  A forward pass is ~200 library calls, which cost far more host time than the kernels take at small batch, so
every input shape is captured once into a CUDA graph and replayed after that:

  * graphs are keyed by (B, L, Rmax, glb_max_num_roi, text, generated shapes): batch, caption length (max(cap_lens)
    for a caption batch), roi slots of ``slabels_feat`` (glb_max_num_roi when the shapes are generated), the roi
    width of the returned ``bt_c_code``, whether the word embeddings come from the batch or from the text encoder,
    and whether the masks come from the batch or from the shape generator.  Rmax is NOT padded to BOXES_NUM to share one graph: the bottom-up paint
    takes a max over the roi axis, and an extra zero slot contributes 0 to that max, which changes the result wherever
    every real roi's product is negative;
  * the first call with a key runs eagerly (the warm-up: packed weight copies, allocator), then captures; later calls
    copy their inputs into the captured static buffers and replay;
  * all graphs share one memory pool, and outputs are cloned out of it, so no two calls alias;
  * a graph records the addresses of the packed fp16 weight copies, so each graph keeps the copies it recorded alive,
    and ``load_state_dict`` (the only way the sampler's weights change) drops every graph.
"""
from __future__ import annotations

import torch

from . import lib as _lib
from . import model, ops
from .config import cfg
from .synth import IMG_SIZES
from .trainer import prepare_data, text_stage

NOISE_BOX = ops.BOX_NOISE

# what G_NET.forward reads, in its argument order (ref: model.py:747)
G_ARGS = ("z", "sent_emb", "words_embs", "glove_words_embs", "slabels_feat", "mask", "hmaps", "rois", "fm_rois",
          "num_rois", "bt_masks", "fm_bt_masks", "glb_max_num_roi")
# what the generated-shape path reads: the layout (boxes and classes), the shape noise, and the label embeddings
GEN_ARGS = ("z", "eps", "noise_shp", "sent_emb", "words_embs", "glove_words_embs", "mask", "rois", "fm_rois", "num_rois",
            "roi_cls", "clabels_emb", "glb_max_num_roi")
# what the text encoder stage computes, and what it reads instead (ref: evaluator.py:337-351)
TEXT_OUT = ("sent_emb", "words_embs", "glove_words_embs", "mask")
TEXT_ARGS = ("captions", "cap_lens", "glove_captions", "max_len")


def _map(x, f):
    if torch.is_tensor(x):
        return f(x)
    if isinstance(x, (list, tuple)):
        return [f(t) for t in x]
    return x


def _copy_into(dst, src):
    if torch.is_tensor(dst):
        dst.copy_(src, non_blocking=True)
    elif isinstance(dst, list):
        for d, s in zip(dst, src):
            d.copy_(s, non_blocking=True)


class _Graph:
    """One captured forward: its static inputs / outputs, its library-call count, and the packed weight copies it
    read (kept alive with it)."""

    def __init__(self, graph, static_in, static_out, launches, keep):
        self.graph, self.static_in, self.static_out = graph, static_in, static_out
        self.launches, self.keep = launches, keep


class GSampler:
    """Eval-mode G_NET forward with the reference's inputs and 6-tuple output, CUDA-graph replayed per input shape."""

    def __init__(self, netG: model.G_NET, netShpG: model.SHP_G_NET | None = None,
                 text_encoder: model.RNN_ENCODER | None = None, glove=None, clabels_emb=None, box_generator=None,
                 image_encoder: model.CNN_ENCODER | None = None, inception: model.INCEPTION_V3 | None = None,
                 inception_fid: model.INCEPTION_V3_FID | None = None):
        """``glove``: the GloVe table (V, 50) as a tensor or an nn.Embedding (the reference's ``glove_emb``);
        ``clabels_emb``: (num_classes, 50) label embeddings (see ops.class_label_emb) used when a batch has none;
        ``box_generator``: a boxgen.BoxGenerator that makes the layout of caption batches without ``rois``;
        ``image_encoder``: the DAMSM CNN_ENCODER that ``encode_image`` runs (R-precision, losses.RPrecision);
        ``inception`` / ``inception_fid``: the scoring networks that ``score_images`` runs (losses.InceptionScore,
        losses.FrechetDistance)."""
        self.netG = netG.eval()
        self.netShpG = netShpG.eval() if netShpG is not None else None
        self.text_encoder = text_encoder.eval() if text_encoder is not None else None
        for net in (self.netG, self.netShpG, self.text_encoder):
            for p in (net.parameters() if net is not None else ()):
                p.requires_grad_(False)
        self.device = next(self.netG.parameters()).device
        glove = getattr(glove, "weight", glove)
        self.glove = glove.detach().to(self.device).float().contiguous() if glove is not None else None
        self.clabels_emb = clabels_emb.detach().to(self.device).float().contiguous() if clabels_emb is not None else None
        self.box_generator = box_generator.to(self.device) if box_generator is not None else None
        self.image_encoder = image_encoder.to(self.device).eval().requires_grad_(False) if image_encoder is not None \
            else None
        self.inception = inception.to(self.device).eval() if inception is not None else None
        self.inception_fid = inception_fid.to(self.device).eval() if inception_fid is not None else None
        self._graphs = {}
        self._box_graphs = {}
        self._pool = None

    @classmethod
    def from_snapshot(cls, path: str, num_classes: int = 80, device="cuda", shape_snapshot: str | None = None,
                      text_snapshot: str | None = None, glove=None, cat_labels=None, cat_label_lens=None,
                      cat_label_order=None, box_checkpoint: str | None = None, mean_std=None, gaussian_dict=None,
                      cat_ids=None, image_snapshot: str | None = None, inception_weights: str | None = None,
                      fid_dims: int = 2048) -> "GSampler":
        """A reference-format generator snapshot (``netG_epoch_N.pth``, what StepBTrainer.save_model writes), and
        optionally a shape generator snapshot (the reference's ``cfg.TEST.NET_SHP_G``) and a text encoder snapshot
        (``cfg.TRAIN.NET_E``; ntoken is read from its ``encoder.weight``); keys with or without the ``module.`` prefix
        that nn.DataParallel adds.  ``glove``: the GloVe table; ``cat_labels`` / ``cat_label_lens`` /
        ``cat_label_order``: the length-sorted class labels, their lengths and the resort indices of the reference's
        load_cat_label (load.py:305-355), from which the label embeddings are computed once (prepare_cat_emb).
        ``box_checkpoint``: the reference's box checkpoint directory, read with ``mean_std``, ``gaussian_dict`` and
        ``cat_ids`` by BoxGenerator.from_reference (its encoder is the text snapshot's network).  ``image_snapshot``:
        the DAMSM image encoder (``image_encoder100.pth``) for ``encode_image``.  ``inception_weights``: torchvision's
        ImageNet file (``inception_v3_google-1a9a5a14.pth``), from which both scoring networks of ``score_images``
        are built, the FID one returning ``fid_dims`` activations (64, 192, 768 or 2048: cfg.TEST.FID_DIMS)."""
        shp = _new_shp_g(num_classes, device) if shape_snapshot is not None else None
        enc = None
        if text_snapshot is not None:
            text_sd = strip_module_prefix(torch.load(text_snapshot, map_location="cpu"))
            enc = model.RNN_ENCODER(text_sd["encoder.weight"].shape[0], nhidden=cfg.TEXT.EMBEDDING_DIM).to(device)
        clabels = None
        if cat_labels is not None:
            if glove is None:
                raise ValueError("cat_labels need the GloVe table (glove=...)")
            gw = getattr(glove, "weight", glove).detach().to(device).float()
            clabels = ops.class_label_emb(gw, cat_labels.to(device), cat_label_lens.to(device),
                                          cat_label_order.to(device))
        box = None
        if box_checkpoint is not None:
            if text_snapshot is None:
                raise ValueError("box_checkpoint needs the text encoder snapshot (text_snapshot=...)")
            from .boxgen import BoxGenerator
            box = BoxGenerator.from_reference(box_checkpoint, text_snapshot, mean_std, gaussian_dict, cat_ids,
                                              device=device)
        img = model.CNN_ENCODER.from_snapshot(image_snapshot, device) if image_snapshot is not None else None
        inc = fid = None
        if inception_weights is not None:
            imagenet = model._imagenet_state_dict(inception_weights)        # one read of the ~100 MB file for both
            inc = model.INCEPTION_V3.from_imagenet(imagenet, device)
            fid = model.INCEPTION_V3_FID.from_imagenet(imagenet, device,
                                                       [model.INCEPTION_V3_FID.BLOCK_INDEX_BY_DIM[fid_dims]])
        s = cls(_new_g(num_classes, device), shp, enc, glove, clabels, box, img, inc, fid)
        s.load_state_dict(torch.load(path, map_location="cpu"))
        if shape_snapshot is not None:
            s.load_shape_state_dict(torch.load(shape_snapshot, map_location="cpu"))
        if text_snapshot is not None:
            s.load_text_state_dict(text_sd)
        return s

    @classmethod
    def from_trainer(cls, trainer) -> "GSampler":
        """The trainer's EMA generator weights (what the reference snapshots); the trainer is not modified."""
        s = cls(_new_g(trainer.netG.num_classes, trainer.device))
        s.load_state_dict(trainer.bG.ema_state_dict())
        return s

    def encode_image(self, fake_imgs):
        """(region_features (B, nef, 17, 17), cnn_code (B, nef)) of generated images through the image encoder (ref:
        evaluator.py:375-376); ``fake_imgs``: the 256x256 images (B, 3, H, W) or the sampler's list of scales (the last
        one is encoded).  Eager, no gradient."""
        if self.image_encoder is None:
            raise ValueError("this sampler has no image encoder: build it with GSampler(netG, image_encoder=...)")
        if isinstance(fake_imgs, (list, tuple)):
            fake_imgs = fake_imgs[-1]
        with torch.no_grad():
            return self.image_encoder(fake_imgs.detach())

    def score_images(self, fake_imgs):
        """(predictions (B, 1000), activations (B, dims)) of generated images through INCEPTION_V3 and
        INCEPTION_V3_FID (ref: evaluator.py:421-434), for losses.InceptionScore and losses.FrechetDistance;
        ``fake_imgs``: the 256x256 images (B, 3, H, W) or the sampler's list of scales (the last one is scored).
        Eager, no gradient."""
        if self.inception is None or self.inception_fid is None:
            raise ValueError("this sampler has no scoring networks: build it with GSampler(netG, inception=..., "
                             "inception_fid=...) or from_snapshot(..., inception_weights=...)")
        if isinstance(fake_imgs, (list, tuple)):
            fake_imgs = fake_imgs[-1]
        with torch.no_grad():
            x = fake_imgs.detach()
            return self.inception(x), self.inception_fid.activations(x)

    def load_state_dict(self, state_dict: dict) -> None:
        """Loads G weights (strict) and drops every captured graph."""
        self._graphs.clear()
        self._box_graphs.clear()
        self.netG.load_state_dict({k: v.to(self.device) for k, v in state_dict.items()}, strict=True)

    def load_shape_state_dict(self, state_dict: dict) -> None:
        """Loads SHP_G_NET weights (strict; a ``module.`` prefix on every key is dropped) and drops every captured
        graph."""
        if self.netShpG is None:
            raise ValueError("this sampler has no shape generator: build it with GSampler(netG, netShpG)")
        self._graphs.clear()
        self.netShpG.load_state_dict(strip_module_prefix(state_dict), strict=True)

    def load_text_state_dict(self, state_dict: dict) -> None:
        """Loads RNN_ENCODER weights (strict; a ``module.`` prefix on every key is dropped) and drops every captured
        graph."""
        if self.text_encoder is None:
            raise ValueError("this sampler has no text encoder: build it with GSampler(netG, text_encoder=...)")
        self._graphs.clear()
        self.text_encoder.load_state_dict(strip_module_prefix(state_dict), strict=True)

    # ------------------------------------------------------------------ inputs
    def _prepare(self, inp: dict, eager: bool = False) -> dict:
        """Device copies of the inputs G_NET reads (+ the derived tensors of a compact batch), with z and the CA_NET
        noise drawn here, outside any graph, when the batch does not bring them.  The box stage of a caption batch
        without ``rois`` runs here too: replayed from its graph, or without graphs when ``eager``."""
        dev = {}
        for k, v in inp.items():
            dev[k] = _map(v, lambda t: t.to(self.device, non_blocking=True))
        if dev.get("rois") is None and dev.get("captions") is not None:
            lay = self._layout(dev, eager)
            n_host = lay.pop("num_rois_host")
            empty = (n_host == 0).nonzero().view(-1).tolist()
            if len(empty) == len(n_host):
                raise ValueError(f"the box generator made no box for any sample (samples {empty}); sample_layout "
                                 "returns the layouts")
            dev.update(rois=lay["rois"], fm_rois=lay["fm_rois"], roi_cls=lay["roi_cls"], num_rois=lay["num_rois"],
                       glb_max_num_roi=int(n_host.max()))
        text = self._text_mode(dev)
        if dev.get("clabels_emb") is None and self.clabels_emb is not None:
            dev["clabels_emb"] = self.clabels_emb
        gen = self._generates(dev)
        if gen and dev.get("roi_cls") is None:
            dev["roi_cls"] = dev["rois"][0][..., 4].to(torch.int64)
        if not gen and "hmaps" not in dev and "roi_cls" in dev:
            prepare_data(dev, self.netG.num_classes)
        b = dev["num_rois"].shape[0]
        if dev.get("z") is None:
            dev["z"] = torch.randn(b, cfg.GAN.Z_DIM, device=self.device)      # noise_img.data.normal_(0, 1)
        if dev.get("eps") is None:
            dev["eps"] = torch.randn(b, cfg.GAN.CONDITION_DIM, device=self.device)   # CA_NET.reparametrize
        if gen and dev.get("noise_shp") is None:                              # noise_shp.data.normal_(0, 1)
            dev["noise_shp"] = torch.randn(b, cfg.ROI.BOXES_NUM, 4 * self.netShpG.nbf, device=self.device)
        keys = GEN_ARGS if gen else (*G_ARGS, "eps")
        if text:
            keys = tuple(k for k in keys if k not in TEXT_OUT) + TEXT_ARGS
        return {k: dev[k] for k in keys}

    def _text_mode(self, dev: dict) -> bool:
        """Whether the batch's word embeddings come from the text encoder (captions and no ``words_embs``).  Checks the
        caption inputs before anything is launched (one device -> host read, like the reference's
        int(torch.max(cap_lens))) and sets ``max_len`` = max(cap_lens)."""
        if dev.get("words_embs") is not None or dev.get("captions") is None:
            return False
        if self.text_encoder is None or self.glove is None:
            raise ValueError("the batch has captions but no words_embs, and this sampler has no text encoder and GloVe "
                             "table: build it with GSampler(netG, text_encoder=..., glove=...) or "
                             "GSampler.from_snapshot(..., text_snapshot=..., glove=...)")
        caps, lens, gcaps = dev["captions"], dev["cap_lens"], dev["glove_captions"]
        b = caps.shape[0]
        if caps.dim() != 2 or lens.shape != (b,) or gcaps.dim() != 2 or gcaps.shape[0] != b:
            raise ValueError("captions (B, T), cap_lens (B,) and glove_captions (B, T') must agree on B")
        for name, t in (("captions", caps), ("cap_lens", lens), ("glove_captions", gcaps)):
            if t.dtype != torch.int64:
                raise ValueError(f"{name} must be int64")
        lo_c, hi_c, lo_g, hi_g, lo_l, hi_l = torch.stack(
            [caps.min(), caps.max(), gcaps.min(), gcaps.max(), lens.min(), lens.max()]).tolist()
        words_num = cfg.TEXT.WORDS_NUM
        if lo_l < 1 or hi_l > min(words_num, caps.shape[1], gcaps.shape[1]):
            raise ValueError(f"cap_lens must lie in [1, {words_num}] and within the caption width, got [{lo_l}, {hi_l}]")
        if lo_c < 0 or hi_c >= self.text_encoder.ntoken:
            raise ValueError(f"caption token ids must lie in [0, {self.text_encoder.ntoken}), got [{lo_c}, {hi_c}]")
        if lo_g < 0 or hi_g >= self.glove.shape[0]:
            raise ValueError(f"GloVe token ids must lie in [0, {self.glove.shape[0]}), got [{lo_g}, {hi_g}]")
        dev["max_len"] = int(hi_l)
        dev["captions"], dev["glove_captions"] = caps.contiguous(), gcaps.contiguous()
        return True

    def _layout(self, dev: dict, eager: bool = False) -> dict:
        """The box stage of a caption batch without ``rois``: checks its inputs (one device -> host read), draws
        ``noise_box`` / ``noise_cnt`` unless the batch brings them, runs the box graph of (B, box caption length) (or,
        with ``eager``, the same library calls without a graph) and reads ``num_rois`` to the host (the second and last
        read)."""
        box = self.box_generator
        if box is None:
            raise ValueError("the batch has captions but no rois, and this sampler has no box generator: build it with "
                             "GSampler(..., box_generator=...) or GSampler.from_snapshot(..., box_checkpoint=...)")
        if self.netShpG is None and dev.get("bt_masks") is None:
            raise ValueError("a batch whose boxes are generated needs a shape generator: build it with "
                             "GSampler(netG, netShpG, ...) or GSampler.from_snapshot(..., shape_snapshot=...)")
        if ("box_captions" in dev) != ("box_cap_lens" in dev):
            raise ValueError("box_captions and box_cap_lens come together: give both or neither")
        caps = dev.get("box_captions", dev["captions"])
        lens = dev.get("box_cap_lens", dev.get("cap_lens"))
        b = caps.shape[0]
        if caps.dim() != 2 or lens is None or lens.shape != (b,) or caps.dtype != torch.int64 or \
                lens.dtype != torch.int64:
            raise ValueError("box captions (B, T) and their lengths (B,) must be int64 and agree on B")
        lo_c, hi_c, lo_l, hi_l = torch.stack([caps.min(), caps.max(), lens.min(), lens.max()]).tolist()
        if lo_l < 1 or hi_l > caps.shape[1]:
            raise ValueError(f"box caption lengths must lie in [1, {caps.shape[1]}] (the caption width), got "
                             f"[{lo_l}, {hi_l}]")
        if lo_c < 0 or hi_c >= box.encoder.ntoken:
            raise ValueError(f"box caption token ids must lie in [0, {box.encoder.ntoken}), got [{lo_c}, {hi_c}]")
        nb, nc = dev.get("noise_box"), dev.get("noise_cnt")
        if nb is None or nc is None:
            d_nb, d_nc = box.draw_noise(b)
            nb, nc = (d_nb if nb is None else nb), (d_nc if nc is None else nc)
        if nb.shape != (b, box.early_stop_len, NOISE_BOX) or nc.shape != (b, box.num_classes):
            raise ValueError(f"noise_box must be ({b}, {box.early_stop_len}, {NOISE_BOX}) and noise_cnt "
                             f"({b}, {box.num_classes})")
        # the graph's static captions have the key's width, max(lengths), whatever width the batch brings
        ins = dict(captions=caps[:, :int(hi_l)].contiguous(), cap_lens=lens, noise_box=nb.float().contiguous(),
                   noise_cnt=nc.float().contiguous())
        key = (b, int(hi_l))
        entry = self._box_graphs.get(key)
        if eager:
            out = box.sample(ins["captions"], ins["cap_lens"], key[1], ins["noise_box"], ins["noise_cnt"])
        elif entry is None:
            out = box.sample(ins["captions"], ins["cap_lens"], key[1], ins["noise_box"], ins["noise_cnt"])
            self._box_graphs[key] = self._capture_box(ins, key[1])
        else:
            for k, v in entry.static_in.items():
                v.copy_(ins[k], non_blocking=True)
            entry.graph.replay()
            _lib.get().launches += entry.launches
            out = {k: _map(v, lambda t: t.clone()) for k, v in entry.static_out.items()}
        out["num_rois_host"] = out["num_rois"].cpu()
        return out

    def _capture_box(self, ins: dict, max_len: int) -> _Graph:
        static_in = {k: v.clone() for k, v in ins.items()}
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        graph = torch.cuda.CUDAGraph()
        n0 = _lib.get().launches
        box = self.box_generator
        with torch.cuda.graph(graph, pool=self._pool):
            static_out = box.sample(static_in["captions"], static_in["cap_lens"], max_len, static_in["noise_box"],
                                    static_in["noise_cnt"])
        launches = _lib.get().launches - n0
        _lib.get().launches = n0
        keep = [c for n in (box.encoder,) for c in _packed_copies(n)] + [box.decoder.packed_weights()]
        return _Graph(graph, static_in, static_out, launches, keep)

    def sample_layout(self, inp: dict) -> dict:
        """The box stage of a caption batch (graph-replayed like ``sample``): ``rois`` (3 scales, (B, BOXES_NUM, 6)
        float64), ``fm_rois``, ``num_rois``, ``roi_cls`` -- the layout tensors a box batch brings -- and the raw
        trajectory ``labels`` (B, S), ``samples`` (B, S, 4) and ``steps`` (B,).  ``box_captions`` with ``box_cap_lens``
        are read when present (the untruncated captions; both or neither), else ``captions`` / ``cap_lens``; ``noise_box`` /
        ``noise_cnt`` are taken from the batch when present."""
        with torch.no_grad():
            dev = {k: _map(v, lambda t: t.to(self.device, non_blocking=True)) for k, v in inp.items()
                   if k in ("captions", "cap_lens", "box_captions", "box_cap_lens", "noise_box", "noise_cnt")}
            if dev.get("captions") is None:
                raise ValueError("sample_layout needs captions")
            out = self._layout(dev)
            out.pop("num_rois_host")
            return out

    def _generates(self, dev: dict) -> bool:
        """Whether the batch's masks come from the shape generator (the batch brings no ``bt_masks``)."""
        if dev.get("bt_masks") is not None:
            return False
        if self.netShpG is None:
            raise ValueError("the batch has no masks (bt_masks) and this sampler has no shape generator: build it with "
                             "GSampler(netG, netShpG) or GSampler.from_snapshot(..., shape_snapshot=...)")
        return True

    @staticmethod
    def _key(dev: dict) -> tuple:
        gen = "noise_shp" in dev
        text = "captions" in dev
        rmax = int(dev["glb_max_num_roi"]) if gen else dev["slabels_feat"].shape[2]
        length = dev["max_len"] if text else dev["words_embs"].shape[2]
        return (dev["z"].shape[0], length, rmax, int(dev["glb_max_num_roi"]), text, gen)

    def _text(self, dev: dict) -> dict:
        """captions -> RNN_ENCODER (words_embs, sent_emb), GloVe lookups and mask (ref: evaluator.py:337-351)."""
        return text_stage(self.text_encoder, self.glove, dev["captions"], dev["cap_lens"], dev["glove_captions"],
                          dev["max_len"])

    def _shapes(self, dev: dict) -> dict:
        """Box maps -> SHP_G_NET -> form_hmaps (ref: evaluator.py:315-328): the raw masks (B, R, 64, 64) and the heat
        maps / per-roi masks G_NET reads, R = glb_max_num_roi."""
        nbf = self.netShpG.nbf
        rmax = int(dev["glb_max_num_roi"])
        b = dev["z"].shape[0]
        maps, fmaps = ops.form_bbox_maps(dev["rois"][0], dev["fm_rois"], dev["roi_cls"], dev["num_rois"], rmax, nbf,
                                         IMG_SIZES[0], cfg.ROI.FM_SIZE)
        z = dev["noise_shp"][:, :rmax].contiguous()                       # noise_shp[:, :max_num_roi]
        raw = self.netShpG.forward_nhwc(z, maps, fmaps)
        s = IMG_SIZES[0]
        raw_masks = ops.to_nchw(raw, 1).view(b, rmax, s, s)
        hmaps, bt_masks, fm_bt_masks = ops.form_gen_hmaps(raw_masks, dev["roi_cls"], dev["num_rois"], IMG_SIZES, nbf)
        return dict(raw_masks=raw_masks, bbox_fmaps=fmaps, hmaps=hmaps, bt_masks=bt_masks, fm_bt_masks=fm_bt_masks)

    def _forward(self, dev: dict, text_out: dict | None = None, shapes_out: dict | None = None):
        if "captions" in dev:
            text = self._text(dev)
            if text_out is not None:
                text_out.update(text)
            dev = dict(dev, **text)
        if "noise_shp" in dev:
            shapes = self._shapes(dev)
            if shapes_out is not None:
                shapes_out.update(shapes)
            d = dict(dev, **shapes)
            d["slabels_feat"] = ops.form_clabels_feat(dev["clabels_emb"], dev["roi_cls"], dev["num_rois"],
                                                      int(dev["glb_max_num_roi"]))
            dev = d
        g = self.netG
        g.ca_net.eps_override = dev["eps"]
        try:
            return g(*(dev[k] for k in G_ARGS))
        finally:
            g.ca_net.eps_override = None

    # ------------------------------------------------------------------ sampling
    def sample_eager(self, inp: dict, text_out: dict | None = None, shapes_out: dict | None = None):
        """The same forward pass without graphs.  ``text_out``: a dict that receives the text stage's outputs
        (``words_embs``, ``sent_emb``, ``mask``, ``glove_words_embs``) of a caption batch, for R-precision.
        ``shapes_out``: a dict that receives ``sample_shapes``' outputs of a batch without masks."""
        with torch.no_grad():
            return self._forward(self._prepare(inp, eager=True), text_out, shapes_out)

    def sample_shapes(self, inp: dict) -> dict:
        """The generated shapes of a batch without masks (eager): ``raw_masks`` (B, R, 64, 64), the SHP_G_NET output the
        reference's evaluator displays (evaluator.py:317-320), ``bbox_fmaps`` (B, R, 16, 16), and what G_NET reads:
        ``hmaps`` (3 scales), ``bt_masks`` (3 scales) and ``fm_bt_masks``, the per-roi ones zero-padded to BOXES_NUM
        slots.  ``noise_shp`` (B, BOXES_NUM, 4 * num_classes) is taken from the batch when present."""
        with torch.no_grad():
            dev = self._prepare({k: v for k, v in inp.items() if k not in ("bt_masks", "fm_bt_masks", "hmaps")},
                                eager=True)
            return self._shapes(dev)

    def encode_text(self, inp: dict) -> dict:
        """The text stage of a caption batch (eager): ``words_embs`` (B, 256, max_len), ``sent_emb`` (B, 256), ``mask``
        (B, max_len) bool and ``glove_words_embs`` (B, 50, max_len), max_len = max(cap_lens)."""
        with torch.no_grad():
            dev = {k: _map(v, lambda t: t.to(self.device, non_blocking=True)) for k, v in inp.items()
                   if k in ("captions", "cap_lens", "glove_captions")}
            if not self._text_mode(dev):
                raise ValueError("encode_text needs captions, cap_lens and glove_captions")
            return self._text(dev)

    def sample(self, inp: dict):
        """fake_imgs, bt_c_codes, att_maps, bt_att_maps, mu, logvar for the batch ``inp`` (the input dict of
        StepATrainer.generate, full or compact); z / eps are taken from it when present.  A batch without ``bt_masks``
        gets its masks from the shape generator (``noise_shp`` taken from it when present)."""
        with torch.no_grad():
            dev = self._prepare(inp)
            key = self._key(dev)
            entry = self._graphs.get(key)
            if entry is None:
                out = self._forward(dev)          # warm-up: packed weights, allocator state
                self._graphs[key] = self._capture(dev)
                return out
            for k, v in entry.static_in.items():
                if k != "glb_max_num_roi":
                    _copy_into(v, dev[k])
            entry.graph.replay()
            _lib.get().launches += entry.launches
            return _clone_out(entry.static_out)

    def _capture(self, dev: dict) -> _Graph:
        static_in = {k: _map(v, lambda t: t.clone()) for k, v in dev.items()}
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        graph = torch.cuda.CUDAGraph()
        n0 = _lib.get().launches
        with torch.cuda.graph(graph, pool=self._pool):
            static_out = self._forward(static_in)
        launches = _lib.get().launches - n0
        _lib.get().launches = n0              # recorded, not executed
        nets = [n for n in (self.netG, self.netShpG, self.text_encoder) if n is not None]
        return _Graph(graph, static_in, static_out, launches, [c for n in nets for c in _packed_copies(n)])


def _new_g(num_classes, device):
    # the constructor's initialisation is overwritten by the load that follows: skip the per-weight QR of the
    # orthogonal initialisation
    fast, model.FAST_INIT = model.FAST_INIT, True
    try:
        return model.G_NET(num_classes).to(device)
    finally:
        model.FAST_INIT = fast


def _new_shp_g(num_classes, device):
    fast, model.FAST_INIT = model.FAST_INIT, True
    try:
        return model.SHP_G_NET(num_classes).to(device)
    finally:
        model.FAST_INIT = fast


def strip_module_prefix(state_dict: dict) -> dict:
    """A state_dict saved from an nn.DataParallel wrapper (every key ``module.``-prefixed, as the reference's evaluator
    and shape trainer save it) as the bare module's."""
    if state_dict and all(k.startswith("module.") for k in state_dict):
        return {k[len("module."):]: v for k, v in state_dict.items()}
    return dict(state_dict)


def _packed_copies(net):
    """Every kernel-native weight copy the network's layers hold right now (kept alive by a graph that read them)."""
    keep = []
    for m in net.modules():
        for c in (getattr(m, "_cache", None), *getattr(m, "_caches", ())):
            if c is not None:
                keep.append((c.f, c.t, dict(c.hl), c.amax))
    return keep


def _clone_out(out):
    fake, btc, att, btatt, mu, logvar = out
    cl = lambda ts: [t.clone() for t in ts]
    return cl(fake), cl(btc), cl(att), cl(btatt), mu.clone(), logvar.clone()
