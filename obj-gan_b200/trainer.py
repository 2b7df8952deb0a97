"""Step-A of ``condGANTrainer.train`` on the H100 kernels: G forward -> three PatD updates -> G update
(PatD terms + KL) -> EMA, with the reference's ordering and optimiser settings
(reference: image_generation/trainer.py:388-406 and 444-462; ``define_optimizers`` 197-224).

What is different from the reference by design (GPU-first, results identical):
  * each network's parameters / gradients / Adam moments live in one flat fp32 buffer, so the optimiser is
    one fused kernel per network (``og_adam_ema``) and the data-parallel exchange is one NCCL all-reduce per
    network over its gradient bucket (one process per GPU instead of nn.DataParallel, trainer.py:136-152);
  * during the G update the discriminators' parameters do not require grad, which skips the weight-gradient
    GEMMs the reference computes and throws away (miscc/losses.py:372-399 + trainer.py:449-459);
  * no per-step ``.item()`` / ``.cpu()`` synchronisation: losses stay on the device.
"""
from __future__ import annotations

import contextlib
import os
import time
import warnings

import torch
import torch.distributed as dist

from . import lib as _lib
from . import losses, model, ops, snapshots
from .config import cfg

ALIGN = 64  # floats; keeps every parameter view 256-byte aligned inside its bucket


def prepare_data(dev: dict, num_classes: int | None = None, into: dict | None = None) -> dict:
    """Device-side tail of the reference's host data path (ref: trainDataset.py:79-128 ``prepare_data``,
    miscc/load.py:160-176, miscc/utils.py:502-522 ``form_clabels_feat``): from the per-roi masks, the roi class ids
    and the class-label embeddings already on the device, build the 80-channel class heat maps of the three
    scales and the (B, 50, Rmax, 1) label-embedding tensor -- 86 % of the bytes the reference copies host->device
    every step are these derived tensors.  ``num_classes``: heat-map channels (None: one per row of
    ``clabels_emb``).  ``into``: dict holding preallocated ``hmaps`` / ``slabels_feat`` buffers (the static inputs of
    a captured graph) to fill instead of allocating."""
    from . import synth
    dst = into if into is not None else dev
    ncls = num_classes if num_classes is not None else dev["clabels_emb"].shape[0]
    cls, nr = dev["roi_cls"], dev["num_rois"]
    clamp = float(dev.get("hmap_clamp", synth.HMAP_CLAMP))
    have = into is not None and "hmaps" in into
    hm = [ops.form_hmaps(m, cls, nr, ncls, clamp, out=(into["hmaps"][i] if have else None))
          for i, m in enumerate(dev["bt_masks"])]
    rmax = int(dev["glb_max_num_roi"])
    sl = ops.form_clabels_feat(dev["clabels_emb"], cls, nr, rmax,
                               out=(into["slabels_feat"] if into is not None and "slabels_feat" in into else None))
    dst["hmaps"], dst["slabels_feat"] = hm, sl
    return dst


def text_stage(text_encoder, glove, captions, cap_lens, glove_captions, max_len: int) -> dict:
    """The frozen text side of a caption batch (ref: trainer.py:365-380, evaluator.py:337-351): RNN_ENCODER ->
    (words_embs (B, 256, max_len), sent_emb (B, 256)), then the GloVe lookups and padding mask (glove_words_embs
    (B, 50, max_len), mask (B, max_len) bool).  ``captions`` / ``cap_lens`` / ``glove_captions`` are int64 device
    tensors, ``glove`` the (V, 50) table on the device, ``max_len`` = max(cap_lens) as a host int.  The sampler and the
    training loop both call this."""
    words, sent = text_encoder(captions, cap_lens, max_len)
    glove_words, mask = ops.text_inputs(captions, glove_captions, glove, max_len)
    return dict(words_embs=words, sent_emb=sent, mask=mask, glove_words_embs=glove_words)


def _length_sort(cap_lens):
    """(order, order as a list, take) for a batch sorted by caption length, longest first, with a stable sort:
    ``take(t, dtype=None)`` gathers the per-sample tensor ``t`` into that order, converting it to ``dtype`` in the
    same pass, into pinned memory when CUDA is available."""
    order = torch.sort(cap_lens, dim=0, descending=True, stable=True).indices
    pin = torch.cuda.is_available()          # a copy from pageable memory blocks the host until the GPU drains
    idx = order.tolist()

    def take(t, dtype=None):
        t = torch.as_tensor(t)
        out = torch.empty(t.shape, dtype=dtype or t.dtype, pin_memory=pin)
        if out.dtype == t.dtype:
            return torch.index_select(t, 0, order, out=out)
        for j, i in enumerate(idx):          # gather and convert in one pass (the float64 masks: ~110 MB at batch 16)
            out[j].copy_(t[i])
        return out

    return order, idx, take


def prepare_reference_batch(data):
    """The reference's ``prepare_data`` (ref: trainDataset.py:79-128) on the host, producing the compact batch that
    ``StepATrainer.to_device`` takes.  ``data`` is what the reference's DataLoader collates from
    ``TrainDataset.__getitem__``: (imgs, captions, glove_captions, cap_lens, hmaps, rois, fm_rois, num_rois, bt_masks,
    fm_bt_masks, class_ids, keys).

    Every per-sample tensor is reordered by caption length, longest first.  The sort is stable: samples with equal
    lengths keep their loader order (the reference's ``torch.sort(cap_lens, 0, True)`` leaves that order unspecified).
    The masks become float32 like the reference's ``.float()`` calls; the box tables keep their float64, as there.
    The loader's float64 ``hmaps`` are not read: ``to_device`` rebuilds them on the device from the masks and the roi
    classes (column 4 of ``rois[0]``), unclamped like the loader's sums (``hmap_clamp`` 0).  The outputs are pinned
    when CUDA is available, so the copies to the device do not block the host.

    Returns (batch, class_ids, keys): the batch dict (with ``max_len`` = max(cap_lens) and ``host_boxes``, the box
    tables the step reads on the host), the class ids as a numpy array and the keys as a list, both in the sorted
    order."""
    imgs, captions, glove_captions, cap_lens, _hmaps, rois, fm_rois, num_rois, bt_masks, fm_bt_masks, class_ids, \
        keys = data
    cap_lens = torch.as_tensor(cap_lens).to(torch.int64).view(-1)
    b = cap_lens.shape[0]
    order, idx, take = _length_sort(cap_lens)
    rois = [take(r) for r in rois]
    roi_cls = torch.empty(rois[0].shape[:2], dtype=torch.int64, pin_memory=torch.cuda.is_available())
    roi_cls.copy_(rois[0][..., 4])
    batch = dict(imgs=[take(x) for x in imgs], captions=take(torch.as_tensor(captions).reshape(b, -1)),
                 glove_captions=take(torch.as_tensor(glove_captions).reshape(b, -1)), cap_lens=take(cap_lens),
                 rois=rois, fm_rois=take(fm_rois), num_rois=take(torch.as_tensor(num_rois).to(torch.int64).view(-1)),
                 bt_masks=[take(m, torch.float32) for m in bt_masks], fm_bt_masks=take(fm_bt_masks, torch.float32),
                 roi_cls=roi_cls, hmap_clamp=0.0)
    batch["glb_max_num_roi"] = int(batch["num_rois"].max())
    batch["max_len"] = int(cap_lens.max())
    batch["host_boxes"] = {"rois": rois, "fm_rois": batch["fm_rois"], "num_rois": batch["num_rois"]}
    return batch, torch.as_tensor(class_ids)[order].numpy(), [keys[i] for i in idx]


TEST_TUPLE_LEN = {0: 17, 1: 17, 2: 14}     # TestDataset.__getitem__ per cfg.TEST.USE_GT_BOX_SEG (testDataset.py:89-103)


def prepare_reference_test_batch(data, mode=None):
    """The reference's test-time ``prepare_data`` / ``prepare_gen_data`` (ref: testDataset.py:109-244) on the host,
    producing the compact batch that ``GSampler.sample_eager`` takes.  ``data`` is what the reference's DataLoader
    collates from ``TestDataset.__getitem__``: for ``mode`` (cfg.TEST.USE_GT_BOX_SEG when None) 0 or 1 the 17 fields
    (imgs, acts, captions, glove_captions, cap_lens, hmaps, bbox_maps_fwd, bbox_maps_bwd, bbox_fmaps, rois, fm_rois,
    num_rois, bt_masks, fm_bt_masks, class_ids, keys, sent_ids), for mode 2 the 14 without hmaps and masks.  A tuple
    of the other length raises ValueError.

    The sort is ``prepare_reference_batch``'s (stable, longest caption first).  Never read: the images (the evaluator
    scores generated images only), the float64 box maps (~420 MB each at batch 16; ``GSampler`` rasterises them on
    the device from ``rois[0]``, ``fm_rois``, the roi classes and ``num_rois`` with the loader's own rules,
    ops.form_bbox_maps) and the float64 heat maps (rebuilt on the device from the masks, unclamped, ``hmap_clamp``
    0).  Mode 0 keeps the ground-truth masks as float32; modes 1 and 2 send no masks, so the sampler generates them.
    The box tables keep their float64.

    Returns (batch, acts, class_ids, keys, sent_ids), all in the sorted order: the batch dict (with ``max_len`` =
    max(cap_lens)), the real images' FID activations as a float64 tensor, the class ids as a numpy array, and the
    keys and sentence ids as lists."""
    mode = cfg.TEST.USE_GT_BOX_SEG if mode is None else mode
    if mode not in TEST_TUPLE_LEN:
        raise ValueError(f"cfg.TEST.USE_GT_BOX_SEG must be 0, 1 or 2, got {mode}")
    if len(data) != TEST_TUPLE_LEN[mode]:
        raise ValueError(f"USE_GT_BOX_SEG = {mode} takes the {TEST_TUPLE_LEN[mode]}-field test tuple, got "
                         f"{len(data)} fields")
    if mode == 2:
        _imgs, acts, captions, glove_captions, cap_lens, _fwd, _bwd, _fmaps, rois, fm_rois, num_rois, class_ids, keys, \
            sent_ids = data
    else:
        _imgs, acts, captions, glove_captions, cap_lens, _hmaps, _fwd, _bwd, _fmaps, rois, fm_rois, num_rois, bt_masks, \
            fm_bt_masks, class_ids, keys, sent_ids = data
    cap_lens = torch.as_tensor(cap_lens).to(torch.int64).view(-1)
    b = cap_lens.shape[0]
    order, idx, take = _length_sort(cap_lens)
    rois = [take(r) for r in rois]
    roi_cls = torch.empty(rois[0].shape[:2], dtype=torch.int64, pin_memory=torch.cuda.is_available())
    roi_cls.copy_(rois[0][..., 4])
    batch = dict(captions=take(torch.as_tensor(captions).reshape(b, -1)),
                 glove_captions=take(torch.as_tensor(glove_captions).reshape(b, -1)), cap_lens=take(cap_lens),
                 rois=rois, fm_rois=take(fm_rois), num_rois=take(torch.as_tensor(num_rois).to(torch.int64).view(-1)),
                 roi_cls=roi_cls)
    if mode == 0:
        batch.update(bt_masks=[take(m, torch.float32) for m in bt_masks], fm_bt_masks=take(fm_bt_masks, torch.float32),
                     hmap_clamp=0.0)
    batch["glb_max_num_roi"] = int(batch["num_rois"].max())
    batch["max_len"] = int(cap_lens.max())
    sent_ids = torch.as_tensor(sent_ids).view(-1).tolist()
    return (batch, take(acts), torch.as_tensor(class_ids)[order].numpy(), [keys[i] for i in idx],
            [sent_ids[i] for i in idx])


def gather_inception_score(score, world, rank, process_group=None):
    """An InceptionScore over every data-parallel rank's predictions: one gather to rank 0 (None on the other ranks).
    Rank r's predictions follow rank r-1's."""
    if world == 1:
        return score
    local = torch.cat(score.predictions, 0)
    n = torch.tensor([local.shape[0]], device=local.device, dtype=torch.int64)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n, group=process_group)
    counts = [int(c) for c in counts]
    pad = local.new_zeros((max(counts), local.shape[1]))
    pad[:local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=process_group)
    if rank != 0:
        return None
    out = losses.InceptionScore(score.num_splits)
    for p, c in zip(parts, counts):
        out.add(p[:c])
    return out


class FlatBucket:
    """Parameters of one network as views of a single flat buffer (+ matching grad / Adam state)."""

    def __init__(self, module: torch.nn.Module, ema: bool = False):
        self.module = module
        self.params = [p for p in module.parameters()]
        dev = self.params[0].device
        offs, total = [], 0
        for p in self.params:
            offs.append(total)
            total += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        self.numel = total
        self.flat = torch.zeros(total, device=dev)
        self.grad = torch.zeros(total, device=dev)
        self.m = torch.zeros(total, device=dev)
        self.v = torch.zeros(total, device=dev)
        for p, o in zip(self.params, offs):
            n = p.numel()
            self.flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat[o:o + n].view(p.shape)
            p.grad = self.grad[o:o + n].view(p.shape)
            p.og_grad_sink = p.grad          # the backward kernels accumulate here directly (ops._grad_sink)
        self.avg = self.flat.clone() if ema else None
        self.offsets = offs
        self.plan = ops.PackPlan()           # fp16 operand copies of this network's conv weights: re-packed in one go
        self.epoch = [0]                     # bumped by THIS network's optimiser step only (ops._epoch_of)
        for p in self.params:
            p.og_pack_plan = self.plan
            p.og_epoch = self.epoch
        self.step = 0
        self.step_dev = torch.zeros((), device=dev, dtype=torch.int64)   # device mirror (CUDA-graph replay)
        ops.bump_param_epoch()

    def zero_grad(self):
        self.grad.zero_()

    def requires_grad_(self, flag: bool):
        for p in self.params:
            p.requires_grad_(flag)

    def adam(self, lr, gscale=1.0):
        self.step += 1
        ops.adam_ema_(self.flat, self.grad, self.m, self.v, self.avg, self.step, lr=lr, b1=0.5, b2=0.999, eps=1e-8,
                      gscale=gscale, decay=0.999, step_dev=self.step_dev, bump=False)
        self.epoch[0] += 1
        self.plan.run()                       # every tensor-core operand copy of this network, two launches

    def ema_state_dict(self):
        """EMA weights keyed like ``module.state_dict()`` (what the reference saves as netG_epoch_%d.pth,
        trainer.py:251-256)."""
        sd = {k: v.clone() for k, v in self.module.state_dict().items()}
        names = [n for n, _ in self.module.named_parameters()]
        for n, p, o in zip(names, self.params, self.offsets):
            sd[n] = self.avg[o:o + p.numel()].view(p.shape).clone()
        return sd


class StepATrainer:
    """Owns G_NET + PAT_D_NET64/128/256 and runs Step-A steps on one GPU (one rank of a DP group)."""

    def __init__(self, num_classes=80, device="cuda", process_group=None, seed=None):
        if seed is not None:
            torch.manual_seed(seed)
        self.device = torch.device(device)
        self.netG = model.G_NET(num_classes)
        self.netsPatD = [model.PAT_D_NET64(), model.PAT_D_NET128(), model.PAT_D_NET256()][:cfg.TREE.BRANCH_NUM]
        self.netG.apply(model.weights_init)
        for d in self.netsPatD:
            d.apply(model.weights_init)
        self.netG.to(self.device)
        for d in self.netsPatD:
            d.to(self.device)
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self._flatten()

    def _flatten(self):
        self.bG = FlatBucket(self.netG, ema=True)
        self.bD = [FlatBucket(d) for d in self.netsPatD]

    def load_reference_state(self, g_sd, d_sds):
        """Load reference-format state_dicts (strict) and rebuild the flat buckets."""
        self.netG.load_state_dict({k: v.to(self.device) for k, v in g_sd.items()}, strict=True)
        for d, sd in zip(self.netsPatD, d_sds):
            d.load_state_dict({k: v.to(self.device) for k, v in sd.items()}, strict=True)
        self._flatten()

    def broadcast_parameters(self):
        """Identical initial weights on every rank (the reference's DataParallel replicates from GPU0)."""
        if self.world > 1:
            for b in [self.bG, *self.bD]:
                dist.broadcast(b.flat, src=0, group=self.pg)
            self.bG.avg.copy_(self.bG.flat)
            for m in [self.netG, *self.netsPatD]:
                for buf in m.buffers():
                    dist.broadcast(buf, src=0, group=self.pg)
            ops.bump_param_epoch()

    def _branch_streams(self):
        """Side streams for the three independent discriminator branches (None: run them in sequence)."""
        if not torch.cuda.is_available() or _lib.DRY_RUN:
            return None
        if not hasattr(self, "_dstreams"):
            self._dstreams = [torch.cuda.Stream() for _ in self.netsPatD]
        return self._dstreams

    def _allreduce(self, bucket):
        if self.world > 1:
            return dist.all_reduce(bucket.grad, op=dist.ReduceOp.SUM, group=self.pg, async_op=True)
        return None

    def to_device(self, inp: dict) -> dict:
        """Host (pinned) batch -> device tensors; non_blocking so copies overlap with queued kernels."""
        out = {}
        for k, v in inp.items():
            if torch.is_tensor(v):
                out[k] = v.to(self.device, non_blocking=True)
            elif isinstance(v, (list, tuple)):
                out[k] = [t.to(self.device, non_blocking=True) for t in v]
            else:
                out[k] = v
        if "hmaps" not in out and "roi_cls" in out:
            self.prepare_data(out)       # compact batch: rebuild the class heat maps / label embeddings on the device
        # box tables stay readable on the host as well: the roi filter of feat_select and the class shuffles of
        # permute_seg are host decisions (like the reference), and reading them back from the device would stall the
        # step (the reference does exactly that: .cpu() in utils.py:447, 467)
        out["host_boxes"] = {"rois": [r.detach().cpu() for r in inp["rois"]], "fm_rois": inp["fm_rois"].detach().cpu(),
                             "num_rois": inp["num_rois"].detach().cpu()}
        return out

    def prepare_data(self, dev: dict, into: dict | None = None) -> dict:
        """Builds the derived inputs of a compact batch on the device (module-level ``prepare_data``)."""
        return prepare_data(dev, getattr(self.netG, "num_classes", None), into)

    def generate(self, inp):
        g = self.netG
        g.ca_net.eps_override = inp.get("eps")
        return g(inp["z"], inp["sent_emb"], inp["words_embs"], inp["glove_words_embs"], inp["slabels_feat"],
                 inp["mask"], inp["hmaps"], inp["rois"], inp["fm_rois"], inp["num_rois"], inp["bt_masks"],
                 inp["fm_bt_masks"], inp["glb_max_num_roi"])

    # ------------------------------------------------------------------ CUDA graph
    def capture(self, inp: dict, warmup: int = 2) -> None:
        """Capture one whole Step-A step (forward, backward, all-reduce, optimiser) into a CUDA graph.  ``inp`` fixes
        the shapes; later ``step`` calls copy their inputs into the captured static buffers and replay.  The ~1200
        kernel launches of a step then cost one graph launch instead of ~0.1 ms of Python/ctypes each.  The ``warmup``
        eager steps it runs first are undone afterwards (weights, Adam state, EMA, BatchNorm buffers restored), so the
        call does not advance training."""
        from . import lib as _l
        self._static = {}
        for k, v in inp.items():
            if torch.is_tensor(v):
                self._static[k] = v.clone()
            elif isinstance(v, (list, tuple)):
                self._static[k] = [t.clone() for t in v]
            else:
                self._static[k] = v
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        # the warm-up steps are REAL optimiser steps on the sample batch: snapshot everything they touch (weights, Adam
        # moments, EMA, step counters, BatchNorm buffers) and put it back, so capture() leaves the training state as
        # it found it
        nets = [self.netG, *self.netsPatD]
        snap = [(b, b.flat.clone(), b.m.clone(), b.v.clone(), None if b.avg is None else b.avg.clone(), b.step,
                 b.step_dev.clone()) for b in [self.bG, *self.bD]]
        bufs = [[t.clone() for t in m.buffers()] for m in nets]
        with torch.cuda.stream(side):
            for _ in range(warmup):          # allocator / kernel-attribute / packed-weight-cache steady state
                self._eager_step(self._static)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        for b, flat, m, v, avg, step, step_dev in snap:
            b.flat.copy_(flat); b.m.copy_(m); b.v.copy_(v); b.step = step; b.step_dev.copy_(step_dev)
            if avg is not None:
                b.avg.copy_(avg)
        for mod, saved in zip(nets, bufs):
            for t, s0 in zip(mod.buffers(), saved):
                t.copy_(s0)
        ops.bump_param_epoch()
        for b in [self.bG, *self.bD]:
            b.plan.run()                     # operand copies of the restored weights
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        n0 = _l.get().launches
        # capture on the SAME side stream as the warm-up: autograd's AccumulateGrad nodes remember the stream they were
        # created on, and gradient accumulation issued on any other stream would fall outside the capture
        with torch.cuda.graph(self._graph, stream=side):
            self._static_out = self._eager_step(self._static)
        self.launches_per_step = _l.get().launches - n0
        for b in [self.bG, *self.bD]:
            b.step -= 1          # the captured pass was recorded, not executed

    def _load_static(self, inp: dict) -> None:
        for k, v in inp.items():
            dst = self._static.get(k)
            if torch.is_tensor(v) and torch.is_tensor(dst):
                if dst.data_ptr() != v.data_ptr():
                    dst.copy_(v, non_blocking=True)
            elif isinstance(v, (list, tuple)):
                for d, t in zip(dst, v):
                    if d.data_ptr() != t.data_ptr():
                        d.copy_(t, non_blocking=True)

    def step(self, inp: dict) -> dict:
        """One Step-A step.  Eager, or a replay of the captured CUDA graph after ``capture``."""
        if getattr(self, "_graph", None) is None:
            return self._eager_step(inp)
        from . import lib as _l
        self._load_static(inp)
        self._graph.replay()
        _l.get().launches += self.launches_per_step
        for b in [self.bG, *self.bD]:
            b.step += 1
        ops.bump_param_epoch()
        return self._static_out

    @staticmethod
    def _nvtx(name):
        """NVTX range around a phase of the step (OBJGAN_NVTX=1; shows up in Nsight timelines), else a no-op."""
        if os.environ.get("OBJGAN_NVTX") == "1" and torch.cuda.is_available():
            return torch.cuda.nvtx.range(name)
        return contextlib.nullcontext()

    def _eager_step(self, inp: dict) -> dict:
        """One Step-A step on device-resident inputs.  Returns losses as device scalars."""
        lr_d, lr_g = cfg.TRAIN.DISCRIMINATOR_LR, cfg.TRAIN.GENERATOR_LR
        gs = 1.0 / self.world
        sent = inp["sent_emb"]
        # (2) generate fake images
        self.bG.requires_grad_(True)
        with self._nvtx("G forward"):
            fake_imgs, _bt_c, _att, _bt_att, mu, logvar = self.generate(inp)
        out = {}
        # (3-1) update the patch discriminators
        streams = self._branch_streams()
        main = torch.cuda.current_stream() if streams else None
        for b in self.bD:
            b.requires_grad_(True)
            b.zero_grad()
        for i, (d, b) in enumerate(zip(self.netsPatD, self.bD)):
            # the three discriminator updates are independent: each runs on its own stream (forked from and joined to
            # the step's stream, so a CUDA-graph capture records them as parallel branches) and their many small
            # kernels fill the GPU together
            if streams:
                streams[i].wait_stream(main)
            with (torch.cuda.stream(streams[i]) if streams else contextlib.nullcontext()):
                err = losses.patD_loss(d, inp["imgs"][i], fake_imgs[i], sent)
                err.backward()
                out[f"errPatD{i}"] = err.detach()
                # the gradient exchange and the optimiser step of this discriminator stay on ITS branch: the
                # all-reduce of the small 64 / 128 discriminators runs under the backward pass of the 256 one
                # (every rank issues the three collectives in the same program order)
                w = self._allreduce(b)
                if w is not None:
                    w.wait()
                b.adam(lr_d, gs)
        for i, b in enumerate(self.bD):
            if streams:
                main.wait_stream(streams[i])
        # (4) update G through the updated discriminators (their weight gradients are not needed)
        for b in self.bD:
            b.requires_grad_(False)
        self.bG.zero_grad()
        with self._nvtx("G loss + backward"):
            err_g, _ = losses.G_loss_pat(self.netsPatD, fake_imgs, sent, streams)
            kl = losses.KL_loss(mu, logvar)
            total = err_g + kl
            total.backward()
        with self._nvtx("G all-reduce + Adam + EMA"):
            w = self._allreduce(self.bG)
            if w is not None:
                w.wait()
            self.bG.adam(lr_g, gs)  # fused Adam + EMA (trainer.py:460-462)
        out["errG"] = err_g.detach()
        out["kl"] = kl.detach()
        out["fake_imgs"] = [f.detach() for f in fake_imgs]
        return out

    def step_from_host(self, host_inp: dict) -> float:
        """The public end-to-end call: pinned host batch in, scalar generator loss out.

        With a captured graph the call is software-pipelined: the host->device copy of THIS batch runs on a copy
        stream into a staging buffer while the previous step is still computing, and the value returned is the
        loss of the PREVIOUS step (its device->host read completes here), so every call still performs one full
        H2D of its inputs and one D2H read of a step result, but neither stalls the GPU.  The first call returns
        its own loss."""
        if getattr(self, "_graph", None) is None:
            out = self.step(self.to_device(host_inp))
            return float((out["errG"] + out["kl"]).item())
        cur = torch.cuda.current_stream()
        if not hasattr(self, "_stage"):
            def clone(v):
                return [t.clone() for t in v] if isinstance(v, (list, tuple)) else (v.clone() if torch.is_tensor(v) else v)
            self._stage = [{k: clone(v) for k, v in self._static.items()} for _ in range(2)]
            self._stage_free = [torch.cuda.Event(), torch.cuda.Event()]
            for e in self._stage_free:
                e.record(cur)
            self._copy_stream = torch.cuda.Stream()
            self._loss_host = [torch.zeros((), pin_memory=True), torch.zeros((), pin_memory=True)]
            self._pending = None
            self._e2e_k = 0
        k = self._e2e_k & 1
        self._e2e_k += 1
        stg = self._stage[k]
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._stage_free[k])       # staging buffer k was consumed two steps ago
            for name, v in host_inp.items():
                d = stg.get(name)
                if torch.is_tensor(v) and torch.is_tensor(d):
                    d.copy_(v, non_blocking=True)
                elif isinstance(v, (list, tuple)):
                    for dd, t in zip(d, v):
                        dd.copy_(t, non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(self._copy_stream)
        cur.wait_event(copied)
        if "hmaps" not in host_inp and "roi_cls" in host_inp:       # compact batch: derived tensors built in place
            self.prepare_data(stg, into=self._static)
        self._load_static({k: v for k, v in stg.items() if k in host_inp})   # device->device into the captured buffers
        self._stage_free[k].record(cur)
        out = self.step(self._static)
        self._loss_host[k].copy_(out["errG"] + out["kl"], non_blocking=True)
        done = torch.cuda.Event()
        done.record(cur)
        prev, self._pending = self._pending, (done, self._loss_host[k])
        if prev is None:
            done.synchronize()
            return float(self._loss_host[k])
        prev[0].synchronize()
        return float(prev[1])


def pin(inp: dict) -> dict:
    out = {}
    for k, v in inp.items():
        if torch.is_tensor(v):
            out[k] = v.pin_memory() if torch.cuda.is_available() else v
        elif isinstance(v, (list, tuple)):
            out[k] = [t.pin_memory() if torch.cuda.is_available() else t for t in v]
        else:
            out[k] = v
    return out


class StepBTrainer(StepATrainer):
    """The reference's complete training step (ref: trainer.py:385-462): generator forward, then the updates of the three
    patch discriminators, the three shape discriminators, the small- and large-scale object discriminators, and the
    generator update through all eight of them (+ the DAMSM terms when an ``image_encoder`` is given + KL) with the
    fused Adam + EMA.  The box filter of ``feat_select`` and the shuffles of ``permute_seg`` are host decisions (as in
    the reference), so this step runs eagerly; Step-A (the data-parallel hot path of the bench) is the captured one."""

    def __init__(self, num_classes=80, device="cuda", process_group=None, seed=None, image_encoder=None):
        super().__init__(num_classes, device, process_group, seed)
        n = cfg.TREE.BRANCH_NUM
        self.netsShpD = [model.SHP_D_NET64(num_classes), model.SHP_D_NET128(num_classes),
                         model.SHP_D_NET256(num_classes)][:n]
        self.netObjSSD, self.netObjLSD = model.OBJ_SS_D_NET(num_classes), model.OBJ_LS_D_NET(num_classes)
        for d in [*self.netsShpD, self.netObjSSD, self.netObjLSD]:
            d.apply(model.weights_init)
            d.to(self.device)
        self.bShp = [FlatBucket(d) for d in self.netsShpD]
        self.bObj = [FlatBucket(self.netObjSSD), FlatBucket(self.netObjLSD)]
        self.image_encoder = image_encoder        # pretrained CNN_ENCODER (stock PyTorch, frozen); None: no DAMSM terms
        if image_encoder is not None:
            for p in image_encoder.parameters():
                p.requires_grad_(False)

    def _d_buckets(self):
        return [*self.bD, *self.bShp, *self.bObj]

    def broadcast_parameters(self):
        super().broadcast_parameters()
        if self.world > 1:
            for b in [*self.bShp, *self.bObj]:
                dist.broadcast(b.flat, src=0, group=self.pg)
            for m in [*self.netsShpD, self.netObjSSD, self.netObjLSD]:
                for buf in m.buffers():
                    dist.broadcast(buf, src=0, group=self.pg)
            ops.bump_param_epoch()

    # ------------------------------------------------------------------ reference-format snapshots
    def save_model(self, model_dir: str, epoch: int) -> list:
        """The reference's snapshot file set (ref: trainer.py:251-273): ``netG_epoch_%d.pth`` holds the EMA weights
        (the reference swaps avg_param_G in before saving), ``netPatD%d.pth`` / ``netShpD%d.pth`` / ``netObjSSD.pth``
        / ``netObjLSD.pth`` the live discriminators; plain ``state_dict`` pickles with the reference's keys, on
        the CPU so either side can load them."""
        os.makedirs(model_dir, exist_ok=True)
        cpu = lambda sd: {k: v.detach().cpu().clone() for k, v in sd.items()}
        files = {f"netG_epoch_{epoch}.pth": cpu(self.bG.ema_state_dict())}
        for i, d in enumerate(self.netsPatD):
            files[f"netPatD{i}.pth"] = cpu(d.state_dict())
        for i, d in enumerate(self.netsShpD):
            files[f"netShpD{i}.pth"] = cpu(d.state_dict())
        files["netObjSSD.pth"] = cpu(self.netObjSSD.state_dict())
        files["netObjLSD.pth"] = cpu(self.netObjLSD.state_dict())
        for name, sd in files.items():
            torch.save(sd, os.path.join(model_dir, name))
        return sorted(files)

    def load_model(self, net_g_path: str) -> int:
        """Resume like the reference's ``build_models`` (ref: trainer.py:152-194): ``cfg.TRAIN.NET_G`` names the
        generator snapshot, the discriminators are read from the same directory; returns the epoch to continue
        from (snapshot epoch + 1).  Rebuilds the flat buckets (fresh Adam moments, like the reference; EMA restarts
        from the loaded weights, ref: trainer.py:303)."""
        load = lambda f: torch.load(f, map_location="cpu")
        to = lambda sd: {k: v.to(self.device) for k, v in sd.items()}
        self.netG.load_state_dict(to(load(net_g_path)), strict=True)
        d = os.path.dirname(net_g_path)
        for i, net in enumerate(self.netsPatD):
            net.load_state_dict(to(load(os.path.join(d, f"netPatD{i}.pth"))), strict=True)
        for i, net in enumerate(self.netsShpD):
            net.load_state_dict(to(load(os.path.join(d, f"netShpD{i}.pth"))), strict=True)
        self.netObjSSD.load_state_dict(to(load(os.path.join(d, "netObjSSD.pth"))), strict=True)
        self.netObjLSD.load_state_dict(to(load(os.path.join(d, "netObjLSD.pth"))), strict=True)
        self._flatten()
        self.bShp = [FlatBucket(n) for n in self.netsShpD]
        self.bObj = [FlatBucket(self.netObjSSD), FlatBucket(self.netObjLSD)]
        name = os.path.basename(net_g_path)
        return int(name[name.rfind("_") + 1:name.rfind(".")]) + 1

    def _update(self, bucket, err, lr, gs):
        """backward + all-reduce + Adam for one discriminator.  ``err`` may be the int 0 of an empty roi set (the
        reference then skips the optimiser step, trainer.py:428-431); with several ranks the exchange must stay
        collective, so the ranks first agree whether ANY of them has a loss, and a rank without one contributes a
        zero gradient."""
        mine = torch.is_tensor(err)
        anyone = mine
        if self.world > 1:
            flag = torch.tensor([1.0 if mine else 0.0], device=bucket.flat.device)
            dist.all_reduce(flag, op=dist.ReduceOp.SUM, group=self.pg)
            anyone = bool(flag.item() > 0)
        if mine:
            err.backward()
        if not anyone:
            return None
        w = self._allreduce(bucket)
        if w is not None:
            w.wait()
        bucket.adam(lr, gs)
        return err.detach() if mine else None

    def step(self, inp: dict, class_ids=None) -> dict:
        lr_d, lr_g = cfg.TRAIN.DISCRIMINATOR_LR, cfg.TRAIN.GENERATOR_LR
        gs = 1.0 / self.world
        sent, imgs, hmaps, rois = inp["sent_emb"], inp["imgs"], inp["hmaps"], inp["rois"]
        fm_rois, num_rois = inp["fm_rois"], inp["num_rois"]
        hb = inp.get("host_boxes")
        if hb is None:                               # device-only batch: one synchronising read of the box tables
            host = lambda t: t.detach().cpu() if torch.is_tensor(t) else t
            hb = {"rois": [host(r) for r in rois], "fm_rois": host(fm_rois), "num_rois": host(num_rois)}
        rois_h, fm_h, nr_h = hb["rois"], hb["fm_rois"], hb["num_rois"]
        self.bG.requires_grad_(True)
        fake_imgs, bt_c_codes, _att, _bt_att, mu, logvar = self.generate(inp)
        bt_c_codes = [c.detach() for c in bt_c_codes]       # ref: trainer.py:393 -- constants for every loss below
        out = {}
        for b in self._d_buckets():
            b.requires_grad_(True)
            b.zero_grad()
        # (3-1) patch discriminators, (3-2) shape discriminators.  The eight discriminator updates run in sequence on the
        # step's stream: forking them onto eight streams (as Step-A does with its three patch discriminators) was
        # measured at batch 16 and stalled the GPU for minutes once consecutive steps were enqueued without a
        # synchronisation in between, so it is not done here.
        for i, (d, b) in enumerate(zip(self.netsPatD, self.bD)):
            out[f"errPatD{i}"] = self._update(b, losses.patD_loss(d, imgs[i], fake_imgs[i], sent), lr_d, gs)
        for i, (d, b) in enumerate(zip(self.netsShpD, self.bShp)):
            out[f"errShpD{i}"] = self._update(b, losses.shpD_loss(d, imgs[i], fake_imgs[i], hmaps[i], rois_h[i], nr_h),
                                              lr_d, gs)
        # (3-3) / (3-4) object discriminators (small scale on the 64-scale boxes, large scale on the feature-map boxes)
        codes = bt_c_codes[-1]
        out["errObjSSD"] = self._update(self.bObj[0], losses.objD_loss(
            self.netObjSSD, imgs[-1], fake_imgs[-1], hmaps[-1], inp["clabels_emb"], codes, rois_h[0], nr_h), lr_d, gs)
        out["errObjLSD"] = self._update(self.bObj[1], losses.objD_loss(
            self.netObjLSD, imgs[-1], fake_imgs[-1], hmaps[-1], inp["clabels_emb"], codes, fm_h, nr_h,
            is_large_scale=True), lr_d, gs)
        # (4) generator
        for b in self._d_buckets():
            b.requires_grad_(False)
        self.bG.zero_grad()
        labels = torch.arange(fake_imgs[0].size(0), device=fake_imgs[0].device)
        err_g, logs = losses.G_loss(self.netsPatD, self.netsShpD, self.netObjSSD, self.netObjLSD, self.image_encoder,
                                    fake_imgs, hmaps, inp["words_embs"], sent, inp["clabels_emb"], codes, labels,
                                    inp["cap_lens"], class_ids, rois_h[0], fm_h, nr_h)
        kl = losses.KL_loss(mu, logvar)
        (err_g + kl).backward()
        w = self._allreduce(self.bG)
        if w is not None:
            w.wait()
        self.bG.adam(lr_g, gs)
        out.update(errG=err_g.detach(), kl=kl.detach(), logs=logs, fake_imgs=[f.detach() for f in fake_imgs])
        return out


class condGANTrainer:
    """The reference's training loop (ref: trainer.py:30-511, ``condGANTrainer``) on this library: the same constructor
    and ``train()``, fed by the reference's own DataLoader.  Each step runs the intake (``prepare_reference_batch``),
    the copies to the device and the heat-map rebuild, the frozen text encoder (``text_stage``), the complete step
    (``StepBTrainer.step``, DAMSM terms included) and INCEPTION_V3 on the 256-pixel images; the predictions stay on the
    device until the end of the epoch, when ``Score/scores_%d.txt`` is written in the reference's format.  Snapshots
    are the reference's file set (``StepBTrainer.save_model``) under ``Model/``; ``cfg.TRAIN.NET_G`` resumes.

    ``dataset`` provides what the reference reads from it: ``n_words``, ``cats_index_dict``, ``cat_labels``,
    ``cat_label_lens``, ``sorted_cat_label_indices`` and ``glove_embed``.  ``inception_weights``: torchvision's
    ImageNet file (``inception_v3_google-1a9a5a14.pth``, its path or its loaded state_dict) for INCEPTION_V3; the
    reference downloads it, this library reads no network.

    Under torchrun (one process per GPU, each with its own shard of the data): every rank trains on its own batches
    and the ranks exchange gradients through ``process_group``; the epoch's Inception score covers every rank's
    predictions, gathered to rank 0 once per epoch, and only rank 0 prints and writes files.

    Every DISPLAY_INTERVAL steps rank 0 writes the reference's attention-map PNGs to ``Image/`` (``save_img_results``)
    from the EMA weights and the noise drawn once in ``setup()``: ``G_average_<epoch>_<i>.png`` and
    ``bt_G_average_<epoch>_<i>.png`` per stage, ``D_average_<epoch>.png`` with the DAMSM word maps.  ``font``: the
    caption font, a TrueType path or a PIL font (default: the reference's cfg.DATA_DIR +
    '/share/Pillow/Tests/fonts/FreeMono.ttf' at size 50); without one no PNG is written and the first display step
    warns.  ``dataset.ixtoword`` names the caption tokens."""

    def __init__(self, output_dir, data_loader, dataset, *, inception_weights, device=None, process_group=None,
                 font=None):
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.model_dir = os.path.join(output_dir, "Model")
        self.image_dir = os.path.join(output_dir, "Image")
        self.score_dir = os.path.join(output_dir, "Score")
        if cfg.TRAIN.FLAG and self.rank == 0:
            for d in (self.model_dir, self.image_dir, self.score_dir):
                os.makedirs(d, exist_ok=True)
        self.batch_size = cfg.TRAIN.BATCH_SIZE
        self.max_epoch = cfg.TRAIN.MAX_EPOCH
        self.snapshot_interval = cfg.TRAIN.SNAPSHOT_INTERVAL
        self.print_interval = cfg.TRAIN.PRINT_INTERVAL
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
        self.ixtoword = getattr(dataset, "ixtoword", None)
        self.font = snapshots.load_font(font)
        self.fixed_noise = None
        self._display = None
        self._warned_font = False

    def build_models(self):
        """(text_encoder, image_encoder, StepBTrainer, INCEPTION_V3, start_epoch), like the reference's build_models
        (ref: trainer.py:75-195): the DAMSM encoders from cfg.TRAIN.NET_E (the image encoder's path is NET_E with
        ``text_encoder`` -> ``image_encoder``), fresh networks or the snapshot of cfg.TRAIN.NET_G, identical on every
        rank."""
        from .sampler import strip_module_prefix
        if not cfg.TRAIN.NET_E:
            raise ValueError("no pretrained text-image encoders: set cfg.TRAIN.NET_E")
        dev = self.device
        image_encoder = model.CNN_ENCODER.from_snapshot(cfg.TRAIN.NET_E.replace("text_encoder", "image_encoder"), dev,
                                                        nef=cfg.TEXT.EMBEDDING_DIM)
        text_encoder = model.RNN_ENCODER(self.n_words, nhidden=cfg.TEXT.EMBEDDING_DIM).to(dev)
        text_encoder.load_state_dict(strip_module_prefix(torch.load(cfg.TRAIN.NET_E, map_location="cpu")), strict=True)
        text_encoder.requires_grad_(False).eval()
        net = StepBTrainer(len(self.cats_index_dict), dev, self.pg, image_encoder=image_encoder)
        start_epoch = net.load_model(cfg.TRAIN.NET_G) if cfg.TRAIN.NET_G else 0
        net.broadcast_parameters()
        inception = model.INCEPTION_V3.from_imagenet(self.inception_weights, dev)
        return text_encoder, image_encoder, net, inception, start_epoch

    def prepare_cat_emb(self):
        """(num_classes, 50) label embeddings on the device (ref: trainer.py:226-242)."""
        as_i64 = lambda t: torch.as_tensor(t).to(self.device, torch.int64)
        return ops.class_label_emb(self.glove, as_i64(self.cat_labels), as_i64(self.cat_label_lens),
                                   as_i64(self.sorted_cat_label_indices))

    def setup(self):
        """Builds the networks, the GloVe table and the label embeddings; returns the epoch to start from."""
        self.text_encoder, self.image_encoder, self.net, self.inception, start = self.build_models()
        glove = getattr(self.glove_emb, "weight", self.glove_emb)
        self.glove = glove.detach().to(self.device).float().contiguous()
        self.clabels_emb = self.prepare_cat_emb()
        # ref: trainer.py:336-337: drawn from the host generator, as there, but only when the PNGs can be written, so
        # that without a font the host random stream (the loader's shuffles) is the one it always was.  Every rank
        # loads the font and draws, so the ranks' streams stay alike; only rank 0 renders.
        if self.font is not None:
            self.fixed_noise = torch.randn(self.batch_size, cfg.GAN.Z_DIM).to(self.device)
        return start

    def train_step(self, data, score=None, z=None, eps=None) -> dict:
        """One step of the loop body (ref: trainer.py:361-469) on one loader batch: intake, copies to the device, text stage, fresh noise (``z`` / the CA_NET
        ``eps`` when given), the complete step, and the Inception predictions of ``fake_imgs[-1]`` added to ``score``
        (a losses.InceptionScore).  Returns the step's outputs (device tensors) with the sorted ``class_ids``
        and ``keys``."""
        batch, class_ids, keys = prepare_reference_batch(data)
        batch = dict(batch, clabels_emb=self.clabels_emb)
        dev = self.net.to_device(batch)
        with torch.no_grad():
            dev.update(text_stage(self.text_encoder, self.glove, dev["captions"], dev["cap_lens"],
                                  dev["glove_captions"], batch["max_len"]))
        b = dev["num_rois"].shape[0]
        dev["z"] = z if z is not None else torch.randn(b, cfg.GAN.Z_DIM, device=self.device)   # noise.normal_(0, 1)
        if eps is not None:
            dev["eps"] = eps
        out = self.net.step(dev, class_ids)
        if self.fixed_noise is not None and self.rank == 0:
            self._display = (dev, batch["captions"])      # the inputs of a display right after this step
        pred = self.inception(out["fake_imgs"][-1])
        if score is not None:
            score.add(pred)
        out.update(predictions=pred, class_ids=class_ids, keys=keys)
        return out

    @staticmethod
    def host_losses(out) -> dict:
        """The step's losses on the host, in one read (the loop reads them on print steps and at epoch ends only)."""
        names = [k for k in out if k.startswith("err") or k == "kl"]
        logs = list(out["logs"])
        vals = [out[k] for k in names if out[k] is not None] + [out["logs"][k] for k in logs]
        host = torch.stack([v.reshape(()).float() for v in vals]).tolist() if vals else []
        it = iter(host)
        res = {k: (next(it) if out[k] is not None else None) for k in names}
        res["logs"] = {k: next(it) for k in logs}
        return res

    def _log(self, epoch, gen_iterations, h):
        """The reference's per-step report (ref: trainer.py:474-476)."""
        n = len(self.net.netsPatD)
        pat = "".join("errPatD%d: %.2f " % (i, h[f"errPatD{i}"]) for i in range(n))
        shp = "".join("errShpD%d: %.2f " % (i, h[f"errShpD{i}"]) for i in range(n))
        ss = "errSSACD: %.2f " % h["errObjSSD"] if h["errObjSSD"] is not None else ""
        ls = "errObjLSD: %.2f " % h["errObjLSD"] if h["errObjLSD"] is not None else ""
        g = "".join("%s: %.2f " % (k, v) for k, v in h["logs"].items()) + "kl_loss: %.2f " % h["kl"]
        print("[%d/%d][%d]" % (epoch, self.max_epoch, gen_iterations) + "\n" + pat + "\n" + shp + "\n" + ss + "\n" +
              ls + "\n" + g)

    def epoch_score(self, score):
        """The epoch's InceptionScore over every rank's predictions: one gather to rank 0 (None on the other
        ranks).  Rank r's predictions follow rank r-1's."""
        return gather_inception_score(score, self.world, self.rank, self.pg)

    def write_score(self, epoch, score):
        """Score/scores_%d.txt in the reference's format (ref: trainer.py:495-506)."""
        mean, std, mean_conf, std_conf = score.result()
        with open(os.path.join(self.score_dir, "scores_%d.txt" % epoch), "w") as fp:
            fp.write("mean, std, mean_conf, std_conf \n")
            fp.write("%f, %f, %f, %f" % (mean, std, mean_conf, std_conf))
        print("inception_score: mean, std, mean_conf, std_conf")
        print("inception_score: %f, %f, %f, %f" % (mean, std, mean_conf, std_conf))

    def save_img_results(self, epoch, writer):
        """ref: trainer.py:275-329 and 478-484: the generator forward with the EMA weights and ``fixed_noise`` on the
        last step's inputs, in train mode (BatchNorm uses the batch statistics and updates its running buffers, which
        keep that update), the image encoder and the DAMSM word maps of the last stage; the weights are restored
        afterwards.  The PNGs go to ``writer``."""
        if self.font is None:
            if not self._warned_font:
                warnings.warn("no caption font (cfg.DATA_DIR + '%s' or font=): the attention-map PNGs are not "
                              "written" % snapshots.FONT_PATH)
                self._warned_font = True
            return
        dev, captions = self._display
        b = dev["num_rois"].shape[0]
        bucket = self.net.bG
        live = bucket.flat.clone()
        self._load_g(bucket.avg)
        try:
            with torch.no_grad():
                inp = {k: v for k, v in dev.items() if k != "eps"}
                inp["z"] = self.fixed_noise[:b]
                fake_imgs, _, att_maps, bt_att_maps, _, _ = self.net.generate(inp)
                region, _ = self.image_encoder(fake_imgs[-1])
                _, attn = ops.words_pairs(region, dev["words_embs"], dev["cap_lens"], cfg.TRAIN.SMOOTH.GAMMA1,
                                          cfg.TRAIN.SMOOTH.GAMMA2)
                idx = torch.arange(b, device=attn.device)
                word_maps = attn[idx, idx]                                # (B, T, 17, 17): caption i's own maps
        finally:
            self._load_g(live)
        jobs = []
        for i in range(len(att_maps)):
            for prefix, maps in (("G", att_maps[i]), ("bt_G", bt_att_maps[i])):
                c = snapshots.super_images(fake_imgs[i + 1], captions, self.ixtoword, maps, lr_images=fake_imgs[i],
                                           font=self.font)
                jobs.append((os.path.join(self.image_dir, "%s_average_%d_%d.png" % (prefix, epoch, i)), c))
        c = snapshots.super_images(fake_imgs[-1], captions, self.ixtoword, word_maps, lens=dev["cap_lens"],
                                   font=self.font)
        jobs.append((os.path.join(self.image_dir, "D_average_%d.png" % epoch), c))
        writer.submit(jobs)

    def _load_g(self, weights):
        """Copies ``weights`` into the generator's flat parameters and re-packs their tensor-core operand copies."""
        bucket = self.net.bG
        bucket.flat.copy_(weights)
        bucket.epoch[0] += 1
        bucket.plan.run()

    def train(self):
        """ref: trainer.py:331-511."""
        start_epoch = self.setup()
        with snapshots.writing(snapshots.PngWriter() if self.rank == 0 else None) as writer:
            self._train(start_epoch, writer)

    def _train(self, start_epoch, writer):
        gen_iterations = 0
        lead = self.rank == 0
        for epoch in range(start_epoch, self.max_epoch):
            start_t = time.time()
            score = losses.InceptionScore(min(10, self.batch_size))
            data_iter = iter(self.data_loader)
            out = None
            for _ in range(self.num_batches):
                out = self.train_step(next(data_iter), score)
                gen_iterations += 1
                if gen_iterations % self.print_interval == 0 and lead:
                    self._log(epoch, gen_iterations, self.host_losses(out))
                if gen_iterations % self.display_interval == 0 and lead:
                    self.save_img_results(epoch, writer)
            if out is None:
                continue
            h = self.host_losses(out)
            end_t = time.time()
            n = len(self.net.netsPatD)
            zero = lambda v: 0.0 if v is None else v
            if lead:
                print("[%d/%d][%d]\n                  Loss_PatD: %.2f Loss_ShpD: %.2f Loss_ObjSSD: %.2f Loss_ObjLSD: %.2f "
                      "Loss_G: %.2f Time: %.2fs"
                      % (epoch, self.max_epoch, self.num_batches, sum(h[f"errPatD{i}"] for i in range(n)),
                         sum(h[f"errShpD{i}"] for i in range(n)), zero(h["errObjSSD"]), zero(h["errObjLSD"]),
                         h["errG"] + h["kl"], end_t - start_t))
            score = self.epoch_score(score)
            if lead:
                self.write_score(epoch, score)
                if epoch % self.snapshot_interval == 0:
                    self.net.save_model(self.model_dir, epoch)
        if lead:
            self.net.save_model(self.model_dir, self.max_epoch)
