"""Sampling from a trained generator: the reference's evaluator path (ref: evaluator.py:108-138 builds G_NET, calls
``netG.eval()`` and loads ``netG_epoch_N.pth``; evaluator.py:312 draws the noise) on the sm_90a kernels.

``GSampler`` holds its own G_NET in eval mode, so BatchNorm normalises with the running statistics and never updates
them.  A forward pass is ~200 library calls, which cost far more host time than the kernels take at small batch, so
every input shape is captured once into a CUDA graph and replayed after that:

  * graphs are keyed by (B, L, Rmax, glb_max_num_roi): batch, caption length, roi slots of ``slabels_feat`` and the
    roi width of the returned ``bt_c_code``.  Rmax is NOT padded to BOXES_NUM to share one graph: the bottom-up paint
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
from . import model
from .config import cfg
from .trainer import prepare_data

# what G_NET.forward reads, in its argument order (ref: model.py:747)
G_ARGS = ("z", "sent_emb", "words_embs", "glove_words_embs", "slabels_feat", "mask", "hmaps", "rois", "fm_rois",
          "num_rois", "bt_masks", "fm_bt_masks", "glb_max_num_roi")


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

    def __init__(self, netG: model.G_NET):
        self.netG = netG.eval()
        for p in self.netG.parameters():
            p.requires_grad_(False)
        self.device = next(self.netG.parameters()).device
        self._graphs = {}
        self._pool = None

    @classmethod
    def from_snapshot(cls, path: str, num_classes: int = 80, device="cuda") -> "GSampler":
        """A reference-format generator snapshot (``netG_epoch_N.pth``, what StepBTrainer.save_model writes)."""
        s = cls(_new_g(num_classes, device))
        s.load_state_dict(torch.load(path, map_location="cpu"))
        return s

    @classmethod
    def from_trainer(cls, trainer) -> "GSampler":
        """The trainer's EMA generator weights (what the reference snapshots); the trainer is not modified."""
        s = cls(_new_g(trainer.netG.num_classes, trainer.device))
        s.load_state_dict(trainer.bG.ema_state_dict())
        return s

    def load_state_dict(self, state_dict: dict) -> None:
        """Loads G weights (strict) and drops every captured graph."""
        self._graphs.clear()
        self.netG.load_state_dict({k: v.to(self.device) for k, v in state_dict.items()}, strict=True)

    # ------------------------------------------------------------------ inputs
    def _prepare(self, inp: dict) -> dict:
        """Device copies of the inputs G_NET reads (+ the derived tensors of a compact batch), with z and the CA_NET
        noise drawn here, outside any graph, when the batch does not bring them."""
        dev = {}
        for k, v in inp.items():
            dev[k] = _map(v, lambda t: t.to(self.device, non_blocking=True))
        if "hmaps" not in dev and "roi_cls" in dev:
            prepare_data(dev, self.netG.num_classes)
        b = dev["sent_emb"].shape[0]
        if dev.get("z") is None:
            dev["z"] = torch.randn(b, cfg.GAN.Z_DIM, device=self.device)      # noise_img.data.normal_(0, 1)
        if dev.get("eps") is None:
            dev["eps"] = torch.randn(b, cfg.GAN.CONDITION_DIM, device=self.device)   # CA_NET.reparametrize
        return {k: dev[k] for k in (*G_ARGS, "eps")}

    @staticmethod
    def _key(dev: dict) -> tuple:
        return (dev["z"].shape[0], dev["words_embs"].shape[2], dev["slabels_feat"].shape[2],
                int(dev["glb_max_num_roi"]))

    def _forward(self, dev: dict):
        g = self.netG
        g.ca_net.eps_override = dev["eps"]
        try:
            return g(*(dev[k] for k in G_ARGS))
        finally:
            g.ca_net.eps_override = None

    # ------------------------------------------------------------------ sampling
    def sample_eager(self, inp: dict):
        """The same forward pass without graphs."""
        with torch.no_grad():
            return self._forward(self._prepare(inp))

    def sample(self, inp: dict):
        """fake_imgs, bt_c_codes, att_maps, bt_att_maps, mu, logvar for the batch ``inp`` (the input dict of
        StepATrainer.generate, full or compact); z / eps are taken from it when present."""
        with torch.no_grad():
            dev = self._prepare(inp)
            key = self._key(dev)
            entry = self._graphs.get(key)
            if entry is None:
                out = self._forward(dev)          # warm-up: packed weights, allocator state
                self._graphs[key] = self._capture(dev)
                return out
            for k in G_ARGS + ("eps",):
                if k != "glb_max_num_roi":
                    _copy_into(entry.static_in[k], dev[k])
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
        return _Graph(graph, static_in, static_out, launches, _packed_copies(self.netG))


def _new_g(num_classes, device):
    # the constructor's initialisation is overwritten by the load that follows: skip the per-weight QR of the
    # orthogonal initialisation
    fast, model.FAST_INIT = model.FAST_INIT, True
    try:
        return model.G_NET(num_classes).to(device)
    finally:
        model.FAST_INIT = fast


def _packed_copies(net):
    """Every kernel-native weight copy the network's layers hold right now (kept alive by a graph that read them)."""
    keep = []
    for m in net.modules():
        c = getattr(m, "_cache", None)
        if c is not None:
            keep.append((c.f, c.t, dict(c.hl), c.amax))
    return keep


def _clone_out(out):
    fake, btc, att, btatt, mu, logvar = out
    cl = lambda ts: [t.clone() for t in ts]
    return cl(fake), cl(btc), cl(att), cl(btatt), mu.clone(), logvar.clone()
