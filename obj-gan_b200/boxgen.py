"""The box generator of caption-to-image sampling: caption -> PreEncoderRNN -> DecoderRNN samples -> layout, the
reference's box_generation/sample.py + Evaluator.evaluate + image_generation/miscc/load.py:load_gen_insanns, on the
device and without files in between.

``BoxGenerator.from_reference`` reads the reference's own files.  Its decoder checkpoint (``model.pt``) is a whole
pickled ``DecoderRNN``; it is read with an unpickler that maps the ``seq2seq.*`` classes to inert stubs, allows only
the globals a module pickle needs, and raises on anything else, so loading it imports and runs none of the reference's
code.
"""
from __future__ import annotations

import collections
import io
import os
import pickle
import types

import numpy as np
import torch
import torch.nn.backends.thnn

from . import model, ops
from .config import cfg

NOISE_BOX = ops.BOX_NOISE


class BoxGenerator:
    """``BoxGenerator(encoder, decoder, mean_std, count_stats, label_to_class, early_stop_len=10)``:
    ``mean_std`` (4, 2) the (mean, std) of x, y, w and the aspect ratio r (mean_std_train2014.txt); ``count_stats``
    (num_classes, 2) the (mu, sigma) of each class's box count (gaussian_dict.npy, rows in categories.txt order);
    ``label_to_class`` (n_labels,) the class row of each decoder label, -1 for the special tokens."""

    def __init__(self, encoder: model.PreEncoderRNN, decoder: model.DecoderRNN, mean_std, count_stats, label_to_class,
                 early_stop_len: int = 10):
        n_labels = decoder.l_output_size
        mean_std = torch.as_tensor(mean_std, dtype=torch.float64)
        count_stats = torch.as_tensor(count_stats, dtype=torch.float64)
        label_to_class = torch.as_tensor(label_to_class, dtype=torch.int64)
        if not 1 <= int(early_stop_len) <= cfg.ROI.BOXES_NUM + 1:
            raise ValueError(f"early_stop_len must lie in [1, {cfg.ROI.BOXES_NUM + 1}] (BOXES_NUM + 1), got "
                             f"{early_stop_len}")
        if mean_std.shape != (4, 2) or not torch.isfinite(mean_std).all():
            raise ValueError("mean_std must be a finite (4, 2) table of (mean, std) for x, y, w, r")
        if count_stats.dim() != 2 or count_stats.shape[1] != 2 or count_stats.shape[0] < 1 or \
                not torch.isfinite(count_stats).all():
            raise ValueError("count_stats must be a finite (num_classes, 2) table of (mu, sigma), one row per class")
        if label_to_class.shape != (n_labels,):
            raise ValueError(f"label_to_class must have one entry per decoder label ({n_labels})")
        nc = count_stats.shape[0]
        if bool(((label_to_class < -1) | (label_to_class >= nc)).any()):
            raise ValueError(f"label_to_class points outside the {nc} classes of count_stats")
        for tok in ("<pad>", "<sos>", "<eos>", "<unk>"):
            if tok in decoder.l_word2index and int(label_to_class[decoder.l_word2index[tok]]) != -1:
                raise ValueError(f"label_to_class must map the special token {tok} to -1")
        self.encoder = encoder.eval()
        self.decoder = decoder.eval()
        for net in (self.encoder, self.decoder):
            for p in net.parameters():
                p.requires_grad_(False)
        self.device = next(self.decoder.parameters()).device
        self.mean_std = mean_std.to(self.device)
        self.count_stats = count_stats.to(self.device)
        self.label_to_class = label_to_class.to(self.device)
        self.early_stop_len = int(early_stop_len)
        self.num_classes = nc

    def to(self, device):
        self.encoder.to(device)
        self.decoder.to(device)
        self.device = torch.device(device)
        self.mean_std, self.count_stats = self.mean_std.to(device), self.count_stats.to(device)
        self.label_to_class = self.label_to_class.to(device)
        return self

    # ------------------------------------------------------------------ sampling
    def draw_noise(self, b: int) -> tuple:
        """(noise_box (B, early_stop_len, 6), noise_cnt (B, num_classes)): per step the uniforms of the two component
        choices at columns 0 and 3 and four standard normals; one standard normal per sample and class for the count
        thresholds."""
        s = self.early_stop_len
        nb = torch.randn(b, s, NOISE_BOX, device=self.device)
        nb[:, :, 0::3] = torch.rand(b, s, 2, device=self.device)
        return nb, torch.randn(b, self.num_classes, device=self.device)

    def sample(self, captions, cap_lens, max_len: int, noise_box, noise_cnt) -> dict:
        """captions (B, >= max_len) int64, cap_lens (B,) in [1, max_len] (device tensors; not read on the host) ->
        the layout (``rois`` (3 scales), ``fm_rois``, ``roi_cls``, ``num_rois``) and the raw trajectory (``labels``,
        ``samples``, ``steps``).  Five library calls whatever B and max_len."""
        _, h, c = self.encoder.encode_state(captions, cap_lens, max_len)
        labels, samples, steps, _ = self.decoder.sample_state(h, c, noise_box, self.early_stop_len)
        rois, fm_rois, roi_cls, num_rois = ops.boxes_to_layout(
            labels, samples, steps, self.mean_std, self.label_to_class, self.count_stats, noise_cnt,
            cfg.ROI.BOXES_NUM, cfg.ROI.ROI_MIN_SIZE)
        return dict(rois=rois, fm_rois=fm_rois, roi_cls=roi_cls, num_rois=num_rois, labels=labels, samples=samples,
                    steps=steps)

    # ------------------------------------------------------------------ the reference's files
    @classmethod
    def from_reference(cls, checkpoint_dir: str, text_snapshot: str, mean_std, gaussian_dict, cat_ids,
                       early_stop_len: int = 10, device="cuda") -> "BoxGenerator":
        """``checkpoint_dir``: a box checkpoint directory (``checkpoints/<name>/`` with ``model.pt`` and
        ``label_index2word.pt``, seq2seq/util/checkpoint.py); ``text_snapshot``: the text encoder the reference's
        sample.py loads into PreEncoderRNN (text_encoder100.pth); ``mean_std``: mean_std_train2014.txt or its (4, 2)
        table; ``gaussian_dict``: gaussian_dict.npy or its {category id: (mu, sigma)}; ``cat_ids``: the COCO category
        ids in categories.txt order (the class rows)."""
        dec = load_reference_decoder(os.path.join(checkpoint_dir, "model.pt"))
        index2word = _restricted_load(os.path.join(checkpoint_dir, "label_index2word.pt"))
        from .sampler import strip_module_prefix
        text_sd = strip_module_prefix(torch.load(text_snapshot, map_location="cpu"))
        enc = model.PreEncoderRNN(text_sd["encoder.weight"].shape[0], nhidden=256)
        enc.load_state_dict(text_sd, strict=True)
        ms = np.loadtxt(mean_std) if isinstance(mean_std, (str, os.PathLike)) else np.asarray(mean_std)
        gd = np.load(gaussian_dict, allow_pickle=True).item() if isinstance(gaussian_dict, (str, os.PathLike)) \
            else gaussian_dict
        cat_ids = [int(c) for c in cat_ids]
        row = {c: i for i, c in enumerate(cat_ids)}
        missing = [c for c in cat_ids if c not in gd]
        if missing:
            raise ValueError(f"gaussian_dict has no statistics for the category ids {missing}")
        stats = [[float(gd[c][0]), float(gd[c][1])] for c in cat_ids]
        l2c = []
        for i in range(dec.l_output_size):
            w = index2word[i]
            if w in ("<pad>", "<sos>", "<eos>", "<unk>"):
                l2c.append(-1)
            elif int(w) in row:
                l2c.append(row[int(w)])
            else:
                raise ValueError(f"decoder label {i} is category id {w}, which is not in cat_ids")
        return cls(enc.to(device), dec.to(device), np.asarray(ms, dtype=np.float64).reshape(4, 2), stats, l2c,
                   early_stop_len)


# ---------------------------------------------------------------------------------------------------------------------
# Loading the reference's pickled DecoderRNN without its code
# ---------------------------------------------------------------------------------------------------------------------
class _Stub:
    """Inert stand-in for a pickled seq2seq.* object: keeps its state and does nothing else."""

    def __setstate__(self, state):
        self.__dict__["_state"] = state


_STUB_MODULES = ("seq2seq.models.DecoderRNN", "seq2seq.models.baseRNN", "seq2seq.models.attention")
_ALLOWED = {
    ("collections", "OrderedDict"): collections.OrderedDict,
    ("torch._utils", "_rebuild_tensor_v2"): torch._utils._rebuild_tensor_v2,
    ("torch._utils", "_rebuild_parameter"): torch._utils._rebuild_parameter,
    ("torch._utils", "_rebuild_parameter_with_state"): getattr(torch._utils, "_rebuild_parameter_with_state", None),
    ("torch", "Size"): torch.Size,
    # torch 0.4 (the reference's pin) pickles a Parameter as Parameter(tensor, requires_grad) and every module's
    # _backend through this function, which current torch keeps as a no-op for old pickles
    ("torch.nn.parameter", "Parameter"): torch.nn.parameter.Parameter,
    ("torch.nn.backends.thnn", "_get_thnn_function_backend"): torch.nn.backends.thnn._get_thnn_function_backend,
    ("torch.nn.functional", "log_softmax"): torch.nn.functional.log_softmax,
    ("torch.distributions.normal", "Normal"): torch.distributions.normal.Normal,
    ("numpy", "dtype"): np.dtype,
    ("builtins", "set"): set, ("__builtin__", "set"): set,     # protocol-2 pickles name builtins __builtin__
    ("builtins", "frozenset"): frozenset, ("__builtin__", "frozenset"): frozenset,
}
for _n in ("Float", "Double", "Half", "Long", "Int", "Byte", "Bool"):
    _ALLOWED[("torch", _n + "Storage")] = getattr(torch, _n + "Storage")


_STUBS = {}


def _stub(module, name):
    """One inert class per pickled global: it keeps the pickled state and runs none of the class's code (a module
    pickled by an older torch need not match the current class's __setstate__)."""
    if (module, name) not in _STUBS:
        _STUBS[(module, name)] = type(name, (_Stub,), {"__module__": "objgan_b200.boxgen.stub"})
    return _STUBS[(module, name)]


def _allowed(module, name):
    if module.startswith("seq2seq."):
        if module in _STUB_MODULES:
            return _stub(module, name)
        raise pickle.UnpicklingError(f"refusing to load the global {module}.{name}")
    if module.startswith("torch.nn.modules.") and not name.startswith("_"):
        import importlib
        obj = getattr(importlib.import_module(module), name, None)
        if isinstance(obj, type) and issubclass(obj, torch.nn.Module):
            return _stub(module, name)
    if module in ("numpy.core.multiarray", "numpy._core.multiarray") and name == "scalar":
        import importlib
        return importlib.import_module("numpy._core.multiarray").scalar
    obj = _ALLOWED.get((module, name))
    if obj is None:
        raise pickle.UnpicklingError(f"refusing to load the global {module}.{name}")
    return obj


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        return _allowed(module, name)


_pickle_module = types.SimpleNamespace(Unpickler=_Unpickler, load=lambda f, **kw: _Unpickler(f, **kw).load(),
                                       __name__="objgan_b200.boxgen.restricted_pickle")
_LEGACY_MAGIC = 0x1950a86a20f9469cfc6c      # the first pickle of torch's legacy (pre-zip) format


def _restricted_load(path):
    """torch.load of a zip-format or legacy-format file through the restricted unpickler, or a plain pickle (such as
    the dill-written vocabularies)."""
    with open(path, "rb") as f:
        data = f.read()
    if data[:2] != b"PK":
        first = _Unpickler(io.BytesIO(data)).load()
        if not (isinstance(first, int) and first == _LEGACY_MAGIC):
            return first
    return torch.load(io.BytesIO(data), map_location="cpu", pickle_module=_pickle_module, weights_only=False)


def _state(obj):
    return obj.__dict__["_state"] if isinstance(obj, _Stub) else obj.__dict__


def load_reference_decoder(path: str) -> model.DecoderRNN:
    """The reference's ``torch.save(decoder)`` (checkpoint.py:91) as this library's DecoderRNN, in eval mode."""
    obj = _restricted_load(path)
    if not isinstance(obj, _Stub) or type(obj).__name__ != "DecoderRNN":
        raise ValueError(f"{path} does not hold a pickled DecoderRNN")
    st = _state(obj)
    sd = collections.OrderedDict()

    def walk(prefix, mod):
        s = _state(mod)
        for k, v in s.get("_parameters", {}).items():
            if v is not None:
                sd[prefix + k] = v.detach()
        for k, v in s.get("_buffers", {}).items():
            if v is not None:
                sd[prefix + k] = v
        for k, m in s.get("_modules", {}).items():
            if m is not None:
                walk(prefix + k + ".", m)
    walk("", obj)
    n = st["l_output_size"]
    names = {i: f"_{i}" for i in range(n)}
    names[st["l_sos_id"]], names[st["l_eos_id"]] = "<sos>", "<eos>"
    word2index = {names[i]: i for i in range(n)}
    rnn = _state(st["_modules"]["rnn"])
    cell = "gru" if type(st["_modules"]["rnn"]).__name__ == "GRU" else "lstm"
    dec = model.DecoderRNN(word2index, st["x_mean"], st["y_mean"], st["w_mean"], st["r_mean"], st["batch_size"],
                           st["max_length"], st["hidden_size"], st["gmm_comp_num"], n_layers=rnn.get("num_layers", 1),
                           rnn_cell=cell, bidirectional=st["bidirectional_encoder"],
                           input_dropout_p=st.get("input_dropout_p", 0), dropout_p=st.get("dropout_p", 0),
                           use_attention=st["use_attention"])
    dec.load_state_dict(sd, strict=True)
    return dec.eval()
