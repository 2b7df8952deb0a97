"""The box generator of caption-to-image sampling: caption -> PreEncoderRNN -> DecoderRNN samples -> layout, the
reference's box_generation/sample.py + Evaluator.evaluate + image_generation/miscc/load.py:load_gen_insanns, on the
device and without files in between.

``Evaluator`` is the other way: a drop-in for the reference's box_generation Evaluator that writes the layout files
(``<folder><key>/<caption index>/boxes.txt``, or ``dev_bbox_test.txt``) for a whole test split, a chunk of captions per
launch, with the files written on a background thread while the device runs the next chunk.

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
import queue
import re
import threading
import time
import types
import warnings

import numpy as np
import torch
import torch.distributed as dist
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


# ---------------------------------------------------------------------------------------------------------------------
# The reference's test split (box_generation/seq2seq/dataset/prepare_dataset.py:81-244), without nltk
# ---------------------------------------------------------------------------------------------------------------------
SPECIAL_LABELS = ("<pad>", "<sos>", "<eos>", "<unk>")


def normalize_string(s: str) -> list:
    """normalize_string (prepare_dataset.py:81-91): '��' -> ' ', lower-case, the tokens of ``\\w+`` (what
    nltk's RegexpTokenizer(r'\\w+') returns), each with its non-ASCII characters removed; empty tokens dropped."""
    tokens = re.findall(r"\w+", s.replace("��", " ").lower())
    return [t for t in (t.encode("ascii", "ignore").decode("ascii") for t in tokens) if t]


def indexes_from_sentence(word2index, words) -> list:
    """indexes_from_sentence (prepare_dataset.py:221-235): the known words' indexes, with <sos> / <eos> around them
    only if the vocabulary has them; unknown words are dropped."""
    seq = [word2index["<sos>"]] if "<sos>" in word2index else []
    seq += [word2index[w] for w in words if w in word2index]
    if "<eos>" in word2index:
        seq.append(word2index["<eos>"])
    return seq


def _lines(path):
    with open(path) as f:
        return f.read().strip().split("\n")


def read_test_tuples(dev_path) -> list:
    """read_langs (prepare_dataset.py:93-113): one [tokens, x, y, w, h, labels] tuple per line of six tab-separated
    fields, the caption normalised.  A line with another field count raises ValueError naming it."""
    tuples = []
    for i, line in enumerate(_lines(dev_path)):
        f = line.split("\t")
        if len(f) != 6:
            raise ValueError(f"{dev_path} line {i + 1}: {len(f)} tab-separated fields, the test split has 6: "
                             f"{line[:80]!r}")
        tuples.append([normalize_string(f[0]), *f[1:]])
    return tuples


def read_keys(dev_filename_path) -> list:
    """The image key of each caption line (filenames_val2014.txt, one per line)."""
    return _lines(dev_filename_path)


def load_cap_vocab(checkpoint_dir):
    """(cap_word2index, cap_index2word) of a box checkpoint (seq2seq/util/checkpoint.py:83-86), read through the
    restricted unpickler in either pickle format."""
    return (_restricted_load(os.path.join(checkpoint_dir, "cap_word2index.pt")),
            _restricted_load(os.path.join(checkpoint_dir, "cap_index2word.pt")))


def caption_indices(keys) -> list:
    """The caption index of every tuple: how many earlier tuples have its key, in file order (evaluator.py:48-52,
    87-89).  Computed from the full key list, so a shard's numbering is the one-process numbering."""
    seen = collections.Counter()
    out = []
    for k in keys:
        out.append(seen[k])
        seen[k] += 1
    return out


def caption_sequences(data, keys, word2index) -> list:
    """Every tuple's caption as token indexes, after checking the split: one key per tuple, and no caption that maps to
    no token (the reference's encoder fails on it).  Raises ValueError naming the first offending line."""
    if len(keys) != len(data):
        raise ValueError(f"{len(keys)} image keys for {len(data)} captions: the key file must have one line per "
                         f"caption line")
    seqs = []
    for i, item in enumerate(data):
        seq = indexes_from_sentence(word2index, item[0])
        if not seq:
            raise ValueError(f"caption line {i + 1} ({' '.join(item[0])!r}, key {keys[i]}) has no word of the caption "
                             f"vocabulary")
        seqs.append(seq)
    return seqs


def box_rows_text(rows, names) -> str:
    """A boxes.txt: one '%.2f,%.2f,%.2f,%.2f,<category id>,0' line per row (evaluator.py:137-139)."""
    return "".join("%.2f,%.2f,%.2f,%.2f,%s,0\n" % (x, y, w, h, names[c]) for (x, y, w, h), c in rows)


def dev_bbox_line(key, words, rows, names) -> str:
    """A dev_bbox_test.txt line (evaluator.py:142-149)."""
    return "%s - %s - " % (key, words) + "".join("%.2f,%.2f,%.2f,%.2f,%s - " % (x, y, w, h, names[c])
                                                for (x, y, w, h), c in rows) + "\n"


class _FileWriter:
    """Writes the files of each chunk on one background thread.  ``submit`` takes a job (its arrays may still be on
    their way from the device: the job's event is waited on first) and blocks while two earlier chunks are queued; an
    error of the writer is raised by the next ``submit`` or by ``close``.  The dev_bbox_test.txt lines are kept in
    ``lines`` for the caller to write."""

    def __init__(self, write):
        self._write = write
        self._q = queue.Queue(maxsize=2)
        self._thread = threading.Thread(target=self._run, name="box-files", daemon=True)
        self._error = None
        self._thread.start()

    def _raise(self):
        if self._error is not None:
            err, self._error = self._error, None
            raise RuntimeError("writing the box layout files failed") from err

    def _run(self):
        while True:
            job = self._q.get()
            try:
                if job is None:
                    return
                if self._error is None:
                    self._write(*job)
            except BaseException as e:      # surfaced on the caller's thread
                self._error = e
            finally:
                self._q.task_done()

    def submit(self, *job):
        self._raise()
        self._q.put(job)

    def close(self, raise_error=True):
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None
        if raise_error:
            self._raise()


def _library_modules(encoder, decoder, label_word2index):
    """This library's PreEncoderRNN / DecoderRNN for the given modules: as they are, or loaded from the state_dict of
    the reference's (whose keys and shapes are the same)."""
    if not isinstance(encoder, model.PreEncoderRNN):
        sd = {k: v.detach().cpu() for k, v in encoder.state_dict().items()}
        enc = model.PreEncoderRNN(sd["encoder.weight"].shape[0], ninput=sd["encoder.weight"].shape[1], nhidden=256)
        enc.load_state_dict(sd, strict=True)
        encoder = enc
    if not isinstance(decoder, model.DecoderRNN):
        sd = {k: v.detach().cpu() for k, v in decoder.state_dict().items()}
        dec = model.DecoderRNN(label_word2index, decoder.x_mean, decoder.y_mean, decoder.w_mean, decoder.r_mean, 1,
                               getattr(decoder, "max_length", 150), decoder.hidden_size, decoder.gmm_comp_num,
                               n_layers=getattr(decoder, "n_layers", 1),
                               rnn_cell="gru" if "GRU" in str(getattr(decoder, "rnn_cell", "lstm")) else "lstm",
                               bidirectional=decoder.bidirectional_encoder,
                               use_attention=getattr(decoder, "use_attention", False))
        dec.load_state_dict(sd, strict=True)
        decoder = dec
    return encoder, decoder


class Evaluator:
    """Drop-in for the reference's box_generation Evaluator (seq2seq/evaluator/evaluator.py): the same constructor, and
    ``evaluate(encoder, decoder, data, keys)`` writes the same files -- with ``output_opt`` 0 one
    ``box_saving_folder + key + '/<j>/boxes.txt'`` per tuple (j: the tuple's caption index among those of its key), with
    1 ``expt_dir/dev_bbox_test.txt`` -- running ``chunk`` captions per launch on the device.

    ``batch_size`` must be 1: every tuple is evaluated once, in file order (the reference's loop at a larger batch runs
    only the first len / batch_size tuples).  The noise of tuple i depends only on (``seed``, i) (og_box_noise), so the
    files do not depend on ``chunk`` or on the number of ranks; it is not numpy's draw sequence.  Under torchrun with an
    initialised process group every rank writes the boxes.txt files of its own contiguous share of the tuples, and rank
    0 writes dev_bbox_test.txt from the rows of all.  A box whose label is a special token (where the reference raises)
    is dropped, with one warning giving the number of captions affected."""

    def __init__(self, batch_size, early_stop_len, expt_dir, dev_cap_lang, dev_label_lang, x_mean_std, y_mean_std,
                 w_mean_std, r_mean_std, gaussian_dict, box_saving_folder, output_opt, *, chunk: int = 1024,
                 seed: int = 0, device=None, process_group=None):
        if batch_size != 1:
            raise ValueError(f"batch_size must be 1 (every tuple once, in file order); got {batch_size}.  The captions "
                             f"per launch are set by chunk=")
        if output_opt not in (0, 1):
            raise ValueError(f"output_opt must be 0 (boxes.txt per caption) or 1 (dev_bbox_test.txt), got {output_opt}")
        if int(chunk) < 1:
            raise ValueError(f"chunk must be >= 1, got {chunk}")
        self.batch_size, self.early_stop_len, self.expt_dir = batch_size, int(early_stop_len), expt_dir
        self.dev_cap_lang, self.dev_label_lang = dev_cap_lang, dev_label_lang
        self.mean_std = np.array([x_mean_std, y_mean_std, w_mean_std, r_mean_std], dtype=np.float64).reshape(4, 2)
        self.gaussian_dict = gaussian_dict
        self.box_saving_folder, self.output_opt = box_saving_folder, output_opt
        self.display_step = 200
        self.chunk, self.seed = int(chunk), int(seed)
        self.device = torch.device(device) if device is not None else \
            torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        # class rows: the category ids of the label vocabulary in index order; the special tokens have none
        i2w = dev_label_lang.index2word
        self.label_to_class, self.class_names, stats = [], [], []
        for i in range(len(i2w)):
            w = i2w[i]
            if w in SPECIAL_LABELS:
                self.label_to_class.append(-1)
                continue
            cid = int(w)
            if cid not in gaussian_dict:
                raise ValueError(f"gaussian_dict has no statistics for category id {cid} (label {i})")
            self.label_to_class.append(len(self.class_names))
            self.class_names.append(str(cid))
            stats.append([float(gaussian_dict[cid][0]), float(gaussian_dict[cid][1])])
        self.count_stats = stats

    @classmethod
    def from_reference(cls, checkpoint_dir: str, text_snapshot: str, dev_path: str, dev_filename_path: str, mean_std,
                       gaussian_dict, box_saving_folder: str, output_opt: int, expt_dir: str = "experiment",
                       early_stop_len: int = 10, **kw) -> "Evaluator":
        """The evaluator of the reference's sample.py --is_training 0, from its files alone: a box checkpoint directory
        (model.pt, the cap_* / label_* vocabularies), the text encoder snapshot, the test split (dev_path, its keys in
        dev_filename_path), mean_std_train2014.txt (or its (4, 2) table) and gaussian_dict.npy (or the dict).  Call
        ``evaluate()`` with no arguments to write the files of that split."""
        cap_w2i, cap_i2w = load_cap_vocab(checkpoint_dir)
        label_i2w = _restricted_load(os.path.join(checkpoint_dir, "label_index2word.pt"))
        label_w2i = {w: i for i, w in label_i2w.items()}
        ms = np.loadtxt(mean_std) if isinstance(mean_std, (str, os.PathLike)) else np.asarray(mean_std)
        ms = np.asarray(ms, dtype=np.float64).reshape(4, 2)
        gd = np.load(gaussian_dict, allow_pickle=True).item() if isinstance(gaussian_dict, (str, os.PathLike)) \
            else gaussian_dict
        ev = cls(1, early_stop_len, expt_dir, types.SimpleNamespace(word2index=cap_w2i, index2word=cap_i2w),
                 types.SimpleNamespace(word2index=label_w2i, index2word=label_i2w), *[tuple(r) for r in ms], gd,
                 box_saving_folder, output_opt, **kw)
        data = read_test_tuples(dev_path)
        keys = read_keys(dev_filename_path)
        caption_sequences(data, keys, cap_w2i)            # refuse a bad split before loading any weights
        from .sampler import strip_module_prefix
        text_sd = strip_module_prefix(torch.load(text_snapshot, map_location="cpu"))
        enc = model.PreEncoderRNN(text_sd["encoder.weight"].shape[0], ninput=text_sd["encoder.weight"].shape[1],
                                  nhidden=256)
        enc.load_state_dict(text_sd, strict=True)
        dec = load_reference_decoder(os.path.join(checkpoint_dir, "model.pt"))
        ev._split = (enc, dec, data, keys)
        return ev

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, encoder=None, decoder=None, data=None, keys=None):
        """Writes the files of every tuple of ``data`` (the reference's dev_tuples: [caption tokens, x, y, w, h,
        labels]) with ``keys`` its image keys, and returns when every file is closed.  With from_reference, the
        arguments default to the files it read."""
        if encoder is None:
            encoder, decoder, data, keys = self._split
        seqs = caption_sequences(data, keys, self.dev_cap_lang.word2index)
        jidx = caption_indices(keys)
        enc, dec = _library_modules(encoder, decoder, self.dev_label_lang.word2index)
        self.generator = BoxGenerator(enc.to(self.device), dec.to(self.device), self.mean_std, self.count_stats,
                                      self.label_to_class, self.early_stop_len)
        n = len(seqs)
        lo, hi = n * self.rank // self.world, n * (self.rank + 1) // self.world
        i2w = self.dev_cap_lang.index2word
        lines, affected = [], [0]

        busy = [0.0]

        def write(start, host, event):
            if event is not None:
                event.synchronize()
            t0 = time.perf_counter()
            b, s = len(host) // (5 * self.early_stop_len + 3), self.early_stop_len
            rows, cls, n_rows, n_valid, n_special = (t.numpy() for t in ops.unpack_box_records(host, b, s))
            rows, cls = rows.tolist(), cls.tolist()
            n_rows, n_valid = n_rows.tolist(), n_valid.tolist()
            affected[0] += int((n_special > 0).sum())
            for q in range(b):
                i = start + q
                r = list(zip(rows[q][:n_rows[q]], cls[q][:n_rows[q]]))
                if self.output_opt == 0:
                    d = self.box_saving_folder + keys[i] + "/%d/" % jidx[i]
                    os.makedirs(d, exist_ok=True)
                    with open(d + "boxes.txt", "w") as f:
                        f.write(box_rows_text(r, self.class_names))
                elif n_valid[q] > 1:
                    lines.append(dev_bbox_line(keys[i], [i2w[w] for w in seqs[i]], r, self.class_names))
            busy[0] += time.perf_counter() - t0

        writer = _FileWriter(write)
        try:
            with torch.no_grad():
                for start in range(lo, hi, self.chunk):
                    stop = min(start + self.chunk, hi)
                    packed = self._device_records(start, seqs[start:stop])
                    if packed.is_cuda:
                        host = torch.empty(packed.shape, dtype=packed.dtype, pin_memory=True)
                        host.copy_(packed, non_blocking=True)
                        event = torch.cuda.Event()
                        event.record()
                    else:
                        host, event = packed, None
                    writer.submit(start, host, event)
                    if self.rank == 0:
                        for d in range((start - lo) * self.world, (stop - lo) * self.world):
                            if (d + 1) % self.display_step == 0 and d < n:
                                print("%07d / %07d" % (d, n))
        except BaseException:
            writer.close(raise_error=False)
            raise
        writer.close()
        t0 = time.perf_counter()
        self._finish(lines, affected[0])
        self.write_seconds = busy[0] + time.perf_counter() - t0      # this rank's time formatting and writing files

    def _device_records(self, start, seqs):
        """The packed og_box_records buffer of tuples start .. start + len(seqs) - 1: encoder state, decoder, rows --
        six library calls whatever the caption lengths."""
        bg, b = self.generator, len(seqs)
        width = max(len(q) for q in seqs)
        caps = np.zeros((b, width), dtype=np.int64)
        for q, seq in enumerate(seqs):
            caps[q, :len(seq)] = seq
        caps = torch.from_numpy(caps).to(self.device, non_blocking=True)
        lens = torch.tensor([len(q) for q in seqs], dtype=torch.int64).to(self.device, non_blocking=True)
        nb, nc = ops.box_noise(self.seed, start, b, self.early_stop_len, bg.num_classes, self.device)
        _, h, c = bg.encoder.encode_state(caps, lens, width)
        labels, samples, steps, _ = bg.decoder.sample_state(h, c, nb, self.early_stop_len)
        return ops.box_records_packed(labels, samples, steps, bg.mean_std, bg.label_to_class, bg.count_stats, nc)

    def _finish(self, lines, affected):
        if self.world > 1:
            got = [None] * self.world if self.rank == 0 else None
            dist.gather_object((lines, affected), got, dst=0, group=self.pg)
            if self.rank == 0:
                lines = [ln for part, _ in got for ln in part]
                affected = sum(a for _, a in got)
        if self.rank == 0:
            if self.output_opt == 1:
                with open("%s/dev_bbox_test.txt" % self.expt_dir, "w") as f:
                    f.writelines(lines)
            if affected:
                warnings.warn(f"{affected} captions sampled a box with a special label (<pad>, <sos> or <unk>); the "
                              f"reference raises on these, here the boxes were dropped")
        if self.world > 1:
            dist.barrier(group=self.pg)                  # every rank's files are closed before any rank returns
