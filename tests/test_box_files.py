"""Writing the box generator's layout files for a test split (CPU): the rows and texts of the restatement
(tests/box_files_oracle.py) against the reference's own Evaluator output, the intake of the reference's test files,
the caption numbering, the vocabulary loader, boxgen.Evaluator's host logic (files, order, refusals, the writer's
errors), its library calls per chunk (DRY_RUN) and a two-rank gloo run against the one-rank tree.

The output_opt = 1 fixture (tests/golden/reference/box_files_dev_bbox.npz) is recorded with the reference importable:

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_box_files.py
"""
import io
import os
import pickle
import socket
import types
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import box_files_oracle as F
import reference_fixtures as fixtures
from dry import dry, record  # noqa: F401
from objgan_b200 import boxgen, model, ops
from oracle import box_oracle as O
from test_box_gen import (CAT_IDS, COUNT_STATS, EDGE_TRAJ, L2I, LABEL_TO_CLASS, LAYOUT_TRAJ, MEAN_STD, MEAN_STD_EDGE,
                          MEAN_STD_ID, MEANS, _traj, hand_cases, layout_fixture, layout_noise_cnt, ref_box)
from test_text_encoder import NTOK

NAMES = [str(c) for c in CAT_IDS]
I2W = {i: w for w, i in L2I.items()}
# a caption vocabulary without <sos> / <eos>, as the image side's (DAMSM) vocabulary is
CAP_I2W = {0: "<end>", 1: "a", 2: "man", 3: "riding", 4: "horse", 5: "on", 6: "the", 7: "beach", 8: "2", 9: "dogs_x"}
CAP_W2I = {w: i for i, w in CAP_I2W.items()}
OPT1_CAPS = [[1, 2, 3, 1, 4], [6, 7], [1, 9, 8], [5], [2, 2, 2, 2, 2, 2, 2]]


# ---------------------------------------------------------------------------------------------------------------------
# the rows and texts against the reference
# ---------------------------------------------------------------------------------------------------------------------
def test_files_text_matches_reference_boxes_txt():
    want = layout_fixture()
    ncnt = layout_noise_cnt()
    for i in range(len(LAYOUT_TRAJ)):
        labels, samples = _traj(i)
        rows, cls, n_valid, n_special = F.records(labels, samples, MEAN_STD, LABEL_TO_CLASS, COUNT_STATS, ncnt[i])
        txt, _ = F.files_text(rows, cls, NAMES, f"img{i}", [], n_valid)
        assert txt == str(want["boxes_txt"][i]), i
        assert n_special == 0
    assert want["boxes_txt"][3] == "" and want["boxes_txt"][4] == ""
    # class 0 capped at two in trajectory 0
    assert str(want["boxes_txt"][0]).count(",1,0\n") == 2


def _layout_equal(got, want):
    r, f, c, n = got
    rw, fw, cw, nw = want
    assert n == nw and torch.equal(r, rw) and torch.equal(f, fw) and torch.equal(c, cw)


def test_records_compose_to_layout():
    """records() through the boxes.txt round trip is box_oracle.layout(), bit for bit, on every stored case."""
    ncnt = layout_noise_cnt()
    for i in range(len(LAYOUT_TRAJ)):
        labels, samples = _traj(i)
        rows, cls, _, _ = F.records(labels, samples, MEAN_STD, LABEL_TO_CLASS, COUNT_STATS, ncnt[i])
        _layout_equal(F.layout_of(rows, cls), O.layout(labels, samples, MEAN_STD, LABEL_TO_CLASS, COUNT_STATS, ncnt[i]))
    for name, (labels, samples, nc, cs, _, _) in hand_cases().items():
        lab, smp = torch.tensor(labels), torch.tensor(samples)
        rows, cls, n_valid, n_special = F.records(lab, smp, MEAN_STD_ID, LABEL_TO_CLASS, cs, nc)
        _layout_equal(F.layout_of(rows, cls), O.layout(lab, smp, MEAN_STD_ID, LABEL_TO_CLASS, cs, nc))
        assert n_special == (3 if name == "special_mid" else 0), name      # <unk>, <pad>, <sos>
    lab, smp = torch.tensor(EDGE_TRAJ[0]), torch.tensor(EDGE_TRAJ[1])
    rows, cls, _, _ = F.records(lab, smp, MEAN_STD_EDGE, LABEL_TO_CLASS, COUNT_STATS, torch.zeros(80))
    _layout_equal(F.layout_of(rows, cls), O.layout(lab, smp, MEAN_STD_EDGE, LABEL_TO_CLASS, COUNT_STATS, torch.zeros(80)))


def test_records_keep_small_boxes_and_unrounded_values():
    labels, samples, nc, cs, _, _ = hand_cases()["min_size_both"]
    rows, cls, n_valid, _ = F.records(torch.tensor(labels), torch.tensor(samples), MEAN_STD_ID, LABEL_TO_CLASS, cs, nc)
    assert cls == [0, 1] and n_valid == 3 and rows[0][2] == 9.0          # dropped by ROI_MIN_SIZE in the layout only
    labels, samples, nc, cs, _, _ = hand_cases()["txt_round"]
    rows, _, _, _ = F.records(torch.tensor(labels), torch.tensor(samples), MEAN_STD_ID, LABEL_TO_CLASS, cs, nc)
    assert "%.2f" % rows[0][0] == "13.00" and rows[0][0] != 13.0


def dev_bbox_fixture():
    """The reference's Evaluator with output_opt = 1 on LAYOUT_TRAJ (the stub decoder of layout_fixture), with the
    captions OPT1_CAPS: the dev_bbox_test.txt it writes."""
    def produce(tmp):
        _, E = ref_box()
        ncnt = layout_noise_cnt()
        keys = [f"img{i}" for i in range(len(LAYOUT_TRAJ))]
        gdict = {c: (float(COUNT_STATS[i, 0]), float(COUNT_STATS[i, 1])) for i, c in enumerate(CAT_IDS)}
        state = {"b": 0}

        class Dec:
            def __call__(self, *a, **kw):
                traj = LAYOUT_TRAJ[state["b"]]
                return None, None, None, None, {
                    "sequence": [torch.tensor([t[0]]) for t in traj],
                    "xy": [(np.float32(t[1]), np.float32(t[2])) for t in traj],
                    "wh": [(np.float32(t[3]), np.float32(t[4])) for t in traj]}

        ev = E.Evaluator(1, 10, tmp, types.SimpleNamespace(index2word=CAP_I2W), types.SimpleNamespace(index2word=I2W),
                         *[tuple(r) for r in MEAN_STD], gdict, tmp + "/gen_masks/", 1)
        real_rb, real_normal = E.random_batch, np.random.normal

        def rb(*a, select_index, **kw):
            state["b"] = select_index
            return (torch.tensor([OPT1_CAPS[select_index]]),) + (None,) * 7

        def logged(mu, sigma, size=None):
            row = [i for i, c in enumerate(CAT_IDS) if gdict[c] == (mu, sigma)]
            assert len(row) == 1
            return np.array([mu + sigma * float(ncnt[state["b"], row[0]])])
        E.random_batch, np.random.normal = rb, logged
        try:
            ev.evaluate(lambda *a: (None, None), Dec(), [0] * len(keys), keys)
        finally:
            E.random_batch, np.random.normal = real_rb, real_normal
        return {"dev_bbox_test": np.array(open(f"{tmp}/dev_bbox_test.txt").read())}

    path = os.path.join(fixtures.GOLD, "box_files_dev_bbox.npz")
    if fixtures.RECORD:
        import tempfile
        with tempfile.TemporaryDirectory() as tmp:
            np.savez_compressed(path, **produce(tmp))
    return str(np.load(path)["dev_bbox_test"])


def test_dev_bbox_line_matches_reference():
    want = dev_bbox_fixture()
    ncnt = layout_noise_cnt()
    got = ""
    for i in range(len(LAYOUT_TRAJ)):
        labels, samples = _traj(i)
        rows, cls, n_valid, _ = F.records(labels, samples, MEAN_STD, LABEL_TO_CLASS, COUNT_STATS, ncnt[i])
        _, line = F.files_text(rows, cls, NAMES, f"img{i}", [CAP_I2W[w] for w in OPT1_CAPS[i]], n_valid)
        got += line or ""
        # the library's own formatters give the same text
        assert (line or "") == (boxgen.dev_bbox_line(f"img{i}", [CAP_I2W[w] for w in OPT1_CAPS[i]],
                                                     list(zip(rows, cls)), NAMES) if n_valid > 1 else "")
    assert got == want
    assert want.count("\n") == 3 and "img3" not in want and "img4" not in want    # one valid step or none: no line


# ---------------------------------------------------------------------------------------------------------------------
# intake of the reference's test files
# ---------------------------------------------------------------------------------------------------------------------
def test_normalize_string_hand_worked():
    assert boxgen.normalize_string("A man riding��a horse.") == ["a", "man", "riding", "a", "horse"]
    assert boxgen.normalize_string("Two dogs_x and 2 CATS, 3rd-place") == ["two", "dogs_x", "and", "2", "cats", "3rd",
                                                                         "place"]
    # \w matches Unicode letters; the ASCII filter then strips them, and a token left empty is dropped
    assert boxgen.normalize_string("Café über 日本 tea") == ["caf", "ber", "tea"]
    assert boxgen.normalize_string("x�y") == ["x", "y"]              # a single U+FFFD is not \w either
    assert boxgen.normalize_string("") == []


def test_indexes_from_sentence_vocabularies():
    words = ["a", "zebra", "man"]
    assert boxgen.indexes_from_sentence(CAP_W2I, words) == [1, 2]          # unknown words dropped, no <unk>
    w2i = dict(CAP_W2I, **{"<sos>": 10, "<eos>": 11})
    assert boxgen.indexes_from_sentence(w2i, words) == [10, 1, 2, 11]
    assert boxgen.indexes_from_sentence(dict(CAP_W2I, **{"<eos>": 11}), ["zebra"]) == [11]
    assert boxgen.indexes_from_sentence(CAP_W2I, ["zebra"]) == []


def _split_files(tmp_path, lines, keys):
    (tmp_path / "dev.txt").write_text("\n".join(lines) + "\n")
    (tmp_path / "keys.txt").write_text("\n".join(keys) + "\n")
    return str(tmp_path / "dev.txt"), str(tmp_path / "keys.txt")


def _line(cap):
    return "\t".join([cap, "1 2", "3 4", "5 6", "1 1", "1 3"])


def test_read_split_and_numbering(tmp_path):
    caps = ["A man", "the beach", "a horse", "riding on", "a man", "dogs_x 2", "on the beach"]
    keys = ["k1", "k2", "k1", "k1", "k3", "k1", "k1"]
    dev, kp = _split_files(tmp_path, [_line(c) for c in caps], keys)
    data = boxgen.read_test_tuples(dev)
    assert [d[0] for d in data] == [c.lower().split() for c in caps] and data[0][1:] == ["1 2", "3 4", "5 6", "1 1",
                                                                                           "1 3"]
    got_keys = boxgen.read_keys(kp)
    assert got_keys == keys
    assert boxgen.caption_indices(keys) == [0, 0, 1, 2, 0, 3, 4]            # repeated key numbered 0..4 in file order
    assert boxgen.caption_sequences(data, got_keys, CAP_W2I)[5] == [9, 8]


def test_split_refusals(tmp_path):
    dev, kp = _split_files(tmp_path, [_line("a man"), _line("a horse")], ["k1"])
    with pytest.raises(ValueError, match="1 image keys for 2 captions"):
        boxgen.caption_sequences(boxgen.read_test_tuples(dev), boxgen.read_keys(kp), CAP_W2I)
    dev, _ = _split_files(tmp_path, [_line("a man"), "a horse\t1\t2\t3\t4", _line("x")], ["k1", "k2", "k3"])
    with pytest.raises(ValueError, match="line 2: 5 tab-separated fields"):
        boxgen.read_test_tuples(dev)
    dev, kp = _split_files(tmp_path, [_line("a man"), _line("a horse"), _line("Zebra!"), _line("")],
                           ["k1", "k2", "k3", "k4"])
    with pytest.raises(ValueError, match="caption line 3 .*no word"):
        boxgen.caption_sequences(boxgen.read_test_tuples(dev), boxgen.read_keys(kp), CAP_W2I)


def test_caption_numbering_one_shard_or_two():
    keys = [f"k{(i * 7) % 5}" for i in range(23)]
    full = boxgen.caption_indices(keys)
    for world in (1, 2, 3):
        got = []
        for rank in range(world):
            lo, hi = len(keys) * rank // world, len(keys) * (rank + 1) // world
            got += full[lo:hi]
        assert got == full
    assert sorted(full[i] for i in range(23) if keys[i] == "k0") == list(range(5))


@pytest.mark.parametrize("fmt", ["pickle", "torch_zip", "torch_legacy"])
def test_cap_vocab_formats(tmp_path, fmt):
    for name, obj in (("cap_word2index.pt", CAP_W2I), ("cap_index2word.pt", CAP_I2W)):
        if fmt == "pickle":                           # dill writes a dict as a plain pickle
            (tmp_path / name).write_bytes(pickle.dumps(obj, protocol=2))
        else:
            torch.save(obj, str(tmp_path / name), _use_new_zipfile_serialization=fmt == "torch_zip")
    w2i, i2w = boxgen.load_cap_vocab(str(tmp_path))
    assert w2i == CAP_W2I and i2w == CAP_I2W


def test_cap_vocab_refuses_other_globals(tmp_path):
    class Evil:
        def __reduce__(self):
            return (os.system, ("true",))
    (tmp_path / "cap_word2index.pt").write_bytes(pickle.dumps({"a": Evil()}))
    (tmp_path / "cap_index2word.pt").write_bytes(pickle.dumps(CAP_I2W))
    with pytest.raises(pickle.UnpicklingError, match="refusing"):
        boxgen.load_cap_vocab(str(tmp_path))
    torch.save({"a": Evil()}, str(tmp_path / "cap_word2index.pt"))
    with pytest.raises(pickle.UnpicklingError, match="refusing"):
        boxgen.load_cap_vocab(str(tmp_path))


# ---------------------------------------------------------------------------------------------------------------------
# boxgen.Evaluator: host logic with the device stage replaced by the oracle
# ---------------------------------------------------------------------------------------------------------------------
def gaussian_dict():
    return {c: (float(COUNT_STATS[i, 0]), float(COUNT_STATS[i, 1])) for i, c in enumerate(CAT_IDS)}


def make_evaluator(tmp, output_opt=0, **kw):
    kw.setdefault("device", "cpu")
    return boxgen.Evaluator(1, 10, str(tmp), types.SimpleNamespace(word2index=CAP_W2I, index2word=CAP_I2W),
                            types.SimpleNamespace(word2index=L2I, index2word=I2W), *[tuple(r) for r in MEAN_STD],
                            gaussian_dict(), str(tmp) + "/gen_masks/", output_opt, **kw)


def _fake_traj(i):
    """A deterministic trajectory for tuple i: one of LAYOUT_TRAJ, or a special label in the middle."""
    if i % 6 == 5:
        return [4, 3, 5, 2], [(0.1, 0.1, 0.1, 0.1)] * 4, layout_noise_cnt()[0]
    t = LAYOUT_TRAJ[i % 5]
    return [s[0] for s in t], [s[1:] for s in t], layout_noise_cnt()[i % 5]


def oracle_packed(start, b, steps=10):
    """The packed og_box_records buffer of tuples start .. start + b - 1 computed by the oracle."""
    packed = torch.zeros(b * steps * 5 + 3 * b, dtype=torch.int64)
    rows, cls, n_rows, n_valid, n_special = ops.unpack_box_records(packed, b, steps)
    for q in range(b):
        lab, smp, nc = _fake_traj(start + q)
        r, c, nv, ns = F.records(torch.tensor(lab), torch.tensor(smp, dtype=torch.float32), MEAN_STD, LABEL_TO_CLASS,
                                 COUNT_STATS, nc)
        for k, (row, cl) in enumerate(zip(r, c)):
            rows[q, k] = torch.tensor(row, dtype=torch.float64)
            cls[q, k] = cl
        n_rows[q], n_valid[q], n_special[q] = len(r), nv, ns
    return packed


def _with_oracle_device(ev):
    ev._device_records = lambda start, seqs: oracle_packed(start, len(seqs))
    return ev


def split(n):
    keys = [f"{100 + (i * 3) % 7}" for i in range(n)]
    data = [[[CAP_I2W[1 + (i + k) % 9] for k in range(1 + i % 4)], "", "", "", "", ""] for i in range(n)]
    return data, keys


def _modules():
    return model.PreEncoderRNN(NTOK, nhidden=256), model.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, bidirectional=True)


def _tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


@pytest.mark.parametrize("chunk", [1, 4, 64])
def test_evaluator_writes_oracle_files(tmp_path, chunk):
    data, keys = split(17)
    ev = _with_oracle_device(make_evaluator(tmp_path, chunk=chunk))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ev.evaluate(*_modules(), data, keys)
    assert [str(x.message) for x in w if "special label" in str(x.message)] == \
        ["2 captions sampled a box with a special label (<pad>, <sos> or <unk>); the reference raises on these, here "
         "the boxes were dropped"]
    tree = _tree(tmp_path / "gen_masks")
    assert len(tree) == 17
    jidx = boxgen.caption_indices(keys)
    for i in range(17):
        lab, smp, nc = _fake_traj(i)
        r, c, nv, _ = F.records(torch.tensor(lab), torch.tensor(smp, dtype=torch.float32), MEAN_STD, LABEL_TO_CLASS,
                                COUNT_STATS, nc)
        txt, _ = F.files_text(r, c, NAMES, keys[i], [], nv)
        assert tree[f"{keys[i]}/{jidx[i]}/boxes.txt"].decode() == txt, i
    assert tree[f"{keys[3]}/{jidx[3]}/boxes.txt"] == b""                 # an empty file for a sample without rows
    ev1 = _with_oracle_device(make_evaluator(tmp_path, 1, chunk=chunk))
    ev1.evaluate(*_modules(), data, keys)
    lines = open(tmp_path / "dev_bbox_test.txt").read()
    want = ""
    for i in range(17):
        lab, smp, nc = _fake_traj(i)
        r, c, nv, _ = F.records(torch.tensor(lab), torch.tensor(smp, dtype=torch.float32), MEAN_STD, LABEL_TO_CLASS,
                                COUNT_STATS, nc)
        want += F.files_text(r, c, NAMES, keys[i], data[i][0], nv)[1] or ""
    assert lines == want and 0 < lines.count("\n") < 17


def test_evaluator_refusals(tmp_path):
    with pytest.raises(ValueError, match="batch_size must be 1"):
        boxgen.Evaluator(4, 10, str(tmp_path), None, types.SimpleNamespace(index2word=I2W), *MEAN_STD,
                         gaussian_dict(), "x/", 0)
    with pytest.raises(ValueError, match="output_opt"):
        make_evaluator(tmp_path, 2)
    gd = gaussian_dict()
    gd.pop(CAT_IDS[7])
    with pytest.raises(ValueError, match=f"category id {CAT_IDS[7]}"):
        boxgen.Evaluator(1, 10, str(tmp_path), None, types.SimpleNamespace(index2word=I2W), *MEAN_STD, gd, "x/", 0)
    data, keys = split(5)
    ev = _with_oracle_device(make_evaluator(tmp_path))
    with pytest.raises(ValueError, match="4 image keys for 5 captions"):
        ev.evaluate(*_modules(), data, keys[:4])
    data[2][0] = ["zebra"]
    with pytest.raises(ValueError, match="caption line 3"):
        ev.evaluate(*_modules(), data, keys)
    assert not (tmp_path / "gen_masks").exists()                         # refused before anything ran


def test_evaluator_writer_error_raised_in_caller(tmp_path):
    data, keys = split(9)
    (tmp_path / "gen_masks").write_text("a file where the folder should be")
    ev = _with_oracle_device(make_evaluator(tmp_path, chunk=2))
    with pytest.raises(RuntimeError, match="writing the box layout files failed"):
        ev.evaluate(*_modules(), data, keys)


def test_evaluator_reference_modules(tmp_path):
    """The reference's PreEncoderRNN / DecoderRNN are accepted and loaded through their state_dicts."""
    try:
        M, _ = ref_box()
    except Exception:
        pytest.skip("the reference's modules are not importable here")
    enc, dec = M.PreEncoderRNN(NTOK, nhidden=256), M.DecoderRNN(L2I, *MEANS, 1, 150, 256, 5, dropout_p=0.2,
                                                                 use_attention=False, bidirectional=True)
    e, d = boxgen._library_modules(enc, dec, L2I)
    assert isinstance(e, model.PreEncoderRNN) and isinstance(d, model.DecoderRNN)
    assert all(torch.equal(a, b) for a, b in zip(d.state_dict().values(), dec.state_dict().values()))
    assert all(torch.equal(a, b) for a, b in zip(e.state_dict().values(), enc.state_dict().values()))


@pytest.mark.parametrize("lens", [[1] * 5, [1, 40, 7, 3, 22, 9, 2]])
def test_device_records_call_count(dry, tmp_path, lens):
    """Six library calls per chunk (noise, embedding gather, gate inputs, encoder state, decoder, rows), whatever the
    caption lengths; the decoder's label table is made once."""
    ev = make_evaluator(tmp_path)
    enc, dec = _modules()
    ev.generator = boxgen.BoxGenerator(enc.eval(), dec.eval(), ev.mean_std, ev.count_stats, ev.label_to_class, 10)
    seqs = [[1 + k % 9 for k in range(n)] for n in lens]
    record(lambda: ev._device_records(0, seqs))
    calls = [name for name, _ in record(lambda: ev._device_records(len(seqs), seqs))]
    assert calls == ["og_box_noise", "og_gather_rows", "og_conv2d_simt", "og_lstm_bidir_state", "og_box_decode",
                     "og_box_records"]
    args = dict(record(lambda: ev._device_records(3, seqs)))
    assert args["og_box_noise"][:5] == (0, 3, len(seqs), 10, 80)


def test_box_noise_seed_checks(dry):
    with pytest.raises(ValueError, match="seed"):
        ops.box_noise(-1, 0, 2, 10, 80, "cpu")
    nb, nc = ops.box_noise(2 ** 40, 5, 2, 10, 80, "cpu")
    assert nb.shape == (2, 10, 6) and nc.shape == (2, 80)


def test_philox_known_answers():
    """Philox4x32-10 known-answer vectors (Random123's kat_vectors)."""
    assert F.philox([[0, 0, 0, 0]], (0, 0)).tolist() == [[0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]]
    assert F.philox([[0xffffffff] * 4], (0xffffffff, 0xffffffff)).tolist() == \
        [[0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]]


# ---------------------------------------------------------------------------------------------------------------------
# two ranks (gloo) against one
# ---------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, root, output_opt):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ev = _with_oracle_device(make_evaluator(root, output_opt, chunk=3))
        assert ev.world == world and ev.rank == rank
        data, keys = split(23)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ev.evaluate(*_modules(), data, keys)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("output_opt", [0, 1])
def test_two_rank_tree_equals_one_rank(tmp_path, output_opt):
    one, two = tmp_path / "one", tmp_path / "two"
    one.mkdir(), two.mkdir()
    data, keys = split(23)
    _with_oracle_device(make_evaluator(one, output_opt, chunk=5)).evaluate(*_modules(), data, keys)
    mp.spawn(_worker, args=(2, _free_port(), str(two), output_opt), nprocs=2, join=True)
    a, b = _tree(one), _tree(two)
    assert len(a) == (23 if output_opt == 0 else 1) and a == b
