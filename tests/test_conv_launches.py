"""CPU record of every library call the convolutions issue, byte for byte, at every row of tests/conv_cases.py.

The host code runs a dry run (lib.DRY_RUN: the GPU's dispatch, and ops._chk accepts host tensors) on CPU tensors from
torch.empty, with ops._call replaced by a recorder that launches nothing.  A record holds,
per call, the entry name, every non-pointer argument (floats exactly), each pointer as the order in which its address
first appeared in the run (0 stays null), and the tap quadruples of og_conv2d_tc / entry quintuples of
og_conv2d_wgrad_tc read from their host arrays during the call.  Tap order is summation order, so a reordered tap list
changes a result's bits while every tolerance test still passes: this test sees it.  ops._p keeps each buffer whose
address it hands out alive until the run ends, so no address can be reused within a run and the pointer numbering
does not depend on the allocator.

tests/golden/conv_launches.json holds one SHA-256 per run; on a mismatch the run's full record is printed.
``python tests/test_conv_launches.py`` rewrites the fixture from the current host code.
"""
import ctypes
import hashlib
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))      # run as a script
from conv_cases import CASES, EDGE_CASES, ENC_CASES  # noqa: E402
from objgan_b200 import lib, model, ops  # noqa: E402
from objgan_b200.lib import PAD_REFLECT  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_launches.json")
PROTOS = lib.parse_header()
ARRAYS = {"og_conv2d_tc": (26, 4), "og_conv2d_wgrad_tc": (17, 5)}   # argument index of the host array, ints per row
ENGINES = ("f16x3", "simt")


class _Recorder:
    def __init__(self):
        self.calls, self.ids, self.keep = [], {}, []

    def p(self, t):
        if t is None:
            return 0
        self.keep.append(t.untyped_storage())     # the storage, not the tensor: autograd may still steal gradients
        return t.data_ptr()

    def call(self, name, *args):
        types = PROTOS[name][:-1]                 # every prototype ends with the stream
        assert len(args) == len(types), (name, len(args), len(types))
        arr = ARRAYS.get(name)
        rec = [name]
        for i, (a, t) in enumerate(zip(args, types)):
            if arr is not None and i == arr[0]:
                rows = (ctypes.c_int * (arr[1] * args[i + 1])).from_address(a)
                rec.append(list(rows))
            elif t is ctypes.c_void_p:
                rec.append(0 if a == 0 else "p%d" % self.ids.setdefault(a, len(self.ids)))
            elif t in (ctypes.c_float, ctypes.c_double):
                rec.append(float(a).hex())
            else:
                assert isinstance(a, int), (name, i, a)
                rec.append(a)
        self.calls.append(rec)


def _recorder(setattr):
    """run(fn) -> the record of the library calls fn issues, with the GPU dispatch on CPU tensors."""
    setattr(lib, "DRY_RUN", True)
    setattr(model, "FAST_INIT", True)

    def run(fn):
        r = _Recorder()
        setattr(ops, "_call", r.call)
        setattr(ops, "_p", r.p)
        fn()
        return r.calls
    return run


@pytest.fixture()
def record(monkeypatch):
    return _recorder(monkeypatch.setattr)


def _conv_run(row, variant):
    N, H, W, Cin, Cout, k, stride, pad, mode, act, bias, split, path = row

    def fn():
        m = model.Conv2dP(Cin, Cout, k, stride, pad, bias, mode, act, split)
        x = torch.empty(N, H, W, ops.cpad(Cin)).requires_grad_(True)
        if variant == "sink":
            for p_ in m.parameters():
                p_.og_grad_sink = torch.empty_like(p_)
        elif variant == "amax":
            ops._tag_amax(x)
        elif variant == "split":           # operand copies a producer wrote (og_norm_apply_split)
            s2d = path == "s2"
            hp = 1 if mode == PAD_REFLECT else 0
            shape = (4 * N, H // 2, W // 2, x.shape[3]) if s2d else (N, H + 2 * hp, W + 2 * hp, x.shape[3])
            x.og_split = (torch.empty(shape, dtype=torch.float16), torch.empty(shape, dtype=torch.float16),
                          torch.empty(1, dtype=torch.int32), hp, s2d, x._version)
        y = m(x)
        y.backward(torch.empty(y.shape))
    return fn


def _enc_run(row):
    d, N, H, W, Cin, Cout, kh, kw, stride, padh, padw, relu, bias, yoff, Cy, path = row

    def fn():
        w = torch.empty(Cout, Cin, kh, kw)
        bn = [tuple(torch.empty(Cout) for _ in range(4))] if bias else None
        layer = ops.EncConv([w], bn, kh, kw, stride, padh, padw, 1e-3, relu)
        oh, ow = layer.out_hw(H, W)
        if d == "fwd":
            ops.enc_conv_fwd(layer, torch.empty(N, H, W, ops.cpad(Cin)), torch.empty(N, oh, ow, Cy), yoff)
        else:
            ops.enc_conv_dgrad(layer, torch.empty(N, oh, ow, Cout), H, W)
    return fn


def _runs(kind):
    """{key: fn} of every recorded run of one table ("conv": CASES + EDGE_CASES, "enc": ENC_CASES)."""
    if kind == "enc":
        return {"enc " + ",".join(map(str, r)): _enc_run(r) for r in ENC_CASES}
    runs = {}
    for r in CASES + EDGE_CASES:
        variants = ("plain", "sink") + (("amax", "split") if r[-1] in ("s1", "s2") else ())
        for v in variants:
            runs["conv %s %s" % (",".join(map(str, r)), v)] = _conv_run(r, v)
    return runs


def _digest(calls):
    return hashlib.sha256(json.dumps(calls, separators=(",", ":")).encode()).hexdigest()


@pytest.mark.parametrize("kind", ["conv", "enc"])
@pytest.mark.parametrize("engine", ENGINES)
def test_conv_launches_are_recorded(engine, kind, record, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    want = json.load(open(GOLDEN))
    bad = []
    for key, fn in _runs(kind).items():
        calls = record(fn)
        if want.get(engine + " " + key) != _digest(calls):
            bad.append((key, calls))
    for key, calls in bad[:1]:
        print(f"\n{engine} {key}: {len(calls)} calls")
        for c in calls:
            print("  ", json.dumps(c))
    assert not bad, f"{len(bad)} runs differ from {os.path.basename(GOLDEN)}: " + "; ".join(k for k, _ in bad[:10])


if __name__ == "__main__":
    out = {}
    run = _recorder(setattr)
    for engine in ENGINES:
        ops.CONV_ENGINE = engine
        for kind in ("conv", "enc"):
            for key, fn in _runs(kind).items():
                out[engine + " " + key] = _digest(run(fn))
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} runs written to {GOLDEN}")
