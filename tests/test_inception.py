"""Scoring networks and metrics (CPU): the oracle's INCEPTION_V3 / INCEPTION_V3_FID forwards (tests/inception_oracle.py)
against the reference's own modules, the state_dict layouts and the ImageNet-file loads, the Inception score, the
confidence and the Frechet distance against the reference's functions, the library calls of the forwards (DRY_RUN: host
logic only) and the guards.

The reference side is stored in tests/golden/reference/inception_*.npz, fid_*.npz and inception_layout.json.
Re-record with the reference and torchvision importable (tests/refimport.py):

    OBJGAN_RECORD_REFERENCE=1 python -m pytest tests/test_inception.py
"""
import json
import os
from unittest import mock

import numpy as np
import pytest
import torch

import inception_oracle as I
import reference_fixtures as fixtures
import refimport
from dry import dry, record  # noqa: F401
from objgan_b200 import losses, model, ops

LAYOUT = os.path.join(fixtures.GOLD, "inception_layout.json")
ENCODER_CALLS = os.path.join(os.path.dirname(fixtures.GOLD), "cnn_encoder_calls.json")
IS_CASES = {"B2_256": (2, 256), "B1_128": (1, 128)}
FID_CASE = (2, 128)

_sd = []


def tv_sd():
    """The test weights over torchvision's Inception3 keys, fixed by their seed."""
    if not _sd:
        _sd.append(I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0))
    return {k: v.clone() for k, v in _sd[0].items()}


def images(b, s, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b, 3, s, s, generator=g) * 2 - 1


def _reference(cls, *args):
    R = refimport.load()
    R.cfg.TRAIN.NET_E = "text_encoder100.pth"
    sd = tv_sd()
    with mock.patch("torch.load", lambda *a, **k: sd):          # the ImageNet file the constructors read
        net = getattr(R.model, cls)(*args)
    return net.eval()


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the reference's modules
# ---------------------------------------------------------------------------------------------------------------------
def is_fixture(name):
    def produce():
        b, s = IS_CASES[name]
        with torch.no_grad():
            return {"probs": _reference("INCEPTION_V3")(images(b, s, 10 + s))}
    return fixtures.recorded(f"inception_v3_{name}", produce, cap=4096)


def fid_fixture(dims):
    def produce():
        R = refimport.load()
        net = _reference("INCEPTION_V3_FID", [I.FID_DIMS[dims]])
        x = images(*FID_CASE, seed=dims)
        R.cfg.TEST.FID_DIMS = dims
        with torch.no_grad():
            fmap = net(x)[0]
            acts = R.utils.get_activations(x, net, FID_CASE[0])
        return {"map": fmap, "acts": torch.from_numpy(acts)}
    return fixtures.recorded(f"inception_fid_{dims}", produce, cap=4096)


@pytest.mark.parametrize("name", list(IS_CASES))
def test_is_oracle_matches_reference(name):
    ref = is_fixture(name)
    b, s = IS_CASES[name]
    with torch.no_grad():
        p = I.inception_v3_forward(tv_sd(), images(b, s, 10 + s))
    assert p.shape == (b, 1000)
    assert _rel(p, ref["probs"].view(b, 1000)) <= 1e-5
    assert ref["probs"].max() < 0.5                       # the test weights keep the softmax far from saturation


@pytest.mark.parametrize("dims", list(I.FID_DIMS))
def test_fid_oracle_matches_reference(dims):
    ref = fid_fixture(dims)
    x = images(*FID_CASE, seed=dims)
    with torch.no_grad():
        fmap = I.inception_fid_forward(tv_sd(), x, [I.FID_DIMS[dims]])[0]
        acts = I.fid_activations(tv_sd(), x, dims)
    assert acts.shape == (FID_CASE[0], dims)
    assert _rel(torch.from_numpy(fixtures.sample(fmap, 4096)), ref["map"]) <= 1e-5
    assert _rel(acts, ref["acts"]) <= 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# layouts and loads
# ---------------------------------------------------------------------------------------------------------------------
def _layout(net):
    return {k: list(v.shape) for k, v in net.state_dict().items()}


def test_state_dict_layouts_match_reference():
    if fixtures.RECORD:
        out = {"INCEPTION_V3": _layout(_reference("INCEPTION_V3"))}
        for b in range(4):
            out[f"INCEPTION_V3_FID_{b}"] = _layout(_reference("INCEPTION_V3_FID", [b]))
        with open(LAYOUT, "w") as f:
            json.dump(out, f, indent=0)
    layout = json.load(open(LAYOUT))
    assert _layout(model.INCEPTION_V3()) == layout["INCEPTION_V3"]
    assert len(layout["INCEPTION_V3"]) == 580
    for b in range(4):
        assert _layout(model.INCEPTION_V3_FID([b])) == layout[f"INCEPTION_V3_FID_{b}"], b
    assert len(layout["INCEPTION_V3_FID_3"]) == 564


@pytest.mark.parametrize("prefix", ["", "module."])
@pytest.mark.parametrize("with_nbt", [True, False])
def test_from_imagenet(tmp_path, prefix, with_nbt):
    sd = {prefix + k: v for k, v in tv_sd().items() if with_nbt or not k.endswith("num_batches_tracked")}
    path = str(tmp_path / "inception_v3_google-1a9a5a14.pth")
    torch.save(sd, path)
    ref = tv_sd()
    net = model.INCEPTION_V3.from_imagenet(path, device="cpu")
    assert torch.equal(net.model.fc.weight, ref["fc.weight"])
    loaded = model.INCEPTION_V3.from_imagenet(model._imagenet_state_dict(path), device="cpu")
    assert all(torch.equal(a, b) for a, b in zip(loaded.state_dict().values(), net.state_dict().values()))
    assert torch.equal(net.model.AuxLogits.conv1.conv.weight, ref["AuxLogits.conv1.conv.weight"])
    assert torch.equal(net.model.Mixed_7c.branch3x3dbl_3b.bn.running_var, ref["Mixed_7c.branch3x3dbl_3b.bn.running_var"])
    for b, name, j, key in ((0, "Conv2d_2b_3x3", 2, "conv.weight"), (1, "Conv2d_4a_3x3", 1, "bn.running_mean"),
                            (3, "Mixed_7c", 2, "branch_pool.conv.weight")):
        fid = model.INCEPTION_V3_FID.from_imagenet(path, device="cpu", output_blocks=[b])
        assert torch.equal(fid.state_dict()[f"blocks.{b}.{j}.{key}"], ref[f"{name}.{key}"])
        assert len(fid.blocks) == b + 1
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop(prefix + "Mixed_6e.branch7x7_2.conv.weight")
        torch.save(bad, path)
        model.INCEPTION_V3.from_imagenet(path, device="cpu")


def test_guards():
    for net in (model.INCEPTION_V3(), model.INCEPTION_V3_FID([1])):
        x = torch.zeros(1, 3, 64, 64)
        net.train()
        with pytest.raises(RuntimeError, match="eval mode only"):
            net(x)
        net.eval()
        next(net.parameters()).requires_grad_(True)
        with pytest.raises(RuntimeError, match="frozen"):
            net(x)
    for bad in ([], [4], [-1]):
        with pytest.raises(ValueError):
            model.INCEPTION_V3_FID(bad)
    with pytest.raises(ValueError, match="no stage"):
        model._trunk_program(lambda name: None, None, "Mixed_8a", ("pooled",))


def test_cpu_input_raises_before_any_launch():
    """The kernels read device memory only: a host image batch is refused before the first library call."""
    for net in (model.INCEPTION_V3(), model.INCEPTION_V3_FID([0])):
        calls = []
        with mock.patch.object(ops, "_call", lambda name, *a: calls.append(name)):
            with pytest.raises(RuntimeError, match="CUDA tensors"):
                net(torch.zeros(1, 3, 64, 64))
            if isinstance(net, model.INCEPTION_V3_FID):
                with pytest.raises(RuntimeError, match="CUDA tensors"):
                    net.activations(torch.zeros(1, 3, 64, 64))
        assert calls == []


# ---------------------------------------------------------------------------------------------------------------------
# library calls (dry run)
# ---------------------------------------------------------------------------------------------------------------------
def _record_calls(fn):
    """The library calls of fn() with their small integer arguments (sizes and flags, not addresses)."""
    return [[name] + [a for a in args if isinstance(a, int) and abs(a) < 2 ** 20] for name, args in record(fn)]


def test_dry_run_library_calls(dry):
    """The forwards issue library calls only; the FID program stops at its last block; CNN_ENCODER's forward and
    input-gradient calls are the ones recorded before the trunk builder was shared."""
    torch.manual_seed(0)
    enc = model.CNN_ENCODER(256)
    enc(torch.zeros(2, 3, 256, 256))                      # folds BatchNorm and packs the weights

    def enc_fwd_bwd():
        enc(torch.zeros(2, 3, 256, 256))
        x = torch.zeros(1, 3, 200, 200, requires_grad=True)
        f, c = enc(x)
        (f.sum() + c.sum()).backward()
    assert _record_calls(enc_fwd_bwd) == json.load(open(ENCODER_CALLS))

    forbid = [mock.patch(f, side_effect=AssertionError("torch compute")) for f in
              ("torch.nn.functional.conv2d", "torch.nn.functional.interpolate", "torch.nn.functional.softmax",
               "torch.softmax", "torch.nn.functional.linear")]
    isnet = model.INCEPTION_V3()
    isnet(torch.zeros(2, 3, 256, 256))
    for p in forbid:
        p.start()
    try:
        calls = _record_calls(lambda: isnet(torch.zeros(2, 3, 256, 256)))
        names = [c[0] for c in calls]
        assert names[0] == "og_inception_input" and names[-1] == "og_softmax_rows"
        assert "og_bilinear_fwd" not in names and "og_nchw_to_nhwc" not in names
        convs = {}
        for dims in (64, 2048):
            fid = model.INCEPTION_V3_FID([model.INCEPTION_V3_FID.BLOCK_INDEX_BY_DIM[dims]])
            fid.activations(torch.zeros(2, 3, 256, 256))
            calls = _record_calls(lambda: fid.activations(torch.zeros(2, 3, 256, 256)))
            assert calls[0][0] == "og_inception_input" and calls[-1][0] == "og_global_avg_fwd"
            convs[dims] = sum(1 for c in calls if c[0].startswith("og_conv2d"))
    finally:
        for p in forbid:
            p.stop()
    assert convs == {64: 3, 2048: 75}, convs


# ---------------------------------------------------------------------------------------------------------------------
# metrics against the reference's functions
# ---------------------------------------------------------------------------------------------------------------------
def predictions(n, seed, zero=False):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, 1000, generator=g) * 3 + torch.randn(n // 10 + 1, 1000, generator=g).repeat_interleave(10, 0)[:n] * 2
    p = torch.softmax(logits, 1).numpy().astype(np.float32)
    if zero:
        p[7, 3] = 0.0
    return p


IS_ROWS = {"160": (160, False), "157": (157, False), "zero": (160, True)}


def score_fixture(name):
    def produce():
        R = refimport.load()
        n, zero = IS_ROWS[name]
        p = predictions(n, n, zero)
        with np.errstate(all="ignore"):
            m, s = R.utils.compute_inception_score(p, 10)
            mc, sc = R.utils.negative_log_posterior_probability(p, 10)
        return {"mean": m, "std": s, "mean_conf": mc, "std_conf": sc}
    return fixtures.recorded(f"inception_score_{name}", produce)


@pytest.mark.parametrize("name", list(IS_ROWS))
def test_inception_score_bitwise(name):
    ref = score_fixture(name)
    n, zero = IS_ROWS[name]
    sc = losses.InceptionScore(10)
    p = torch.from_numpy(predictions(n, n, zero))
    sc.add(p[:100])
    sc.add(p[100:])
    with np.errstate(all="ignore"):
        got = sc.result()
    for key, v in zip(("mean", "std", "mean_conf", "std_conf"), got):
        r = float(ref[key])
        assert (np.isnan(v) and np.isnan(r)) if (zero and key in ("mean", "std")) else v == r, (key, v, r)


def fid_sets(name):
    rng = np.random.default_rng(5)
    if name == "full_rank":
        a = rng.standard_normal((500, 64)) @ rng.standard_normal((64, 64)) * 0.3 + 1.0
        b = rng.standard_normal((500, 64)) @ rng.standard_normal((64, 64)) * 0.25 + 1.2
    else:       # one set collapsed to a single image: scipy's sqrtm of the 3 x 3 zero product is not finite
        a = np.repeat(np.round(rng.standard_normal((1, 3)) * 8) / 8, 40, 0)     # dyadic: its covariance is exactly 0
        b = rng.standard_normal((40, 3)) * 1.5
    return a.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)


def fid_ref_fixture(name):
    def produce():
        R = refimport.load()
        from scipy import linalg
        sqrtm = linalg.sqrtm
        real, fake = fid_sets(name)
        mu1, s1 = R.utils.calculate_activation_statistics(real)
        mu2, s2 = R.utils.calculate_activation_statistics(fake)
        # scipy 1.18 dropped sqrtm's disp argument; disp=False returned (sqrtm, error estimate)
        shim = lambda a, disp=True: sqrtm(a) if disp else (sqrtm(a), None)
        with mock.patch.object(R.utils.linalg, "sqrtm", shim):
            d = R.utils.calculate_frechet_distance(mu1, s1, mu2, s2)
        return {"fid": float(d), "retry": float(not np.isfinite(sqrtm(s1.dot(s2))).all())}
    return fixtures.recorded(f"fid_{name}", produce)


@pytest.mark.parametrize("name", ["full_rank", "singular"])
def test_frechet_distance_matches_reference(name):
    ref = fid_ref_fixture(name)
    real, fake = fid_sets(name)
    assert float(ref["retry"]) == (1.0 if name == "singular" else 0.0)
    d = losses.frechet_distance(real.mean(0), np.cov(real, rowvar=False), fake.mean(0), np.cov(fake, rowvar=False))
    assert abs(d - float(ref["fid"])) <= 1e-12 * abs(float(ref["fid"])), (d, float(ref["fid"]))
