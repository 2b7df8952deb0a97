"""Scoring networks and metrics on the GPU: og_inception_input, og_softmax_rows and og_moments_f64 against float64,
INCEPTION_V3 and INCEPTION_V3_FID (every FID dim) on both engines against the float64 oracle (tests/inception_oracle.py),
the Inception score and the FID against the same formulas on oracle outputs, GSampler.score_images, and bitwise-equal
repeat forwards.  Measured errors are printed (pytest -s) and recorded in DESIGN.md section 8."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception_oracle as I
from objgan_b200 import losses, model, ops, synth
from objgan_b200.ops import _p
from objgan_b200.sampler import GSampler, _new_g

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]


@pytest.fixture
def engine(request, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", request.param)
    return request.param


def _rel_max(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def images(b, s, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(b, 3, s, s, generator=g) * 2 - 1).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
def _input_f64(x, mode):
    x = x.double()
    m, s = I.MEAN, I.STD
    if mode == model.IS_INPUT:
        x = x * 0.5 + 0.5
        x = torch.stack([(x[:, c] - m[c]) / s[c] for c in range(3)], 1)
        return F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=True)
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) * 0.5 + 0.5
    return torch.stack([x[:, c] * (s[c] / 0.5) + (m[c] - 0.5) / 0.5 for c in range(3)], 1)


@pytest.mark.parametrize("mode", [model.IS_INPUT, model.FID_INPUT])
@pytest.mark.parametrize("size", [64, 256, 299])
def test_inception_input(mode, size):
    x = images(3, size, size)
    y = torch.full((3, 299, 299, 8), float("nan"), device=DEV)
    ops._call("og_inception_input", _p(x), 3, size, size, 299, mode, _p(y))
    err = _rel_max(y[..., :3].permute(0, 3, 1, 2), _input_f64(x, mode))
    print(f"og_inception_input mode {mode} from {size}: max error / max |ref| {err:.2e}")
    # the fp32 source coordinate r * o (like ATen's) is off by up to 2 * size * 2^-24, which moves the blend by that
    # much of a neighbour difference (at most 2 max |ref|); plus the roundings of the affine and the blend
    assert err <= 4 * size * 2.0 ** -24 + 2e-6
    assert torch.equal(y[..., 3:], torch.zeros_like(y[..., 3:]))


def test_softmax_rows():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(37, 1000, generator=g) * torch.linspace(0.1, 27, 37).view(37, 1)
    x[0, 5], x[1, 7], x[2, :] = 80.0, -80.0, 0.0
    x = x.clamp(-80, 80).to(DEV)
    y = ops.softmax_rows(x)
    ref = torch.softmax(x.double(), 1)
    big = ref > 1e-30
    rel = ((y.double() - ref).abs()[big] / ref[big]).max().item()
    print(f"og_softmax_rows: max relative error {rel:.2e}")
    assert rel <= 2e-5
    assert (y.double() - ref).abs()[~big].max().item() <= 1e-30 if (~big).any() else True
    assert torch.equal(y, ops.softmax_rows(x))


@pytest.mark.parametrize("d", [64, 300, 2048])
def test_moments_f64(d):
    """Batches of 16, 16 and 5 rows with |mean| / std up to 1e3 against np.mean / np.cov of the same fp32 values."""
    g = torch.Generator().manual_seed(d)
    mu = torch.randn(d, generator=g) * torch.logspace(-1, 3, d)
    x = (mu + torch.randn(37, d, generator=g) * torch.rand(d, generator=g).add(0.5)).float()
    runs = []
    for _ in range(2):
        m = losses._Moments(d)
        for a, b in ((0, 16), (16, 32), (32, 37)):
            m.add(x[a:b].to(DEV))
        runs.append(m.statistics())
    xn = x.double().numpy()
    rmu, rcov = xn.mean(0), np.cov(xn, rowvar=False)
    emu = np.abs(runs[0][0] - rmu).max() / np.abs(rmu).max()
    ecov = np.abs(runs[0][1] - rcov).max() / np.abs(rcov).max()
    print(f"og_moments_f64 d={d}: mean {emu:.1e}, covariance {ecov:.1e}")
    assert emu <= 1e-12 and ecov <= 1e-12
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])


# ---------------------------------------------------------------------------------------------------------------------
# the networks against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
_nets = {}


def nets():
    if not _nets:
        sd = I.inception3_test_state_dict(model._Inception3().state_dict(), seed=0)
        _nets["sd64"] = {k: (v.double() if v.is_floating_point() else v).to(DEV) for k, v in sd.items()}
        _nets["is"] = model.INCEPTION_V3()
        _nets["is"].load_state_dict({"model." + k: v for k, v in sd.items()})
        _nets["is"].to(DEV)
        for dims, b in model.INCEPTION_V3_FID.BLOCK_INDEX_BY_DIM.items():
            f = model.INCEPTION_V3_FID([b])
            f.load_state_dict(f.from_torchvision(sd))
            _nets[dims] = f.to(DEV)
    return _nets


_oracle = {}


def oracle(kind, b):
    if (kind, b) not in _oracle:
        x = images(b, 256, 40 + b)
        with torch.no_grad():
            if kind == "is":
                _oracle[kind, b] = I.inception_v3_forward(nets()["sd64"], x.double())
            else:       # (the block's map, its pixel average)
                fmap = I.inception_fid_forward(nets()["sd64"], x.double(), [I.FID_DIMS[kind]])[0]
                _oracle[kind, b] = (fmap, F.adaptive_avg_pool2d(fmap, (1, 1)).flatten(1))
    return _oracle[kind, b]


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("b", [1, 3, 16])
def test_inception_v3_forward(engine, b):
    p = nets()["is"](images(b, 256, 40 + b))
    ref = oracle("is", b)
    err = _rel_max(p, ref)
    print(f"INCEPTION_V3 {engine} B={b}: max error / max prob {err:.2e}")
    assert p.shape == (b, 1000)
    assert err <= 1e-4          # measured on an H100: at most 8.7e-6 (f16x3, B=16)


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
@pytest.mark.parametrize("b", [1, 3, 16])
@pytest.mark.parametrize("dims", [64, 192, 768, 2048])
def test_inception_fid_forward(engine, b, dims):
    net = nets()[dims]
    x = images(b, 256, 40 + b)
    acts = net.activations(x)
    rmap, ref = oracle(dims, b)
    err = _rel_max(acts, ref)
    fmap = net(x)[0]
    merr = _rel_max(fmap, rmap)
    print(f"INCEPTION_V3_FID dims {dims} {engine} B={b}: max error / max |act| {err:.2e}, map {merr:.2e}")
    assert acts.shape == (b, dims) and fmap.shape == rmap.shape
    assert err <= 3e-5          # measured on an H100: at most 2.9e-6 (dims 64, B=3)
    assert merr <= 1e-4         # measured on an H100: at most 8.1e-6 (dims 64, B=16)


@pytest.mark.parametrize("engine", ENGINES, indirect=True)
def test_repeat_forwards_bitwise(engine):
    x = images(16, 256, 7)
    n = nets()
    assert torch.equal(n["is"](x), n["is"](x))
    assert torch.equal(n[2048].activations(x), n[2048].activations(x))


def test_host_input_raises():
    """A CUDA-resident network refuses a host image batch before any launch."""
    n = nets()
    for fn in (n["is"], n[64], n[768].activations):
        with pytest.raises(RuntimeError, match="CUDA tensors"):
            fn(torch.zeros(1, 3, 64, 64))


def test_bn_refold_after_load():
    net = nets()["is"]
    x = images(1, 128, 9)
    p0 = net(x)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    sd2 = dict(sd)
    sd2["model.Conv2d_1a_3x3.bn.running_var"] = sd["model.Conv2d_1a_3x3.bn.running_var"] * 2
    net.load_state_dict(sd2)
    p1 = net(x)
    net.load_state_dict(sd)
    assert not torch.equal(p0, p1) and torch.equal(p0, net(x))


# ---------------------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------------------
def test_inception_score_10_batches():
    """10 batches of 16 (the evaluator's 10 splits) against the same formulas on the float64 oracle's predictions."""
    n = nets()
    sc, ref = losses.InceptionScore(10), []
    for i in range(10):
        x = images(16, 64, 500 + i)
        sc.add(n["is"](x))
        with torch.no_grad():
            ref.append(I.inception_v3_forward(n["sd64"], x.double()).cpu().numpy())
    got = sc.result()
    p = np.concatenate(ref, 0)
    want = losses.inception_score(p, 10) + losses.negative_log_posterior(p, 10)
    err = max(abs(a - b) / abs(b) for a, b in zip(got[::2], want[::2]))
    print(f"Inception score {got}, float64 oracle {tuple(float(v) for v in want)}: relative error {err:.2e}")
    assert err <= 1e-5          # measured on an H100: 8.1e-7
    assert all(abs(a - b) <= 1e-4 * abs(want[0]) for a, b in zip(got[1::2], want[1::2]))


def test_fid_dims64():
    """256 images per side at dims 64 (full rank): the FID against the same formula on the oracle's activations."""
    n = nets()
    fd, fake, real = losses.FrechetDistance(64), [], []
    for i in range(16):
        xf, xr = images(16, 64, 600 + i), images(16, 64, 700 + i) * 0.5
        fd.add(n[64].activations(xf), n[64].activations(xr))
        with torch.no_grad():
            fake.append(I.fid_activations(n["sd64"], xf.double(), 64).cpu().numpy())
            real.append(I.fid_activations(n["sd64"], xr.double(), 64).cpu().numpy())
    fake, real = np.concatenate(fake), np.concatenate(real)
    want = losses.frechet_distance(real.mean(0), np.cov(real, rowvar=False), fake.mean(0), np.cov(fake, rowvar=False))
    got = fd.result()
    print(f"FID dims 64: {got:.6e}, float64 oracle {want:.6e}: relative error {abs(got - want) / want:.2e}")
    assert abs(got - want) <= 1e-5 * want     # measured on an H100: 3.7e-7


def test_fid_dims2048_moments():
    """At dims 2048 the covariance of a test-sized set is singular; compare the moments instead (batches 16, 16, 5)."""
    n = nets()
    fd, acts = losses.FrechetDistance(2048), []
    for i, b in enumerate((16, 16, 5)):
        x = images(b, 128, 800 + i)
        fd.add(n[2048].activations(x))
        with torch.no_grad():
            acts.append(I.fid_activations(n["sd64"], x.double(), 2048).cpu().numpy())
    acts = np.concatenate(acts)
    mu, sigma = fd.fake.statistics()
    emu = np.abs(mu - acts.mean(0)).max() / np.abs(acts.mean(0)).max()
    rcov = np.cov(acts, rowvar=False)
    ecov = np.abs(sigma - rcov).max() / np.abs(rcov).max()
    print(f"FID dims 2048 moments: mean {emu:.2e}, covariance {ecov:.2e}")
    assert emu <= 2e-5 and ecov <= 5e-4      # measured on an H100: 2.0e-6 and 5.8e-5


def test_sampler_score_images():
    n = nets()
    s = GSampler(_new_g(80, DEV), inception=n["is"], inception_fid=n[2048])
    batch = synth.make_inputs(4, seed=900, parity=True)
    fake_imgs = s.sample(batch)[0]
    pred, acts = s.score_images(fake_imgs)
    with torch.no_grad():
        x = fake_imgs[-1].double()
        rp = I.inception_v3_forward(n["sd64"], x)
        ra = I.fid_activations(n["sd64"], x, 2048)
    assert pred.shape == (4, 1000) and acts.shape == (4, 2048)
    assert _rel_max(pred, rp) <= 1e-4 and _rel_max(acts, ra) <= 3e-5
    with pytest.raises(ValueError):
        GSampler(_new_g(80, DEV)).score_images(fake_imgs)
