"""GPU tests of eval-mode BatchNorm and of the generator sampler (objgan_b200.sampler.GSampler): the eval-mode G
forward against the oracle (tests/oracle_eval.py, pinned to the reference's G_NET after eval() by
tests/test_eval_mode.py), the eval BatchNorm operator forward / backward against torch's CPU F.batch_norm(training=False),
the gradient w.r.t. z through the eval-mode generator, and graph replay against eager sampling."""
import pytest
import torch
import torch.nn.functional as F

import oracle_eval
from objgan_b200 import lib, model, ops, synth, trainer
from objgan_b200.lib import NA_GLU, NA_LRELU, NA_NONE
from objgan_b200.sampler import GSampler
from oracle import objgan_oracle as O
from test_eval_mode import eval_fixture, eval_inputs, eval_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
ENGINES = ["simt", "f16x3"]


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


def close(a, b, tol=1e-3, what=""):
    r = rel(a, b)
    assert r <= tol, (what, r)


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _flat(out):
    """The 6-tuple as a flat list of tensors."""
    fake, btc, att, btatt, mu, logvar = out
    return [*fake, *btc, *att, *btatt, mu, logvar]


def _to_dev(inp):
    return {k: (v.to(DEV) if torch.is_tensor(v) else [t.to(DEV) for t in v] if isinstance(v, list) else v)
            for k, v in inp.items()}


def _g(sd, eval_mode=True):
    g = model.G_NET(80)
    g.load_state_dict(sd, strict=True)
    g.to(DEV)
    return g.eval() if eval_mode else g


def _run(g, d, z=None):
    g.ca_net.eps_override = d["eps"]
    return g(d["z"] if z is None else z, d["sent_emb"], d["words_embs"], d["glove_words_embs"], d["slabels_feat"],
             d["mask"], d["hmaps"], d["rois"], d["fm_rois"], d["num_rois"], d["bt_masks"], d["fm_bt_masks"],
             d["glb_max_num_roi"])


_sd_cache = {}


def _eval_sd(B):
    """_g_sd() weights with the running statistics of the reference fixture (10 train-mode passes)."""
    if B not in _sd_cache:
        want = eval_fixture(B)
        _sd_cache[B] = (eval_state_dict(want), want["in__eps"])
    sd, eps = _sd_cache[B]
    return {k: v.clone() for k, v in sd.items()}, eps


# ---------------------------------------------------------------------------------------------------
# eval-mode G forward
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B", [1, 3])
def test_g_eval_forward(B, engine, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    sd, eps = _eval_sd(B)
    inp = eval_inputs(B)
    inp["eps"] = eps
    with torch.no_grad():
        ref = oracle_eval.g_net_forward_eval(sd, inp)
    g = _g(sd)
    d = _to_dev(inp)
    with torch.no_grad():
        out = _run(g, d)
    for i, (a, b) in enumerate(zip(_flat(out), _flat(ref))):
        close(a, b, what=f"output {i}")
    for k, v in g.state_dict().items():           # eval() leaves running_mean / running_var / num_batches_tracked
        if "running" in k or "num_batches" in k:
            assert torch.equal(v.cpu(), sd[k]), k
    g.train()
    with torch.no_grad():
        out_t = _run(g, d)
    for i in range(3):                            # batch statistics give clearly different images
        assert rel(out_t[0][i], out[0][i]) > 0.05, i


# ---------------------------------------------------------------------------------------------------
# operator: eval BatchNorm + activation, forward and backward
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", [NA_GLU, NA_LRELU, NA_NONE])
@pytest.mark.parametrize("dims", [1, 2])
def test_bn_eval_act(act, dims):
    torch.manual_seed(9)
    if dims == 1:
        n, c, h, w = 5, 48, 1, 1
        x = torch.randn(n, c) * 2 + 0.7
    else:
        n, c, h, w = 3, 16, 37, 41                # 4551 pixels: many CTAs share each channel's parameter gradients
        x = torch.randn(n, c, h, w) * 2 + 0.7
    x.requires_grad_(True)
    gamma = torch.randn(c).requires_grad_(True)
    beta = torch.randn(c).requires_grad_(True)
    rm, rv = torch.randn(c) * 0.5, torch.rand(c) * 3 + 0.1
    yn = F.batch_norm(x, rm, rv, gamma, beta, False, 0.1, 1e-5)
    if act == NA_GLU:
        yr = O.glu(yn)
    elif act == NA_LRELU:
        yr = F.leaky_relu(yn, 0.2)
    else:
        yr = yn
    gy = torch.randn_like(yr)
    yr.backward(gy)
    co = yr.shape[1]

    def run():
        xg = x.detach().to(DEV).requires_grad_(True)
        xn = xg.view(n, 1, 1, c) if dims == 1 else ops.to_nhwc(xg)
        gg = gamma.detach().to(DEV).requires_grad_(True)
        bb = beta.detach().to(DEV).requires_grad_(True)
        bufs = (rm.to(DEV), rv.to(DEV), torch.zeros((), dtype=torch.long, device=DEV))
        out = ops.batch_norm_act(xn, gg, bb, bufs, act, training=False)
        y = out.view(n, co) if dims == 1 else ops.to_nchw(out, co)
        y.backward(gy.to(DEV))
        assert torch.equal(bufs[0].cpu(), rm) and torch.equal(bufs[1].cpu(), rv) and int(bufs[2]) == 0
        return y.detach(), xg.grad, gg.grad, bb.grad

    a = run()
    for t, r, what in zip(a, (yr, x.grad, gamma.grad, beta.grad), ("fwd", "dx", "dgamma", "dbeta")):
        close(t, r, what=what)
    b = run()
    for t, u in zip(a, b):                        # fixed-order reductions: bitwise repeatable
        assert torch.equal(t, u)


# ---------------------------------------------------------------------------------------------------
# gradient w.r.t. z through the eval-mode generator (latent optimisation)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine,l2,mx", [("simt", 5e-3, 3e-2), ("f16x3", 3e-2, 1e-1)])
def test_grad_z_eval(engine, l2, mx, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    sd, _ = _eval_sd(3)
    inp = eval_inputs(2)
    wts = [torch.randn(f.shape, generator=torch.Generator().manual_seed(i)) for i, f in enumerate(inp["imgs"])]
    z = inp["z"].clone().requires_grad_(True)
    ref = oracle_eval.g_net_forward_eval(sd, dict(inp, z=z))
    gz_ref, = torch.autograd.grad(sum((f * w).sum() for f, w in zip(ref[0], wts)), [z])
    g = _g(sd)
    for p in g.parameters():
        p.requires_grad_(False)
    d = _to_dev(inp)
    zg = d["z"].clone().requires_grad_(True)
    out = _run(g, d, zg)
    sum((f * w.to(DEV)).sum() for f, w in zip(out[0], wts)).backward()
    assert rel_l2(zg.grad, gz_ref) <= l2, rel_l2(zg.grad, gz_ref)
    assert rel(zg.grad, gz_ref) <= mx, rel(zg.grad, gz_ref)
    for k, v in g.state_dict().items():
        if "running" in k or "num_batches" in k:
            assert torch.equal(v.cpu(), sd[k]), k


# ---------------------------------------------------------------------------------------------------
# sampler
# ---------------------------------------------------------------------------------------------------
def _same(a, b, tol=1e-4, what=""):
    """Every output within tol of max|output|; returns whether all were bitwise equal."""
    exact = True
    for i, (x, y) in enumerate(zip(_flat(a), _flat(b))):
        assert x.shape == y.shape, (what, i)
        if x.numel():
            close(x, y, tol, what=f"{what} output {i}")
        exact = exact and torch.equal(x, y)
    return exact


@pytest.mark.parametrize("engine", ENGINES)
def test_sampler_graph_matches_eager(engine, monkeypatch):
    monkeypatch.setattr(ops, "CONV_ENGINE", engine)
    sd, _ = _eval_sd(3)
    s = GSampler(_g(sd))
    ia = synth.make_inputs(2, seed=61, parity=True)
    ia2 = synth.make_inputs(2, seed=62, parity=True)
    ib = synth.make_inputs(3, seed=63, parity=True)
    assert ia["slabels_feat"].shape == ia2["slabels_feat"].shape and ia["glb_max_num_roi"] == ia2["glb_max_num_roi"]
    a1 = s.sample(ia)                             # eager warm-up, then capture of key A
    b1 = s.sample(ib)                             # key B
    n0 = lib.get().launches
    a2 = s.sample(ia)                             # replay A
    assert lib.get().launches - n0 > 100          # the replay accounts for the library calls it recorded
    b2 = s.sample(ib)                             # replay B
    a3 = s.sample(ia2)                            # replay A with other inputs
    assert len(s._graphs) == 2
    exact = [_same(a2, a1, what="A"), _same(b2, b1, what="B"), _same(a3, s.sample_eager(ia2), what="A'")]
    print("graph replay bitwise equal to eager:", exact)
    # no aliasing: every call returned its own storage, and a later replay did not overwrite an earlier result
    ptrs = [t.data_ptr() for o in (a1, a2, a3, b1, b2) for t in _flat(o) if t.numel()]
    assert len(ptrs) == len(set(ptrs))
    _same(a2, s.sample_eager(ia), what="A after A'")
    assert not torch.equal(a2[0][0], a3[0][0])


def _snapshot(t):
    bks = [t.bG, *t._d_buckets()]
    state = [(b.flat.clone(), b.m.clone(), b.v.clone(), None if b.avg is None else b.avg.clone(), b.step,
              b.step_dev.clone()) for b in bks]
    nets = [t.netG, *t.netsPatD, *t.netsShpD, t.netObjSSD, t.netObjLSD]
    bufs = [[x.clone() for x in m.buffers()] for m in nets]
    return state, bufs


def _equal_snapshots(a, b):
    for x, y in zip(a[0], b[0]):
        for u, v in zip(x, y):
            assert (u is None and v is None) or (torch.equal(u, v) if torch.is_tensor(u) else u == v)
    for x, y in zip(a[1], b[1]):
        assert all(torch.equal(u, v) for u, v in zip(x, y))


def test_sampler_from_trainer_and_snapshot(tmp_path):
    t = trainer.StepBTrainer(device=DEV, seed=3)
    inp = synth.make_inputs(2, seed=4, parity=True)
    inp.pop("eps")
    dev = t.to_device(inp)
    for _ in range(2):
        trainer.StepATrainer.step(t, dev)         # two Step-A steps (G forward, patch discriminators, G update, EMA)
    torch.cuda.synchronize()
    before = _snapshot(t)
    s = GSampler.from_trainer(t)
    torch.cuda.synchronize()
    _equal_snapshots(before, _snapshot(t))
    x = synth.make_inputs(3, seed=71, parity=True)
    ref = model.G_NET(80).to(DEV)
    ref.load_state_dict(t.bG.ema_state_dict(), strict=True)
    ref.eval()
    with torch.no_grad():
        want = _run(ref, _to_dev(x))
    got = s.sample(x)
    _same(got, want, 1e-6, what="from_trainer")
    t.save_model(str(tmp_path), 2)
    s2 = GSampler.from_snapshot(str(tmp_path / "netG_epoch_2.pth"), device=DEV)
    _same(s2.sample(x), got, 1e-6, what="from_snapshot")
    _same(s2.sample(x), s.sample(x), 1e-6, what="from_snapshot, replayed")
    _equal_snapshots(before, _snapshot(t))


def test_sampler_reload_drops_graphs():
    sd_a, _ = _eval_sd(3)
    torch.manual_seed(12)
    other = model.G_NET(80)
    other.apply(model.weights_init)
    sd_b = {k: v.clone() for k, v in other.state_dict().items()}
    for k in sd_b:                                # the fixture's running statistics, so both are eval-mode sensible
        if "running" in k or "num_batches" in k:
            sd_b[k] = sd_a[k].clone()
    x = synth.make_inputs(2, seed=81, parity=True)
    s = GSampler(_g(sd_a))
    s.sample(x)
    first = s.sample(x)                           # replay with weights A
    s.load_state_dict(sd_b)
    assert not s._graphs
    fresh = GSampler(_g(sd_b))
    want = fresh.sample(x)
    _same(s.sample(x), want, 1e-6, what="reloaded, eager")
    _same(s.sample(x), want, 1e-6, what="reloaded, replay")
    assert not torch.equal(first[0][2], want[0][2])


def test_sampler_full_size():
    sd, _ = _eval_sd(3)
    s = GSampler(_g(sd))
    x = synth.make_inputs(16, seed=91)            # B = 16, L = 18, Rmax = glb_max_num_roi = 10
    assert x["words_embs"].shape[2] == 18 and x["slabels_feat"].shape[2] == 10 and x["glb_max_num_roi"] == 10
    s.sample(x)
    got = s.sample(x)                             # replay
    assert len(s._graphs) == 1
    assert all(torch.isfinite(t).all() for t in _flat(got))
    _same(got, s.sample_eager(x), what="B=16")
    compact = synth.compact(x)                    # the compact batch builds hmaps / slabels_feat on the device
    _same(s.sample(compact), got, 1e-6, what="compact batch")
