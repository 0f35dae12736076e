"""GPU suite for smirk_b200.MICA: the forward (shape_params and the ArcFace features) against the torch restatement
(tests/mica_ref.py) run in fp32 on the same GPU with cuDNN TF32 off, the golden fixture of the reference class, the shape
loss and its gradient against F.mse_loss autograd, checkpoint loading, re-packing, determinism, batch independence,
CUDA-graph capture, and a pretraining-shaped step.  Errors are max-abs error over max-abs.  Tolerances: 1e-4 at
precisions 0 and 3; 5e-3 at precision 1 (TF32), or twice the error of cuDNN TF32 itself where that is larger (DESIGN §6
"MICA shape loss")."""
import copy
import os
import tempfile

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from smirk_b200 import synth_inputs

import encoder_train_ref as tr
import make_golden_mica as mg
import mica_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {0: 1e-4, 3: 1e-4}


def _err(a, ref):
    a, ref = torch.as_tensor(a), torch.as_tensor(ref)
    return ((a.detach().cpu().double() - ref.detach().cpu().double()).abs().max() / ref.detach().cpu().double().abs().max()).item()


@pytest.fixture(scope="module")
def sd():
    return mica_ref.mica_state_dict(mg.SEED)


@pytest.fixture(scope="module")
def sd_dev(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


@pytest.fixture
def no_tf32():
    """The fp32 oracle: cuDNN and cuBLAS without TF32, restored afterwards."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def make(sd, precision):
    import smirk_b200
    m = smirk_b200.MICA(checkpoint=None)
    m.load_state_dict(sd)
    for p in m.parameters():
        p.requires_grad = False
    m = m.eval().to(DEV)
    m.precision = precision
    return m


def oracle(sd_dev, img, tf32=False):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        with torch.no_grad():
            return mica_ref.mica_ref(sd_dev, img.to(DEV))
    finally:
        torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("B", [1, 2, 5, 32])
@pytest.mark.parametrize("precision", [0, 1, 3])
def test_forward_vs_fp32_oracle(sd, sd_dev, no_tf32, precision, B):
    m = make(sd, precision)
    img = mica_ref.probe_images(B, 20 + B).to(DEV)
    shape, feat = oracle(sd_dev, img)
    got = m(img)["shape_params"]
    assert got.shape == (B, 300) and not got.requires_grad
    e_s, e_f = _err(got, shape), _err(m.arcface_features(img), feat)
    if precision == 1:
        s32, f32 = oracle(sd_dev, img, tf32=True)
        cudnn = max(_err(s32, shape), _err(f32, feat))
        tol = 5e-3 if cudnn <= 5e-3 else 2 * cudnn
        print("B=%d TF32: shape %.2e features %.2e; cuDNN TF32 %.2e (gate %.2e)" % (B, e_s, e_f, cudnn, tol))
    else:
        tol = TOL[precision]
        print("B=%d precision %d: shape %.2e features %.2e" % (B, precision, e_s, e_f))
    assert e_s <= tol and e_f <= tol


def test_precision0_vs_golden(sd, golden):
    gold = golden("mica")
    m = make(sd, 0)
    img = mg.golden_images().to(DEV)
    assert _err(m.arcface_features(img), gold["features"]) <= 1e-4
    assert _err(m(img)["shape_params"], gold["shape_params"]) <= 1e-4
    for D in (300, 100):
        s = mg.golden_shape_params(D).to(DEV).requires_grad_()
        loss = m.calculate_mica_shape_loss(s, img)
        g, = torch.autograd.grad(loss, [s])
        assert _err(loss, gold["loss_%d" % D]) <= 1e-4 and _err(g, gold["grad_%d" % D]) <= 1e-4


@pytest.mark.parametrize("D", [300, 100])
def test_shape_loss_and_gradient_vs_autograd(sd, D, capsys):
    m = make(sd, 1)
    B = 4
    img = mica_ref.probe_images(B, 40).to(DEV)
    mica_shape = m(img)["shape_params"]
    g = torch.Generator().manual_seed(41)
    s0 = (torch.randn(B, D, generator=g) * 0.05).to(DEV)
    s = s0.clone().requires_grad_()
    loss = m.calculate_mica_shape_loss(s, img.view(B, 3, 112, 112))
    assert ("Truncating the MICA output to %d dimensions" % D in capsys.readouterr().out) == (D < 300)
    (loss * 3.0).backward()
    r = s0.clone().requires_grad_()
    want = F.mse_loss(r, mica_shape[:, :D])
    (want * 3.0).backward()
    assert loss.shape == () and loss.requires_grad
    assert _err(loss, want) <= 1e-6 and _err(s.grad, r.grad) <= 1e-6
    again = m.calculate_mica_shape_loss(s0, img)
    assert torch.equal(again, loss.detach())                  # deterministic


def test_checkpoint_constructor_equals_load_state_dict(sd):
    import smirk_b200
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        mica_ref.write_checkpoint(sd, root)
        os.chdir(root)
        try:
            a = smirk_b200.MICA().eval().to(DEV)
        finally:
            os.chdir(old)
    img = mica_ref.probe_images(2, 50).to(DEV)
    with torch.no_grad():
        assert torch.equal(a(img)["shape_params"], make(sd, 0)(img)["shape_params"])


def test_weight_change_repacks(sd):
    m = make(sd, 3)
    img = mica_ref.probe_images(2, 60).to(DEV)
    before = m(img)["shape_params"]
    with torch.no_grad():
        m.arcface.layer3[7].bn2.weight.mul_(1.5)
        m.regressor.output.bias.add_(0.25)
    after = m(img)["shape_params"]
    fresh = make({k: v.cpu() for k, v in m.state_dict().items()}, 3)
    assert not torch.equal(before, after) and torch.equal(after, fresh(img)["shape_params"])
    c = copy.deepcopy(m)
    assert torch.equal(c(img)["shape_params"], after) and c._native.handle is not m._native.handle


@pytest.mark.parametrize("precision", [0, 1, 3])
def test_deterministic(sd, precision):
    m = make(sd, precision)
    img = mica_ref.probe_images(5, 70).to(DEV)
    a, b = m(img)["shape_params"], m(img)["shape_params"]
    assert torch.equal(a, b)


@pytest.mark.parametrize("precision", [0, 1, 3])
def test_batch_independent(sd, precision):
    m = make(sd, precision)
    img = mica_ref.probe_images(5, 80).to(DEV)
    full = m(img)["shape_params"]
    for i in range(5):
        assert torch.equal(m(img[i:i + 1])["shape_params"], full[i:i + 1]), i


def test_cuda_graph_replay_equals_eager(sd):
    m = make(sd, 1)
    img = mica_ref.probe_images(3, 90).to(DEV)
    eager = m(img)["shape_params"].clone()
    x = torch.zeros_like(img)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m(x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(x)["shape_params"]
    x.copy_(img)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


# ---- a config_pretrain-shaped step ----------------------------------------------------------------------------------
def _make_encoder(precision):
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    e = enc.to(DEV).train().allow_train_mode_(True)
    for mod in e.modules():
        if hasattr(mod, "precision"):
            mod.precision = precision
    return e


def _pretrain_loss(out, fl, rd, tgt, mica_loss):
    """SmirkTrainer.step1 with config_pretrain.yaml: 100 * landmark MSE (FAN first 17, mediapipe) + 1e-2 * expression
    regularisation + 10 * the MICA shape loss."""
    fo = fl(out)
    ro = rd(fo["vertices"], out["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
    lmk = F.mse_loss(ro["landmarks_fan"][:, :17, :2], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"][..., :2], tgt["mp"])
    reg = torch.sum(out["expression_params"] ** 2) / out["expression_params"].shape[0]
    return 100.0 * lmk + 1e-2 * reg + 10.0 * mica_loss(out["shape_params"])


def test_pretrain_step_sgd_parity(sd, sd_dev, no_tf32, asset_root):
    """Three SGD steps of the pretraining step (train-mode encoder, FLAME, Renderer, MICA at precision 0) against the same
    steps with the oracle encoder and the oracle MICA."""
    import smirk_b200
    fl, rd = smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV)
    B = 4
    g = torch.Generator().manual_seed(1800)
    tgt = {"fan": torch.rand(B, 68, 2, generator=g).to(DEV) - 0.5, "mp": torch.rand(B, 105, 2, generator=g).to(DEV) - 0.5}
    imgs = [synth_inputs.images(B, 1810 + s) for s in range(3)]
    mica_imgs = [mica_ref.probe_images(B, 1820 + s).to(DEV) for s in range(3)]
    enc = _make_encoder(0)
    ref = tr.from_module(enc)
    mica = make(sd, 0)
    opt_d = torch.optim.SGD(enc.parameters(), lr=1e-7)
    opt_r = torch.optim.SGD(ref.parameters(), lr=1e-7)
    for step, img in enumerate(imgs):
        opt_d.zero_grad(); opt_r.zero_grad()
        mi = mica_imgs[step]
        _pretrain_loss(enc(img.to(DEV)), fl, rd, tgt, lambda s: mica.calculate_mica_shape_loss(s, mi)).backward()
        with torch.no_grad():
            ms = oracle(sd_dev, mi)[0]
        ro = {k: v.to(DEV) for k, v in ref(img).items()}
        _pretrain_loss(ro, fl, rd, tgt, lambda s: mica_ref.shape_loss_ref(s, ms)).backward()
        opt_d.step(); opt_r.step()
    rs = ref.state_dict()
    errs = {k: _err(v, rs[k]) for k, v in enc.state_dict().items() if v.dtype == torch.float32}
    top = max(errs, key=errs.get)
    print("pretraining step: after 3 SGD steps, parameters and statistics worst %.2e (%s)" % (errs[top], top))
    assert errs[top] <= 1e-4
