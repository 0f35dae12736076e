"""GPU suite for the train-mode generator (batch-statistics BatchNorm, running statistics, parameter gradients), at the
trainer's configuration (6, 3, 32, 5).

Forward outputs and running statistics are checked against torch's own train-mode BatchNorm in the restatement
(tests/generator_train_ref.py, oracle/generator_ref with its ops swapped, run in float64 on the GPU); every parameter
gradient and the input gradient against autograd through it with the device's ReLU masks and pool choices replayed; one
step against the reference class's golden file.  Also: the opt-in, eval after training, the frozen input-gradient path,
determinism and CUDA-graph capture, and config_train's generator steps through the drop-in classes (encoder -> FLAME ->
Renderer -> masking -> generator -> 10 L1 + 10 VGG + 100 landmarks, and the frozen / unfrozen alternation).
Tolerances: max-abs error over max-abs of each tensor, 1e-4 at precisions 0 and 3 (fp32 / 3xTF32); TF32 (precision 1) is
looser in train mode, as the encoder's, see DESIGN.md §6 "Generator training"."""
import contextlib
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from smirk_b200 import synth_inputs

import generator_train_ref as gtr

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFG = (6, 3, 32, 5)
TOL = {0: 1e-4, 1: 3e-2, 3: 1e-4}
GRAD_TOL = {0: 1e-4, 1: 1e-1, 3: 1e-4}


@pytest.fixture(scope="module")
def base(native_lib):
    import smirk_b200
    g = smirk_b200.SmirkGenerator(*CFG)
    g.load_state_dict(synth_inputs.random_state_dict(g.state_dict(), seed=7))
    return g


def _make(base, precision, momentum=0.1):
    g = copy.deepcopy(base).to(DEV).train().allow_train_mode_(True)
    g.precision = precision
    for m in g.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = momentum
    return g


def _inputs(B, seed):
    x = torch.cat([synth_inputs.images(B, seed), synth_inputs.masked_images(B, seed + 1)], 1)[:, :CFG[0]].contiguous()
    gy = torch.randn(B, CFG[1], 224, 224, generator=torch.Generator().manual_seed(seed + 2))
    return x, gy


def _err(a, ref):
    a, ref = a.detach().cpu().double(), ref.detach().cpu().double()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


@contextlib.contextmanager
def fp32_cudnn():
    """torch's convolutions in fp32 (cuDNN's TF32 off), restored afterwards."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _stats(m):
    return {k: v for k, v in m.state_dict().items() if "running_" in k or "num_batches" in k}


@pytest.mark.parametrize("momentum", [0.1, None])
@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("B", [2, 8, 32])
def test_forward_and_running_stats_two_steps(base, B, precision, momentum):
    g = _make(base, precision, momentum)
    sd = gtr.cpu_state(base, DEV, torch.float64)
    worst = 0.0
    for step in range(2):
        x, _ = _inputs(B, 100 + step)
        with torch.no_grad():
            y = g(x.to(DEV))
            ref = gtr.generator_train_ref(sd, x.to(DEV, torch.float64), res_blocks=CFG[3], momentum=momentum)
        worst = max(worst, _err(y, ref))
        for k, v in _stats(g).items():
            if "num_batches" in k:
                assert int(v) == int(sd[k]) == step + 1, k
            else:
                worst = max(worst, _err(v, sd[k]))
    print("B %d precision %d momentum %s: worst max-abs err / max-abs %.2e" % (B, precision, momentum, worst))
    assert worst <= TOL[precision]


def _device_grads(g, x, gy, input_grad=True):
    xl = x.to(DEV).requires_grad_(input_grad)
    y = g(xl)
    params = list(g.parameters())
    grads = torch.autograd.grad((y * gy.to(DEV)).sum(), ([xl] if input_grad else []) + params)
    return (grads[0] if input_grad else None), dict(zip([k for k, _ in g.named_parameters()], grads[1 if input_grad else 0:])), y


def _replay_grads(base, g, x, gy, momentum=0.1):
    """Autograd in float64 through the oracle with the device's discrete choices, on the statistics g had before its last
    step -> (input gradient, {parameter: gradient}, {upconvN: sum over pixels of |gradient of its output|} per channel)."""
    with torch.no_grad():
        replay = {k: v.double() for k, v in gtr.relu_outputs(g.saved_activations(x.to(DEV))).items()}
    sd = gtr.cpu_state(base, DEV, torch.float64)
    xl = x.to(DEV, torch.float64).requires_grad_()
    ups = {}
    y = gtr.generator_train_ref(sd, xl, res_blocks=CFG[3], momentum=momentum, replay=replay, record=ups)
    (y * gy.to(DEV, torch.float64)).sum().backward()
    terms = {k: u.grad.abs().sum((0, 2, 3)) for k, u in ups.items()}
    return xl.grad, {k: v.grad for k, v in sd.items() if v.requires_grad}, terms


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("B", [2, 8])
def test_every_gradient_vs_replay_oracle(base, B, precision):
    if precision == 1 and B == 8:
        pytest.skip("one TF32 case is enough")
    g = _make(base, precision)
    x, gy = _inputs(B, 200 + B)
    ref_x, ref_p, terms = _replay_grads(base, copy.deepcopy(g), x, gy)
    gx, gp, _ = _device_grads(g, x, gy)
    errs = {"input": _err(gx, ref_x)}
    errs.update({k: _err(v, ref_p[k]) for k, v in gp.items()})
    # An up-convolution's bias gradient is a near-cancelling sum, the sum over pixels of the gradient of its output: that
    # output feeds a conv and a batch-statistics BatchNorm, which remove a per-channel shift except at the zero-padded
    # border.  Its max-abs is far below the size of its terms, and an fp32 sum carries rounding of the terms' size, so it
    # is measured per channel against the sum of |terms| (the sum's condition).
    for k in [k for k in errs if k.startswith("upconv") and k.endswith(".bias")]:
        plain = errs[k]
        errs[k] = ((gp[k].double() - ref_p[k]).abs() / terms[k.split(".")[0]]).max().item()
        print("%s: max-abs err / max-abs %.2e; per channel, err / sum |terms| %.2e" % (k, plain, errs[k]))
    worst = max(errs, key=errs.get)
    print("B %d precision %d: worst %s %.2e (of %d tensors)" % (B, precision, worst, errs[worst], len(errs)))
    assert len(errs) == 1 + len(list(base.parameters()))
    assert errs[worst] <= GRAD_TOL[precision], errs


def test_detached_input_and_no_grad(base):
    from smirk_b200 import _lib
    x, gy = _inputs(2, 300)
    g1, g2 = _make(base, 0), _make(base, 0)
    _, full, y1 = _device_grads(g1, x, gy, input_grad=True)
    _, det, y2 = _device_grads(g2, x, gy, input_grad=False)
    assert torch.equal(y1, y2)
    for k in full:
        assert torch.equal(full[k], det[k]), k
    g3 = _make(base, 0)
    n0 = _lib.lib().smk_launch_count()
    with torch.no_grad():
        y3 = g3(x.to(DEV))
    n1 = _lib.lib().smk_launch_count()
    g4 = _make(base, 0).requires_grad_(False)
    y4 = g4(x.to(DEV))                              # grad mode on, nothing requires grad: no autograd node, no backward
    n2 = _lib.lib().smk_launch_count()
    assert n1 - n0 == n2 - n1 and not y4.requires_grad
    assert torch.equal(y3, y1) and torch.equal(y4, y1)
    for k, v in _stats(g3).items():
        assert torch.equal(v, _stats(g1)[k]), k


def test_two_forwards_one_backward(base):
    g = _make(base, 3)
    (x1, gy1), (x2, gy2) = _inputs(2, 400), _inputs(2, 410)
    a, b = x1.to(DEV).requires_grad_(), x2.to(DEV).requires_grad_()
    loss = (g(a) * gy1.to(DEV)).sum() + (g(b) * gy2.to(DEV)).sum()
    ga, gb = torch.autograd.grad(loss, [a, b])
    ref = _make(base, 3)
    assert torch.equal(ga, _device_grads(ref, x1, gy1)[0])
    assert torch.equal(gb, _device_grads(ref, x2, gy2)[0])


def test_opt_in_eval_after_train_and_frozen_path(base):
    import smirk_b200
    from smirk_b200 import _lib, smirk_encoder
    from oracle import generator_ref
    x, gy = _inputs(3, 500)
    plain = copy.deepcopy(base).to(DEV).train()
    with pytest.raises(RuntimeError, match="train-mode.*allow_train_mode_"):
        plain(x.to(DEV))
    assert copy.deepcopy(plain.allow_train_mode_(True))._train_allowed()
    smirk_encoder.set_train_mode_default(True)
    try:
        assert smirk_b200.SmirkGenerator()._train_allowed()
    finally:
        smirk_encoder.set_train_mode_default(False)
    g = _make(base, 0)
    for s in range(2):
        with torch.no_grad():
            g(_inputs(2, 510 + s)[0].to(DEV))
    ge = g.eval()
    with torch.no_grad():
        y = ge(x.to(DEV))
        y_copy = copy.deepcopy(ge)(x.to(DEV))
    ref = generator_ref.generator_forward_ref({k: v.cpu() for k, v in ge.state_dict().items()}, x, res_blocks=CFG[3])
    assert _err(y, ref) <= 1e-4 and torch.equal(y, y_copy)
    frozen = ge.requires_grad_(False)             # utils.freeze_module: eval, frozen -> the input-gradient path as before
    n0 = _lib.lib().smk_launch_count()
    frozen(x.to(DEV).requires_grad_())
    assert _lib.lib().smk_launch_count() - n0 == 38


# ---- config_train's generator steps through the drop-in classes ---------------------------------------------------------

@pytest.fixture(scope="module")
def chain_mods(asset_root, native_lib):
    """(encoder base, FLAME, Renderer, VGG loss): the encoder with random_state_dict(seed=7) weights, the VGG loss with the
    weights of its golden file, both frozen where the trainer keeps them."""
    import smirk_b200
    import make_golden_vgg_loss as mv
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    vgg = smirk_b200.VGGPerceptualLoss(weights=None)
    vgg.load_state_dict(mv.golden_state_dict())
    return enc, smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV), vgg.to(DEV)


def _chain_data(B, seed):
    """Images, the masking step's output (it carries no gradient; synthetic here) and landmark targets of one batch."""
    g = torch.Generator().manual_seed(seed)
    tgt = {"fan": (torch.rand(B, 68, 2, generator=g) - 0.5).to(DEV), "mp": (torch.rand(B, 105, 2, generator=g) - 0.5).to(DEV)}
    return synth_inputs.images(B, seed + 1), synth_inputs.masked_images(B, seed + 2).to(DEV), tgt


def _step1_loss(enc_out, fl, rd, generator, vgg, img, masked, tgt):
    """smirk_trainer.py step1 with config_train.yaml's weights: FLAME -> Renderer -> cat(rendered, masked) -> generator
    -> 10 L1 + 10 VGG against the image, + 100 landmark MSE (FAN first 17, mediapipe)."""
    fo = fl(enc_out)
    ro = rd(fo["vertices"], enc_out["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
    y = generator(torch.cat([ro["rendered_img"], masked], 1))
    lmk = F.mse_loss(ro["landmarks_fan"][:, :17, :2], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"][..., :2], tgt["mp"])
    return 10.0 * F.l1_loss(y, img) + 10.0 * vgg(y, img) + 100.0 * lmk


def _train_pair(enc_base, gen_base, precision):
    enc = copy.deepcopy(enc_base).to(DEV).train().allow_train_mode_(True)
    for m in enc.modules():
        if hasattr(m, "precision"):
            m.precision = precision
    return enc, _make(gen_base, precision)


def _optimizer(cls, enc_params, gen_params, **kw):
    # the landmark loss gives the pose backbone gradients of order 1e4: its rate is small, as in the encoder's own test
    return cls([{"params": enc_params, "lr": 1e-7 if cls is torch.optim.SGD else 1e-5},
                {"params": gen_params, "lr": 1e-4}], **kw)


def test_config_train_step1_sgd_matches_oracle_chain_and_adam_lowers_loss(base, chain_mods):
    """Three SGD steps of step1 on the device (encoder and generator in train mode, precision 0).  Alongside, the oracle
    generator (generator_train_ref on the GPU in fp32, the device generator's ReLU and pool choices replayed, as the frozen
    generator's chain test does) takes the same three steps on the generator inputs the device chain produced, with the
    generator's part of the loss (10 L1 + 10 VGG) and the same optimizer.  The inputs are the device chain's because the
    chain is not smooth in them: the rasteriser's coverage is discrete, so after one update two chains whose encoders
    differ by rounding render different silhouette pixels (measured: about 100 pixels by up to 0.29 after one step), and
    the generators would no longer see one input.  The encoder's own parity is its test's.  Gate, max-abs error over
    max-abs of each tensor: the generator's parameters and statistics after the three steps within 1e-5.  Then 20 Adam
    steps of the whole chain lower the loss."""
    enc_base, fl, rd, vgg = chain_mods
    enc, gen = _train_pair(enc_base, base, 0)
    gsd = gtr.cpu_state(base, DEV)
    seen = {}

    def dev_gen(xx):                               # the device generator, keeping its input for the oracle
        seen["x"] = xx.detach()
        return gen(xx)
    opt = _optimizer(torch.optim.SGD, list(enc.parameters()), list(gen.parameters()))
    opt_r = _optimizer(torch.optim.SGD, [], [v for v in gsd.values() if v.requires_grad])
    with fp32_cudnn():
        for step in range(3):
            img, masked, tgt = _chain_data(2, 1900 + 10 * step)
            opt.zero_grad(); opt_r.zero_grad()
            _step1_loss(enc(img.to(DEV)), fl, rd, dev_gen, vgg, img.to(DEV), masked, tgt).backward()
            with torch.no_grad():
                replay = gtr.relu_outputs(gen.saved_activations(seen["x"]))
            y = gtr.generator_train_ref(gsd, seen["x"], res_blocks=CFG[3], replay=replay)
            (10.0 * F.l1_loss(y, img.to(DEV)) + 10.0 * vgg(y, img.to(DEV))).backward()
            opt.step(); opt_r.step()
    gerr = {k: _err(v, gsd[k]) for k, v in gen.state_dict().items() if v.dtype == torch.float32}
    top = max(gerr, key=gerr.get)
    print("config_train step1, 3 SGD steps: generator parameters and statistics worst %.2e (%s)" % (gerr[top], top))
    assert gerr[top] <= 1e-5
    enc, gen = _train_pair(enc_base, base, 3)
    opt = _optimizer(torch.optim.Adam, list(enc.parameters()), list(gen.parameters()))
    data = [_chain_data(2, 1950 + 10 * s) for s in range(3)]
    losses = []
    for s in range(20):
        img, masked, tgt = data[s % 3]
        opt.zero_grad()
        loss = _step1_loss(enc(img.to(DEV)), fl, rd, gen, vgg, img.to(DEV), masked, tgt)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print("config_train step1, Adam: loss %.4f -> %.4f" % (losses[0], losses[-1]))
    assert losses[-1] < losses[0]


def test_config_train_frozen_unfrozen_alternation(base, chain_mods):
    """step2's alternation (set_freeze_status flips freeze_generator_in_second_path): a frozen generator (eval,
    requires_grad_(False), as utils.freeze_module leaves it) takes the eval input-gradient path, keeps its parameters and
    statistics and still passes the gradient to the encoder; an unfrozen one trains, and the two kinds of step
    alternate on one module."""
    enc_base, fl, rd, vgg = chain_mods
    enc, gen = _train_pair(enc_base, base, 3)
    opt = _optimizer(torch.optim.SGD, list(enc.parameters()), list(gen.parameters()))
    for s in range(4):
        frozen = s % 2 == 0
        gen.eval().requires_grad_(False) if frozen else gen.train().requires_grad_(True)
        before = {k: v.clone() for k, v in gen.state_dict().items()}
        img, masked, tgt = _chain_data(2, 2000 + 10 * s)
        opt.zero_grad()
        _step1_loss(enc(img.to(DEV)), fl, rd, gen, vgg, img.to(DEV), masked, tgt).backward()
        g_enc = [p.grad for p in enc.expression_encoder.parameters() if p.grad is not None]
        assert g_enc and all(torch.isfinite(t).all() for t in g_enc) and any(float(t.abs().max()) > 0 for t in g_enc), s
        assert all((p.grad is None) == frozen for p in gen.parameters()), s
        opt.step()
        changed = {k for k, v in gen.state_dict().items() if not torch.equal(v, before[k])}
        if frozen:
            assert not changed, s
        else:
            assert "conv.weight" in changed and "encoder1.enc1norm1.running_mean" in changed
            assert all(int(v) == int(before[k]) + 1 for k, v in gen.state_dict().items() if "num_batches" in k)


def test_config_train_step1_deterministic_and_cuda_graph(base, chain_mods):
    """step1's forward + backward (every encoder and generator gradient, running statistics) is bitwise the same twice at
    B = 32, and a CUDA graph of it replays bitwise equal to eager steps."""
    enc_base, fl, rd, vgg = chain_mods
    img, masked, tgt = _chain_data(32, 2100)
    runs = []
    for _ in range(2):
        enc, gen = _train_pair(enc_base, base, 3)
        params = list(enc.parameters()) + list(gen.parameters())
        grads = torch.autograd.grad(_step1_loss(enc(img.to(DEV)), fl, rd, gen, vgg, img.to(DEV), masked, tgt), params)
        runs.append((grads, list(_stats(gen).values()) + [v for k, v in enc.state_dict().items() if "running" in k]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    B = 2
    (enc, gen), (enc_e, gen_e) = _train_pair(enc_base, base, 3), _train_pair(enc_base, base, 3)
    params, params_e = list(enc.parameters()) + list(gen.parameters()), list(enc_e.parameters()) + list(gen_e.parameters())
    data = [_chain_data(B, 2110 + 10 * s) for s in range(3)]
    x, masked, tgt = data[0][0].to(DEV), data[0][1].clone(), {k: v.clone() for k, v in data[0][2].items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                     # warm-up: handles and workspaces exist before capture
        torch.autograd.grad(_step1_loss(enc(x), fl, rd, gen, vgg, x, masked, tgt), params)
    torch.cuda.current_stream().wait_stream(s)
    torch.autograd.grad(_step1_loss(enc_e(x), fl, rd, gen_e, vgg, x, masked, tgt), params_e)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.autograd.grad(_step1_loss(enc(x), fl, rd, gen, vgg, x, masked, tgt), params)
    for step in (1, 2):                            # capture ran nothing: both have seen one step
        img, m2, t2 = data[step]
        with torch.no_grad():
            x.copy_(img.to(DEV)); masked.copy_(m2)
            for k in tgt:
                tgt[k].copy_(t2[k])
        graph.replay()
        want = torch.autograd.grad(_step1_loss(enc_e(img.to(DEV)), fl, rd, gen_e, vgg, img.to(DEV), m2, t2), params_e)
        assert all(torch.equal(a, b) for a, b in zip(out, want)), step
    assert all(torch.equal(a, b) for a, b in zip(_stats(gen).values(), _stats(gen_e).values()))
    assert all(torch.equal(a, enc_e.state_dict()[k]) for k, a in enc.state_dict().items() if "running" in k)


def test_train_step_against_the_golden_file(golden):
    """One precision-0 train step on the inputs of tests/golden/generator_train.npz (the reference's SmirkGenerator):
    output and running statistics to 1e-4; the sampled gradients are reported (cosine, asserted >= 0.99, and relative
    L2), since a flipped ReLU or pool choice changes a gradient by a whole term."""
    import smirk_b200
    import make_golden_generator_train as mg
    gold = golden("generator_train")
    sd, x, gy = mg.inputs()
    g = smirk_b200.SmirkGenerator(*mg.CFG)
    g.load_state_dict(sd)
    g = g.to(DEV).train().allow_train_mode_(True)
    y, grads = mg.step(g, x.to(DEV), gy)
    rec = mg.record(y, g.state_dict(), {k: v.cpu() for k, v in grads.items()})
    assert _err(torch.from_numpy(rec["out"]), torch.from_numpy(gold["out"])) <= 1e-4
    assert list(rec["num_batches_tracked"]) == list(gold["num_batches_tracked"])
    for i, n in enumerate(gold["stats_names"]):
        assert _err(torch.from_numpy(rec["stats_sample"][i]), torch.from_numpy(gold["stats_sample"][i])) <= 1e-4, n
    a, b = torch.from_numpy(rec["grad_sample"]).double(), torch.from_numpy(gold["grad_sample"]).double()
    cos = F.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()
    rel = ((a - b).norm() / b.norm()).item()
    worst = min(range(len(a)), key=lambda i: F.cosine_similarity(a[i], b[i], dim=0).item())
    print("golden train step: sampled gradients cosine %.6f, relative L2 %.2e (lowest per tensor: %s %.4f)"
          % (cos, rel, gold["grad_names"][worst], F.cosine_similarity(a[worst], b[worst], dim=0).item()))
    assert cos >= 0.99


def test_deterministic_and_cuda_graph(base):
    x, gy = _inputs(32, 800)
    runs = []
    for _ in range(2):
        g = _make(base, 0)
        gx, gp, y = _device_grads(g, x, gy)
        runs.append((y, gx, gp, _stats(g)))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert all(torch.equal(v, runs[1][2][k]) for k, v in runs[0][2].items())
    assert all(torch.equal(v, runs[1][3][k]) for k, v in runs[0][3].items())
    # graph: forward + backward of B = 2 captured after one eager warm-up step; replays equal eager steps
    x, gy = _inputs(2, 810)
    g, eager = _make(base, 3), _make(base, 3)
    sx, sgy = x.to(DEV).requires_grad_(), gy.to(DEV)
    params = list(g.parameters())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.autograd.grad((g(sx) * sgy).sum(), [sx] + params)
    torch.cuda.current_stream().wait_stream(s)
    _device_grads(eager, x, gy)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.autograd.grad((g(sx) * sgy).sum(), [sx] + params)
    for step in range(2):            # capture ran no kernels: the module has seen one step, as `eager` has
        x2, gy2 = _inputs(2, 820 + step)
        with torch.no_grad():
            sx.copy_(x2.to(DEV)); sgy.copy_(gy2.to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        gx, gp, _ = _device_grads(eager, x2, gy2)
        assert torch.equal(out[0], gx)
        assert all(torch.equal(a, gp[k]) for a, (k, _) in zip(out[1:], g.named_parameters()))
        assert all(torch.equal(v, _stats(eager)[k]) for k, v in _stats(g).items())
