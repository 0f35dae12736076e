"""GPU suite (-m gpu) for smirk_b200.ExpressionLoss: the features and the loss against the torch restatement
(tests/expression_ref.py, run in fp32 on the same GPU with cuDNN's TF32 off), the input gradients against the replay oracle
(autograd in float64 through the restatement with the device's own ReLU masks and pool taps), the golden fixture of the
reference class, determinism, batch independence, CUDA-graph capture, and the loss inside a trainer-shaped chain.

Probe pairs: gen = expression_ref.probe_images (smooth face-like images in [0, 1]), tar = gen + 0.3 N(0, 1) pixel noise,
clamped to [0, 1] (expression_ref.perturbed): per-face l2 about 1.3, cos about 9e-3.  Errors are max-abs error over max-abs: 1e-4 at precisions 0 and 3; at precision 1 5e-3, or
twice cuDNN TF32's own error on the same problem where that is larger."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from smirk_b200 import synth_inputs

import expression_ref
import make_golden_expression_loss as mg
from test_gpu_parity import rel_close
from test_gpu_generator_grad import gen as generator, mods  # noqa: F401  (mods: a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_MODS = {}
TOL = {0: 1e-4, 1: 5e-3, 3: 1e-4}
METRICS = ("l2", "l1", "cos")


def expr(precision=0):
    import smirk_b200
    if precision not in _MODS:
        m = smirk_b200.ExpressionLoss(checkpoint=None)
        m.load_state_dict(mg.golden_state_dict())
        m.precision = precision
        _MODS[precision] = m.to(DEV)
    return _MODS[precision]


def sd_on(dev, dtype=torch.float32):
    return {k: (v.to(dev, dtype) if v.is_floating_point() else v.to(dev)) for k, v in mg.golden_state_dict().items()}


@contextlib.contextmanager
def cudnn_tf32(on):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = on
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def pair(B, seed):
    gen = expression_ref.probe_images(B, seed)
    return gen, expression_ref.perturbed(gen, seed)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max())


def device_loss_and_grads(m, gen, tar, need, use_mean=False, metric="l2"):
    gl, tl = gen.to(DEV).requires_grad_(bool(need & 1)), tar.to(DEV).requires_grad_(bool(need & 2))
    loss = m(gl, tl, use_mean=use_mean, metric=metric)
    wrt = [t for t in (gl, tl) if t.requires_grad]
    grads = torch.autograd.grad(loss.sum(), wrt)
    return loss.detach(), grads[0] if need & 1 else None, grads[-1] if need & 2 else None


def replay_grads(m, gen, tar, use_mean, metric):
    saved = m.saved_activations(gen.to(DEV), tar.to(DEV))
    gl, tl = gen.to(DEV, torch.float64).requires_grad_(), tar.to(DEV, torch.float64).requires_grad_()
    loss = expression_ref.expression_loss_replay_ref(sd_on(DEV, torch.float64), gl, tl, saved, use_mean, metric)
    gg, gt = torch.autograd.grad(loss.sum(), [gl, tl])
    return loss.detach(), gg, gt


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("B", [1, 2, 5, 32])
def test_features_and_loss_vs_restatement(native_lib, precision, B):
    m = expr(precision)
    gen, tar = (t.to(DEV) for t in pair(B, 100 + B))
    sd = sd_on(DEV)
    with torch.no_grad():
        with cudnn_tf32(False):
            rf = expression_ref.backbone_ref(sd, gen)
            rft = expression_ref.backbone_ref(sd, tar)
        with cudnn_tf32(True):
            tf = expression_ref.backbone_ref(sd, gen)
        tol = TOL[precision] if precision != 1 else max(TOL[1], 2 * rel(tf, rf))
        f = m.features(gen)
        assert f.shape == (B, 2048) and f.dtype == torch.float32
        ferr = rel(f, rf)
        print("precision %d B %d: features err %.2e (cuDNN TF32 %.2e)" % (precision, B, ferr, rel(tf, rf)))
        assert ferr <= tol
        for metric in METRICS:
            for use_mean in (True, False):
                got = m(gen, tar, use_mean=use_mean, metric=metric)
                ref = expression_ref.metric_ref(rf, rft, use_mean, metric)
                assert got.shape == ref.shape and got.dtype == torch.float32
                err = rel(got, ref)
                print("  %s use_mean %d: loss %.6g, err / loss %.2e" % (metric, use_mean, float(ref.abs().max()), err))
                assert err <= tol, (metric, use_mean)


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("need", [1, 2, 3])
@pytest.mark.parametrize("metric", METRICS)
def test_input_grads_vs_replay_oracle(native_lib, precision, need, metric):
    m = expr(precision)
    B, use_mean = 2, need != 2
    gen, tar = pair(B, 200 + need)
    loss, gg, gt = device_loss_and_grads(m, gen, tar, need, use_mean, metric)
    with torch.no_grad():
        assert torch.equal(loss, m(gen.to(DEV), tar.to(DEV), use_mean=use_mean, metric=metric))   # grad-mode forward = forward
    rl, rgg, rgt = replay_grads(m, gen, tar, use_mean, metric)
    assert rel(loss, rl) <= TOL[precision]
    for got, ref, want in ((gg, rgg, need & 1), (gt, rgt, need & 2)):
        if want:
            assert torch.isfinite(got).all()
            err = rel_close(got, ref, TOL[precision])
            print("precision %d need %d %s: max-abs err / max-abs %.2e" % (precision, need, metric, err / float(ref.abs().max())))
        else:
            assert got is None


def test_golden(native_lib, golden):
    gold = golden("expression_loss")
    gen, tar = (t.to(DEV) for t in mg.golden_inputs())
    m = expr(0)
    with torch.no_grad():
        assert rel(m.features(gen).cpu(), torch.from_numpy(gold["features_gen"])) <= 1e-4
        assert rel(m.features(tar).cpu(), torch.from_numpy(gold["features_tar"])) <= 1e-4
        for metric in METRICS:
            assert rel(m(gen, tar, True, metric).cpu(), torch.from_numpy(gold["loss_%s_mean" % metric])) <= 1e-4
            assert rel(m(gen, tar, False, metric).cpu(), torch.from_numpy(gold["loss_%s" % metric])) <= 1e-4
    gl = gen.clone().requires_grad_()
    g, = torch.autograd.grad(m(gl, tar, metric="l2", use_mean=False).mean(), [gl])
    got, ref = mg.subsample(g).cpu().double(), torch.from_numpy(gold["g_gen"]).double()
    cos = float((got * ref).sum() / (got.norm() * ref.norm()))
    print("golden: g_gen max-abs err / max-abs %.2e, cosine %.6f" % (rel(got, ref), cos))
    assert cos >= 0.99


def test_against_plain_autograd_reported(native_lib):
    """Reported, not gated: ReLU-mask and argmax flips against the oracle's own fp32 forward, relative L2 and cosine of
    the gradients against plain autograd; asserted: cosine >= 0.99 (gross-error guard)."""
    gen, tar = pair(2, 300)
    sd = sd_on(DEV)
    gl, tl = gen.to(DEV).requires_grad_(), tar.to(DEV).requires_grad_()
    with cudnn_tf32(False):
        rgg, rgt = torch.autograd.grad(expression_ref.expression_loss_ref(sd, gl, tl, True, "l2"), [gl, tl])
        own = expression_ref.oracle_saved(sd, gen.to(DEV), tar.to(DEV))
    for precision in (0, 1, 3):
        m = expr(precision)
        _, gg, gt = device_loss_and_grads(m, gen, tar, 3, True, "l2")
        sv = m.saved_activations(gen.to(DEV), tar.to(DEV))
        mask_flips = sum(int(((sv[k] > 0) != (own[k] > 0)).sum()) for k in expression_ref.names())
        arg_flips = int((sv["pool_argmax"] != own["pool_argmax"]).sum())
        got, ref = torch.cat([gg.flatten(), gt.flatten()]).double(), torch.cat([rgg.flatten(), rgt.flatten()]).double()
        rl2 = float((got - ref).norm() / ref.norm())
        cos = float((got * ref).sum() / (got.norm() * ref.norm()))
        print("precision %d: %d ReLU-mask flips of %d, %d argmax flips of %d, rel L2 %.2e, cosine %.6f"
              % (precision, mask_flips, sum(own[k].numel() for k in expression_ref.names()), arg_flips,
                 own["pool_argmax"].numel(), rl2, cos))
        assert cos >= 0.99


def test_bitwise_properties(native_lib):
    """Reproducible loss and gradient, the per-face loss of a face independent of the batch, the no-grad and grad-mode
    forwards equal."""
    for precision in (0, 1, 3):
        m = expr(precision)
        gen, tar = pair(5, 400)
        a = device_loss_and_grads(m, gen, tar, 3, False, "cos")
        b = device_loss_and_grads(m, gen, tar, 3, False, "cos")
        assert all(torch.equal(p, q) for p, q in zip(a, b))
        with torch.no_grad():
            for metric in METRICS:
                full = m(gen.to(DEV), tar.to(DEV), use_mean=False, metric=metric)
                for i in (0, 3):
                    one = m(gen[i:i + 1].to(DEV), tar[i:i + 1].to(DEV), use_mean=False, metric=metric)
                    assert torch.equal(one[0], full[i]), (precision, metric, i)
        _, gg1, gt1 = device_loss_and_grads(m, gen[3:4], tar[3:4], 3, False, "cos")
        assert torch.equal(gg1[0], a[1][3]) and torch.equal(gt1[0], a[2][3])


def test_cuda_graph_forward_backward(native_lib):
    for precision in (1, 3):
        m = expr(precision)
        gen, tar = pair(2, 500)
        sg, stg = gen.to(DEV).requires_grad_(), tar.to(DEV).requires_grad_()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                torch.autograd.grad(m(sg, stg, metric="cos"), [sg, stg])
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gl = m(sg, stg, metric="cos")
            gg, gt = torch.autograd.grad(gl, [sg, stg])
        g2, t2 = pair(2, 501)
        with torch.no_grad():
            sg.copy_(g2.to(DEV))
            stg.copy_(t2.to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        el, eg, et = device_loss_and_grads(m, g2, t2, 3, True, "cos")
        assert torch.equal(gl.detach(), el) and torch.equal(gg, eg) and torch.equal(gt, et)


@pytest.mark.parametrize("precision", [0, 3])
def test_trainer_shaped_chain(mods, precision):  # noqa: F811
    """smirk_trainer.py's emotion-loss path: FLAME -> Renderer -> masking -> frozen eval generator ->
    ExpressionLoss(recon, img, metric='l2', use_mean=False).mean(), gradients to the expression, jaw and cam parameters,
    against the same chain through the oracles (the generator's and the loss's replay variants with the device's own
    discrete choices; the loss's in float64), at 2e-4."""
    from oracle import flame_ref, generator_replay_ref, grad_ref
    fl, rd, c, rc = mods
    g, e = generator(precision=precision), expr(precision)
    B = 2
    p = synth_inputs.flame_params(B, 1400)
    img = synth_inputs.images(B, 1401)
    masked = synth_inputs.masked_images(B, 1402)
    keep = torch.ones(B, 1, 224, 224)
    grad_keys = ("expression_params", "jaw_params", "cam")

    def loss_fn(flame, render, generator_, loss_e, leaves, masked, img):
        fo = flame(leaves)
        ro = render(fo["vertices"], leaves["cam"])
        y = generator_(torch.cat([ro["rendered_img"] * keep.to(img.device), masked], 1))
        return loss_e(y, img).mean()
    leaves = {k: vv.clone().to(DEV).requires_grad_(k in grad_keys) for k, vv in p.items()}
    loss_fn(fl, rd, g, lambda a, b: e(a, b, metric="l2", use_mean=False), leaves, masked.to(DEV), img.to(DEV)).backward()
    with torch.no_grad():                              # the device's own choices on its own inputs
        fo_d = fl({k: t.detach() for k, t in leaves.items()})
        x_d = torch.cat([rd(fo_d["vertices"], leaves["cam"].detach())["rendered_img"], masked.to(DEV)], 1)
        g_saved = {k: t.cpu() for k, t in g.saved_activations(x_d).items()}
        e_saved = {k: t.cpu() for k, t in e.saved_activations(g(x_d), img.to(DEV)).items()}
    gsd = {k: t.cpu() for k, t in g.state_dict().items()}
    esd = {k: (v.double() if v.is_floating_point() else v) for k, v in mg.golden_state_dict().items()}
    ref_leaves = {k: vv.clone().requires_grad_(k in grad_keys) for k, vv in p.items()}
    loss_fn(lambda q: flame_ref.flame_forward_ref(c, q), lambda vv, cam: grad_ref.render_forward_grad_ref(rc, vv, cam),
            lambda xx: generator_replay_ref.generator_forward_replay_ref(gsd, xx, g_saved, res_blocks=5),
            lambda a, b: expression_ref.expression_loss_replay_ref(esd, a.double(), b.double(), e_saved, False, "l2"), ref_leaves,
            masked, img).backward()
    for k in grad_keys:
        assert torch.isfinite(leaves[k].grad).all(), k
        # 2e-4: the oracle chain runs the generator and renderer in fp32 on the CPU (generator_ref casts its weights to
        # fp32); on H100 the device chain measured 1.03e-4 (cam, precision 0) and 6.5e-5 (precision 3) from it.
        err = rel_close(leaves[k].grad, ref_leaves[k].grad, 2e-4)
        print("precision %d %s: max-abs err / max-abs %.2e" % (precision, k, err / float(ref_leaves[k].grad.abs().max())))
    assert float(leaves["cam"].grad.abs().max()) > 0
