"""GPU suite (-m gpu) for smirk_b200.VGGPerceptualLoss: the loss against the torch restatement (tests/vgg_ref.py, run
in fp32 on the same GPU), the input gradients against the replay oracle (autograd through the restatement with the
device's own ReLU masks, pool indices and L1 signs), the golden fixture of the reference class, determinism, batch
independence, the launch count, CUDA-graph capture, and the loss inside a trainer-shaped chain.

Tolerances: 1e-4 relative at precisions 0 and 3, 5e-3 at precision 1 (TF32), the generator's stated tolerances; gradients
by max-abs error over the oracle's max-abs."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from smirk_b200 import synth_inputs

import make_golden_vgg_loss as mg
import vgg_ref
from test_gpu_parity import rel_close
from test_gpu_generator_grad import gen, mods  # noqa: F401  (mods: a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_VGGS = {}
TOL = {0: 1e-4, 1: 5e-3, 3: 1e-4}


def vgg(precision=0):
    import smirk_b200
    if precision not in _VGGS:
        m = smirk_b200.VGGPerceptualLoss(weights=None)
        m.load_state_dict(mg.golden_state_dict())
        m.precision = precision
        _VGGS[precision] = m.to(DEV)
    return _VGGS[precision]


def sd_on(dev):
    return {k: v.to(dev) for k, v in mg.golden_state_dict().items()}


@contextlib.contextmanager
def fp32_cudnn():
    """The oracle's convolutions in fp32 (cuDNN's TF32 off), restored afterwards."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def inputs(B, seed):
    return synth_inputs.images(B, seed) * 2 - 1, synth_inputs.images(B, seed + 1) * 2 - 1


def device_loss_and_grads(m, x, y, need):
    xl, yl = x.to(DEV).requires_grad_(bool(need & 1)), y.to(DEV).requires_grad_(bool(need & 2))
    loss = m(xl, yl)
    wrt = [t for t in (xl, yl) if t.requires_grad]
    grads = torch.autograd.grad(loss, wrt)
    gx = grads[0] if need & 1 else None
    gy = grads[-1] if need & 2 else None
    return loss.detach(), gx, gy


def replay_grads(m, x, y):
    saved = m.saved_activations(x.to(DEV), y.to(DEV))
    xl, yl = x.to(DEV).requires_grad_(), y.to(DEV).requires_grad_()
    with fp32_cudnn():
        loss = vgg_ref.vgg_loss_replay_ref(sd_on(DEV), xl, yl, saved)
        gx, gy = torch.autograd.grad(loss, [xl, yl])
    return loss.detach(), gx, gy


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("B", [1, 2, 5, 32])
def test_loss_vs_restatement(native_lib, precision, B):
    m = vgg(precision)
    x, y = inputs(B, 500 + B)
    with torch.no_grad():
        got = m(x.to(DEV), y.to(DEV))
        with fp32_cudnn():
            ref = vgg_ref.vgg_loss_ref(sd_on(DEV), x.to(DEV), y.to(DEV))
    assert got.shape == () and got.dtype == torch.float32
    err = abs(float(got) - float(ref)) / abs(float(ref))
    print("precision %d B %d: loss %.6f, rel err %.2e" % (precision, B, float(got), err))
    assert err <= TOL[precision]


@pytest.mark.parametrize("precision", [0, 1, 3])
@pytest.mark.parametrize("need", [1, 2, 3])
@pytest.mark.parametrize("B", [1, 2, 3])
def test_input_grads_vs_replay_oracle(native_lib, precision, need, B):
    m = vgg(precision)
    x, y = inputs(B, 600 + need)
    loss, gx, gy = device_loss_and_grads(m, x, y, need)
    with torch.no_grad():
        assert torch.equal(loss, m(x.to(DEV), y.to(DEV)))            # the grad-mode forward's loss is the forward's
    rl, rgx, rgy = replay_grads(m, x, y)
    assert abs(float(rl) - float(loss)) <= TOL[precision] * abs(float(rl))
    for got, ref, want in ((gx, rgx, need & 1), (gy, rgy, need & 2)):
        if want:
            assert torch.isfinite(got).all()
            err = rel_close(got, ref, TOL[precision])
            print("precision %d need %d B %d: max-abs err / max-abs %.2e" % (precision, need, B, err / float(ref.abs().max())))
        else:
            assert got is None


@pytest.mark.parametrize("precision", [0, 3])
def test_golden(native_lib, golden, precision):
    """The reference class's loss at 1e-4.  Its gradients come from the reference's own fp32 forward, whose ReLU masks
    differ from the device's wherever an activation sits within rounding of zero, and each such flip moves the gradient
    by a whole term: their error is reported, and a gross-error guard (cosine >= 0.99) asserted, as for the generator."""
    gold = golden("vgg_loss")
    x, y = mg.golden_inputs()
    loss, gx, gy = device_loss_and_grads(vgg(precision), x, y, 3)
    err = abs(float(loss) - float(gold["loss"])) / abs(float(gold["loss"]))
    for k, got in (("g_x", gx), ("g_y", gy)):
        got, ref = mg.subsample(got).cpu().double(), torch.from_numpy(gold[k]).double()
        cos = float((got * ref).sum() / (got.norm() * ref.norm()))
        print("precision %d: loss rel err %.2e, %s max-abs err / max-abs %.2e, rel L2 %.2e, cosine %.6f"
              % (precision, err, k, float((got - ref).abs().max() / ref.abs().max()), float((got - ref).norm() / ref.norm()), cos))
        assert cos >= 0.99
    assert err <= 1e-4


def test_x_is_y_gives_exact_zeros(native_lib):
    for precision in (0, 1, 3):
        x = inputs(2, 700)[0].to(DEV).requires_grad_()
        loss = vgg(precision)(x, x)
        g, = torch.autograd.grad(loss, [x])
        assert float(loss.detach()) == 0.0 and float(g.abs().max()) == 0.0
        xd, yd = x.detach(), x.detach().clone()
        loss, gx, gy = device_loss_and_grads(vgg(precision), xd, yd, 3)
        assert float(loss) == 0.0 and float(gx.abs().max()) == 0.0 and float(gy.abs().max()) == 0.0


def test_deterministic_and_batch_independent(native_lib):
    """Also the gradients: at B = 32 each tap's scale g / numel is exactly 2^-5 of B = 1's, and fp32 and TF32 rounding
    commute with a power of two, so 32 times an image's B = 32 gradient is its B = 1 gradient bit for bit."""
    for precision in (0, 1, 3):
        m = vgg(precision)
        x, y = inputs(32, 710)
        a = device_loss_and_grads(m, x, y, 3)
        b = device_loss_and_grads(m, x, y, 3)
        assert all(torch.equal(p, q) for p, q in zip(a, b))
        full = m.saved_activations(x.to(DEV), y.to(DEV))
        for i in (0, 17):
            _, gx, gy = device_loss_and_grads(m, x[i:i + 1], y[i:i + 1], 3)
            assert torch.equal(a[1][i] * 32, gx[0]) and torch.equal(a[2][i] * 32, gy[0]), (precision, i)
            one = m.saved_activations(x[i:i + 1].to(DEV), y[i:i + 1].to(DEV))
            for k, v in one.items():
                if k.startswith("sign"):
                    assert torch.equal(v[0], full[k][i]), (precision, i, k)
                else:
                    assert torch.equal(v[0], full[k][i]) and torch.equal(v[1], full[k][32 + i]), (precision, i, k)


def test_launch_counts_and_module_properties(native_lib):
    from smirk_b200 import _lib
    L = _lib.lib()
    x, y = (t.to(DEV) for t in inputs(3, 720))
    for precision in (0, 1, 3):
        m = vgg(precision)
        m(x, y)
        n0 = L.smk_launch_count()
        l0 = m(x, y)
        n1 = L.smk_launch_count()
        l1 = m(x.clone().requires_grad_(), y)
        n2 = L.smk_launch_count()
        l1.backward()
        n3 = L.smk_launch_count()
        assert (n1 - n0, n2 - n1, n3 - n2) == (19, 19, 15), (precision, n1 - n0, n2 - n1, n3 - n2)
        assert torch.equal(l0, l1.detach()) and not l0.requires_grad
        assert torch.equal(m.train()(x, y), l0) and torch.equal(m.eval()(x, y), l0)


def test_cuda_graph_forward_backward(native_lib):
    for precision in (1, 3):
        m = vgg(precision)
        x, y = inputs(2, 730)
        sx, sy = x.to(DEV).requires_grad_(), y.to(DEV).requires_grad_()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                torch.autograd.grad(m(sx, sy), [sx, sy])
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gl = m(sx, sy)
            gx, gy = torch.autograd.grad(gl, [sx, sy])
        x2, y2 = inputs(2, 731)
        with torch.no_grad():
            sx.copy_(x2.to(DEV))
            sy.copy_(y2.to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        el, ex, ey = device_loss_and_grads(m, x2, y2, 3)
        assert torch.equal(gl.detach(), el) and torch.equal(gx, ex) and torch.equal(gy, ey)


def test_against_plain_autograd_reported(native_lib):
    """Reported, not gated: sign-map and ReLU-mask elements that differ from the oracle's own fp32 forward, relative L2
    and cosine of the gradients against plain autograd; asserted: cosine >= 0.99 (gross-error guard)."""
    x, y = mg.golden_inputs()
    sd = sd_on(DEV)
    xl, yl = x.to(DEV).requires_grad_(), y.to(DEV).requires_grad_()
    with fp32_cudnn():
        loss = vgg_ref.vgg_loss_ref(sd, xl, yl)
        rgx, rgy = torch.autograd.grad(loss, [xl, yl])
        own = vgg_ref.oracle_saved(sd, x.to(DEV), y.to(DEV))
    for precision in (0, 1, 3):
        m = vgg(precision)
        _, gx, gy = device_loss_and_grads(m, x, y, 3)
        sv = m.saved_activations(x.to(DEV), y.to(DEV))
        sign_flips = sum(int((sv[k] != own[k]).sum()) for k in vgg_ref.SIGNS)
        mask_flips = sum(int(((sv[k] > 0) != (own[k] > 0)).sum()) for k in vgg_ref.NAMES)
        got, ref = torch.cat([gx.flatten(), gy.flatten()]).double(), torch.cat([rgx.flatten(), rgy.flatten()]).double()
        rl2 = float((got - ref).norm() / ref.norm())
        cos = float((got * ref).sum() / (got.norm() * ref.norm()))
        print("precision %d: %d sign flips of %d, %d ReLU-mask flips of %d, rel L2 %.2e, cosine %.6f"
              % (precision, sign_flips, sum(own[k].numel() for k in vgg_ref.SIGNS), mask_flips,
                 sum(own[k].numel() for k in vgg_ref.NAMES), rl2, cos))
        assert cos >= 0.99


@pytest.mark.parametrize("precision", [0, 3])
def test_trainer_shaped_chain(mods, precision):  # noqa: F811
    """The reconstruction path of smirk_trainer.py: FLAME -> Renderer -> frozen generator -> 10 * VGG + L1 against the
    image, gradients to the expression, jaw and cam parameters, against the same chain through the oracles (the
    generator's and the loss's replay variants with the device's own discrete choices)."""
    from oracle import flame_ref, generator_replay_ref, grad_ref
    fl, rd, c, rc = mods
    g, v = gen(precision=precision), vgg(precision)
    B = 2
    p = synth_inputs.flame_params(B, 1300)
    img = synth_inputs.images(B, 1301)
    masked = synth_inputs.masked_images(B, 1302)
    keep = torch.ones(B, 1, 224, 224)
    grad_keys = ("expression_params", "jaw_params", "cam")

    def loss_fn(flame, render, generator, loss_vgg, leaves, masked, img):
        fo = flame(leaves)
        ro = render(fo["vertices"], leaves["cam"])
        y = generator(torch.cat([ro["rendered_img"] * keep.to(img.device), masked], 1))
        return 10.0 * loss_vgg(y, img) + F.l1_loss(y, img)
    leaves = {k: vv.clone().to(DEV).requires_grad_(k in grad_keys) for k, vv in p.items()}
    loss_fn(fl, rd, g, v, leaves, masked.to(DEV), img.to(DEV)).backward()
    with torch.no_grad():                              # the device's own choices on its own inputs
        fo_d = fl({k: t.detach() for k, t in leaves.items()})
        x_d = torch.cat([rd(fo_d["vertices"], leaves["cam"].detach())["rendered_img"], masked.to(DEV)], 1)
        g_saved = {k: t.cpu() for k, t in g.saved_activations(x_d).items()}
        v_saved = {k: t.cpu() for k, t in v.saved_activations(g(x_d), img.to(DEV)).items()}
    gsd = {k: t.cpu() for k, t in g.state_dict().items()}
    vsd = mg.golden_state_dict()
    ref_leaves = {k: vv.clone().requires_grad_(k in grad_keys) for k, vv in p.items()}
    loss_fn(lambda q: flame_ref.flame_forward_ref(c, q), lambda vv, cam: grad_ref.render_forward_grad_ref(rc, vv, cam),
            lambda xx: generator_replay_ref.generator_forward_replay_ref(gsd, xx, g_saved, res_blocks=5),
            lambda a, b: vgg_ref.vgg_loss_replay_ref(vsd, a, b, v_saved), ref_leaves, masked, img).backward()
    for k in grad_keys:
        assert torch.isfinite(leaves[k].grad).all(), k
        err = rel_close(leaves[k].grad, ref_leaves[k].grad, 1e-4)
        print("precision %d %s: max-abs err / max-abs %.2e" % (precision, k, err / float(ref_leaves[k].grad.abs().max())))
    assert float(leaves["cam"].grad.abs().max()) > 0
