"""GPU suite for the encoder's input gradient (a frozen, eval-mode SmirkEncoder under autograd).

g_img is checked against the mask-replay oracle (oracle/encoder_replay_ref.py: autograd through the oracle forward with
the device's own ReLU / clamp choices), against plain autograd and the golden file of the reference module (reported:
mask flips, relative L2, cosine), and for the properties of the autograd path: grad-mode forward outputs and launches,
None upstream gradients, frozen-weights / train-mode errors, the trainer's freeze state, a generator -> encoder cycle
chain, determinism, batch independence, CUDA-graph capture and two forwards sharing one backward."""
import copy

import pytest
import torch

from smirk_b200 import synth_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ("pose_params", "cam", "shape_params", "expression_params", "eyelid_params", "jaw_params")
TOL = {0: 1e-4, 1: 5e-3, 2: 5e-3, 3: 1e-4}
LARGE, SMALL = 46, 34                   # backward launches per backbone: head, cn, 3 per inverted-residual block, 2 for block 0


@pytest.fixture(scope="module")
def encoder(native_lib):
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    return enc.eval().requires_grad_(False).to(DEV)


def _with(enc, precision):
    e = copy.deepcopy(enc)
    e.precision = precision
    for name in ("pose_encoder", "shape_encoder", "expression_encoder"):
        if hasattr(e, name):
            getattr(e, name).precision = precision
    return e


def _upstream(B, seed=5):
    g = torch.Generator().manual_seed(seed)
    widths = {"pose_params": 3, "cam": 3, "shape_params": 300, "expression_params": 50, "eyelid_params": 2, "jaw_params": 3}
    return {k: torch.randn(B, w, generator=g) for k, w in widths.items()}


def _loss(out, up):
    return sum((out[k] * up[k].to(out[k].device)).sum() for k in out)


def _device_grad(enc, img, up):
    x = img.to(DEV).requires_grad_()
    out = enc(x)
    g, = torch.autograd.grad(_loss(out, up), x)
    return out, g.cpu()


def _replay_grad(enc, img, up, sub=None):
    """g_img of the replay oracle fed the device's saved tensors (sub: the sub-encoder's module path, or None)."""
    from oracle import encoder_replay_ref as rr
    sd = {k: v.cpu() for k, v in enc.state_dict().items()}
    if sub is not None:                                   # a sub-encoder's state dict lives under its path in a SmirkEncoder
        import smirk_b200
        full = smirk_b200.SmirkEncoder().eval().requires_grad_(False)
        sd = {sub + "." + k: v for k, v in sd.items()}
        sd.update({k: v for k, v in full.state_dict().items() if not k.startswith(sub + ".")})
    saved = {k: v.cpu() for k, v in enc.saved_activations(img.to(DEV)).items()}
    if sub is not None:                                   # the absent backbones get no gradient: any masks do
        ref_act = rr.encoder_activations_ref(sd, img)[1]
        saved = {k: saved.get(k, ref_act[k].detach()) for k in rr.saved_names()}
    x = img.clone().requires_grad_()
    out = rr.encoder_forward_replay_ref(sd, x, saved)
    g, = torch.autograd.grad(sum((out[k] * up[k]).sum() for k in up), x)
    return g


def _gate(g, ref, tol):
    err = (g - ref).abs().max().item() / ref.abs().max().item()
    assert err <= tol, err
    return err


@pytest.mark.parametrize("precision", [0, 1, 2, 3])
@pytest.mark.parametrize("B", [1, 3])
def test_input_gradient_matches_replay_oracle(encoder, precision, B):
    enc = _with(encoder, precision)
    img, up = synth_inputs.images(B, 900 + B), _upstream(B)
    _, g = _device_grad(enc, img, up)
    err = _gate(g, _replay_grad(enc, img, up), TOL[precision])
    print("precision %d B %d: max-abs error / max-abs = %.2e" % (precision, B, err))


@pytest.mark.parametrize("precision", [0, 3])
def test_input_gradient_at_batch_32(encoder, precision):
    enc = _with(encoder, precision)
    img, up = synth_inputs.images(32, 932), _upstream(32)
    _, g = _device_grad(enc, img, up)
    _gate(g, _replay_grad(enc, img, up), TOL[precision])


@pytest.mark.parametrize("precision", [0, 3])
@pytest.mark.parametrize("sub", ["pose_encoder", "shape_encoder", "expression_encoder"])
def test_sub_encoder_alone(encoder, precision, sub):
    enc = _with(getattr(encoder, sub), precision)
    img = synth_inputs.images(2, 941)
    out0 = enc(img.to(DEV))
    up = {k: v for k, v in _upstream(2).items() if k in out0}
    _, g = _device_grad(enc, img, up)
    _gate(g, _replay_grad(enc, img, up, sub=sub), TOL[precision])


@pytest.mark.parametrize("precision", [0, 3])
def test_each_upstream_output_alone_and_none_launches_nothing(encoder, precision):
    from smirk_b200 import _lib
    L = _lib.lib()
    enc = _with(encoder, precision)
    img = synth_inputs.images(2, 951)
    up_all = _upstream(2)
    for key, launches in (("cam", SMALL + 1), ("shape_params", LARGE + 1), ("jaw_params", LARGE + 1)):
        up = {key: up_all[key]}
        x = img.to(DEV).requires_grad_()
        out = enc(x)
        loss = _loss({key: out[key]}, up)
        torch.cuda.synchronize()
        n0 = L.smk_launch_count()
        g, = torch.autograd.grad(loss, x)
        torch.cuda.synchronize()
        assert L.smk_launch_count() - n0 == launches, key
        _gate(g.cpu(), _replay_grad(enc, img, up), TOL[precision])


def test_flips_and_cosine_against_autograd_and_golden(encoder, golden):
    """The device's masks against the oracle's own (flip counts) and g_img against plain autograd and the reference's
    golden file: reported; cosine >= 0.99 asserted."""
    from oracle import encoder_replay_ref as rr, make_golden_encoder_grad as mg
    sd = {k: v.cpu() for k, v in encoder.state_dict().items()}
    img = mg.encoder_input()
    x = img.clone().requires_grad_()
    out, act = rr.encoder_activations_ref(sd, x)
    g_ref, = torch.autograd.grad(rr.loss(out, mg.upstream()), x)
    gold = golden("encoder_grad")
    for precision in (0, 3):
        enc = _with(encoder, precision)
        dev = enc.saved_activations(img.to(DEV))
        flips = sum(int(((dev[k].cpu() > 0) != (act[k].detach() > 0)).sum()) for k in act if ".encoder." in k)
        _, g = _device_grad(enc, img, mg.upstream())
        rel = ((g - g_ref).norm() / g_ref.norm()).item()
        cos = torch.nn.functional.cosine_similarity(g.flatten().double(), g_ref.flatten().double(), dim=0).item()
        gs = torch.from_numpy(gold["g_img_sub"]).double()
        cos_g = torch.nn.functional.cosine_similarity(g[:, :, ::4, ::4].flatten().double(), gs.flatten(), dim=0).item()
        print("precision %d: %d mask flips, rel L2 %.2e, cosine %.6f (autograd) %.6f (golden)" % (precision, flips, rel, cos, cos_g))
        assert cos >= 0.99 and cos_g >= 0.99


@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_grad_mode_forward_is_the_forward(encoder, precision):
    from smirk_b200 import _lib
    L = _lib.lib()
    enc = _with(encoder, precision)
    img = synth_inputs.images(3, 961).to(DEV)
    enc(img)                                                   # handle and workspaces exist
    torch.cuda.synchronize(); n0 = L.smk_launch_count()
    with torch.no_grad():
        a = enc(img)
    torch.cuda.synchronize(); n1 = L.smk_launch_count()
    b = enc(img.clone().requires_grad_())
    torch.cuda.synchronize(); n2 = L.smk_launch_count()
    assert n2 - n1 == n1 - n0
    for k in KEYS:
        assert torch.equal(a[k], b[k].detach()), k
        assert b[k].requires_grad
    c = enc(img)                                               # an image that needs no grad: the forward-only path
    assert all(not c[k].requires_grad and torch.equal(c[k], a[k]) for k in KEYS)


def test_unfrozen_and_train_mode_raise(encoder):
    img = synth_inputs.images(1, 971).to(DEV).requires_grad_()
    e = copy.deepcopy(encoder)
    e.shape_encoder.shape_layers[0].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match=r"requires_grad_\(False\)"):
        e(img)
    e.expression_encoder(img)                                  # the expression encoder alone is frozen: runs
    e = copy.deepcopy(encoder).train()
    with pytest.raises(RuntimeError, match="train-mode"):
        e(img)
    with pytest.raises(RuntimeError, match="train-mode"):
        e(img.detach())


def _freeze_module(m):                                         # the reference's utils.freeze_module
    m.requires_grad_(False)
    m.eval()


def test_trainer_freeze_state_and_generator_encoder_cycle_chain(encoder):
    """The reference trainer's cycle path: parent SmirkEncoder in train mode, its three sub-encoders frozen by
    freeze_module; a frozen generator renders the image the encoder reads; the cycle loss (expression, jaw, eyelid,
    shape MSE) reaches the generator's input only through the encoder's input gradient.  Against the oracle chain with
    the device's choices, precision 0."""
    import smirk_b200
    from oracle import encoder_replay_ref as rr, generator_replay_ref as gr
    enc = copy.deepcopy(encoder)
    enc.train()
    for m in (enc.pose_encoder, enc.shape_encoder, enc.expression_encoder):
        _freeze_module(m)
    gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
    gen = gen.eval().requires_grad_(False).to(DEV)
    B = 2
    x = torch.cat([synth_inputs.images(B, 981), synth_inputs.images(B, 982)], 1)
    tg = torch.Generator().manual_seed(9)
    target = {"expression_params": torch.randn(B, 50, generator=tg), "jaw_params": torch.randn(B, 3, generator=tg) * 0.1,
              "eyelid_params": torch.rand(B, 2, generator=tg), "shape_params": torch.randn(B, 300, generator=tg)}

    def cycle(feats):
        return sum(torch.nn.functional.mse_loss(feats[k], target[k].to(feats[k].device)) for k in target)

    xd = x.to(DEV).requires_grad_()
    y = gen(xd)
    gx, = torch.autograd.grad(cycle(enc(y)), xd)
    # oracle chain with the device's choices
    gsd = {k: v.cpu() for k, v in gen.state_dict().items()}
    esd = {k: v.cpu() for k, v in enc.state_dict().items()}
    gsv = {k: v.cpu() for k, v in gen.saved_activations(x.to(DEV)).items()}
    esv = {k: v.cpu() for k, v in enc.saved_activations(y.detach()).items()}
    xr = x.clone().requires_grad_()
    yr = gr.generator_forward_replay_ref(gsd, xr, gsv)
    feats = rr.encoder_forward_replay_ref(esd, yr, esv)
    gxr, = torch.autograd.grad(cycle(feats), xr)
    _gate(gx.cpu(), gxr, 1e-4)


def test_determinism_batch_independence_graph_and_shared_backward(encoder):
    enc = _with(encoder, 3)
    img, up = synth_inputs.images(32, 991), _upstream(32)
    _, g1 = _device_grad(enc, img, up)
    _, g2 = _device_grad(enc, img, up)
    assert torch.equal(g1, g2)                                 # bitwise deterministic
    big = synth_inputs.images(256, 992)
    big[5:8] = img[:3]
    upb = {k: torch.cat([v[:5] * 0, v[:3], torch.zeros(248, v.shape[1])]) for k, v in _upstream(32).items()}
    ups = {k: v[5:8] for k, v in upb.items()}
    _, gb = _device_grad(enc, big, upb)
    _, gs = _device_grad(enc, img[:3], ups)
    assert (gb[5:8] - gs).abs().max() <= 1e-5 * gs.abs().max()     # rows independent of the batch
    assert gb[:5].abs().max() == 0 and gb[8:].abs().max() == 0
    # two forwards, one backward: each keeps its own activations
    a, b = synth_inputs.images(2, 993), synth_inputs.images(2, 994)
    xa, xb = a.to(DEV).requires_grad_(), b.to(DEV).requires_grad_()
    upa = _upstream(2, 1)
    loss = _loss(enc(xa), upa) + _loss(enc(xb), upa)
    ga, gb2 = torch.autograd.grad(loss, [xa, xb])
    assert torch.equal(ga.cpu(), _device_grad(enc, a, upa)[1]) and torch.equal(gb2.cpu(), _device_grad(enc, b, upa)[1])
    # CUDA graph of forward + backward
    x = img[:4].to(DEV).clone().requires_grad_()
    upd = {k: v[:4].to(DEV) for k, v in up.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            gw, = torch.autograd.grad(_loss(enc(x), upd), x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gg, = torch.autograd.grad(_loss(enc(x), upd), x)
    with torch.no_grad():
        x.copy_(img[4:8].to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gg.cpu(), _device_grad(enc, img[4:8], {k: v[:4] for k, v in up.items()})[1])
