"""Live eval handles (``live_weights_(True)``): the eval path of SmirkEncoder, each sub-encoder and SmirkGenerator on weights
refreshed on the device from the module's tensors is bitwise the host-packed handle's — outputs, saved activations and
input gradient, with random weights and running statistics — also after optimizer steps in train mode (no handle
rebuilt, no host sync), and in a CUDA graph replayed after new weights are copied in.  The refresh adds its pinned launch
count; a weight modified in place before the backward raises autograd's version error; a live handle never refreshed
fails with the library's message."""
import copy
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GEN_CFG = (6, 3, 32, 5)
BATCHES = (1, 7, 32)
# Refresh launches (include/smirk_b200_live.h): fold batches of 160 BatchNorms + pack batches of 40 jobs.
REFRESH_LAUNCHES = {None: 1 + 7, "pose_encoder": 1 + 2, "shape_encoder": 1 + 3, "expression_encoder": 1 + 3, "generator": 1 + 2}


@pytest.fixture(scope="module")
def enc_base(native_lib):
    import smirk_b200
    from smirk_b200 import synth_inputs
    m = smirk_b200.SmirkEncoder()
    m.load_state_dict(synth_inputs.random_state_dict(m.state_dict(), seed=21))
    return m


@pytest.fixture(scope="module")
def gen_base(native_lib):
    import smirk_b200
    from smirk_b200 import synth_inputs
    m = smirk_b200.SmirkGenerator(*GEN_CFG)
    m.load_state_dict(synth_inputs.random_state_dict(m.state_dict(), seed=22))
    return m


def _set_precision(m, p):
    for k in m.modules():
        if hasattr(k, "precision"):
            k.precision = p
    return m


def _encoder(base, part, precision, live):
    m = _set_precision(copy.deepcopy(base).to(DEV).eval().requires_grad_(False), precision)
    m.live_weights_(live)
    return m if part is None else getattr(m, part)


def _images(B, seed, C=3):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, C, 224, 224, generator=g).to(DEV)


def _outputs(out):
    return [out[k] for k in sorted(out)] if isinstance(out, dict) else [out]


def _run(m, x, seed):
    """-> (no-grad outputs, saved activations, input gradient of a fixed random projection of the outputs)."""
    with torch.no_grad():
        y = _outputs(m(x))
    sv = m.saved_activations(x)
    xi = x.clone().requires_grad_()
    out = _outputs(m(xi))
    g = torch.Generator().manual_seed(seed)
    loss = sum((o * torch.randn(o.shape, generator=g).to(DEV)).sum() for o in out)
    gx, = torch.autograd.grad(loss, xi)
    return y, sv, gx


def _same(a, b):
    ya, sa, ga = a
    yb, sb, gb = b
    assert len(ya) == len(yb) and all(torch.equal(u, v) for u, v in zip(ya, yb))
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa), [k for k in sa if not torch.equal(sa[k], sb[k])]
    assert torch.equal(ga, gb)


@pytest.mark.parametrize("part", [None, "pose_encoder", "shape_encoder", "expression_encoder"])
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_encoder_live_equals_host_handle(enc_base, part, precision):
    host, live = _encoder(enc_base, part, precision, False), _encoder(enc_base, part, precision, True)
    for B in BATCHES:
        x = _images(B, 100 + B)
        _same(_run(live, x, B), _run(host, x, B))
    assert live._native.handle is None and live._native.live_handle is not None


@pytest.mark.parametrize("precision", [0, 1, 3])
def test_generator_live_equals_host_handle(gen_base, precision):
    host = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False)
    live = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False).live_weights_(True)
    host.precision = live.precision = precision
    for B in BATCHES:
        x = _images(B, 200 + B, GEN_CFG[0])
        _same(_run(live, x, B), _run(host, x, B))
    assert live._native.handle is None and live._native.live_handle is not None


def _train_steps(m, make_x, steps=3):
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    for s in range(steps):
        out = _outputs(m(make_x(s)))
        loss = sum((o ** 2).mean() for o in out)
        opt.zero_grad()
        loss.backward()
        opt.step()


@pytest.mark.parametrize("which", ["encoder", "generator"])
def test_live_eval_after_optimizer_steps_needs_no_rebuild(enc_base, gen_base, which):
    if which == "encoder":
        m = _set_precision(copy.deepcopy(enc_base).to(DEV), 3)
        cin = 3
    else:
        m = copy.deepcopy(gen_base).to(DEV)
        m.precision, cin = 3, GEN_CFG[0]
    m.allow_train_mode_(True).live_weights_(True)
    x = _images(4, 300, cin)
    with torch.no_grad():
        m.eval()(x)                                      # the live handle exists before the steps
    h = m._native.live_handle
    m.train()
    _train_steps(m, lambda s: _images(4, 310 + s, cin))
    m.eval()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            y = _outputs(m(x))
        xi = x.clone().requires_grad_()
        m.requires_grad_(False)
        gx, = torch.autograd.grad(sum(o.sum() for o in _outputs(m(xi))), xi)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m._native.live_handle is h and m._native.handle is None
    ref = copy.deepcopy(m).live_weights_(False)
    with torch.no_grad():
        y_ref = _outputs(ref(x))
    xr = x.clone().requires_grad_()
    g_ref, = torch.autograd.grad(sum(o.sum() for o in _outputs(ref(xr))), xr)
    assert all(torch.equal(a, b) for a, b in zip(y, y_ref)) and torch.equal(gx, g_ref)


def _copy_new_values(m, seed):
    from smirk_b200 import synth_inputs
    new = synth_inputs.random_state_dict(m.state_dict(), seed=seed)
    with torch.no_grad():
        for k, v in m.state_dict(keep_vars=True).items():
            v.copy_(new[k])


@pytest.mark.parametrize("which", ["encoder", "generator"])
def test_captured_live_eval_reads_the_weights_of_replay_time(enc_base, gen_base, which):
    if which == "encoder":
        m, cin = _encoder(enc_base, None, 3, True), 3
    else:
        m = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False).live_weights_(True)
        m.precision, cin = 3, GEN_CFG[0]
    x = _images(2, 400, cin).requires_grad_()

    def step():
        out = _outputs(m(x))
        return [o.detach() for o in out], torch.autograd.grad(sum((o * (k + 1)).sum() for k, o in enumerate(out)), x)[0]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for seed in (31, 32):
        _copy_new_values(m, seed)
        graph.replay()
        ref = copy.deepcopy(m).live_weights_(False)
        xr = x.detach().clone().requires_grad_()
        out = _outputs(ref(xr))
        g_ref, = torch.autograd.grad(sum((o * (k + 1)).sum() for k, o in enumerate(out)), xr)
        assert all(torch.equal(a, b.detach()) for a, b in zip(static[0], out)) and torch.equal(static[1], g_ref), seed


@pytest.mark.parametrize("part", [None, "pose_encoder", "shape_encoder", "expression_encoder", "generator"])
def test_refresh_adds_its_pinned_launches(enc_base, gen_base, part):
    from smirk_b200 import _lib
    L = _lib.lib()
    if part == "generator":
        mods = [copy.deepcopy(gen_base).to(DEV).eval() for _ in range(2)]
        mods[1].live_weights_(True)
        x = _images(2, 500, GEN_CFG[0])
    else:
        mods = [_encoder(enc_base, part, 3, live) for live in (False, True)]
        x = _images(2, 500)
    counts = []
    for m in mods:
        with torch.no_grad():
            m(x)                                         # handles and workspaces exist
            n0 = L.smk_launch_count()
            m(x)
        counts.append(L.smk_launch_count() - n0)
    assert counts[1] - counts[0] == REFRESH_LAUNCHES[part], counts


@pytest.mark.parametrize("which", ["encoder", "generator"])
def test_weight_modified_before_backward_raises(enc_base, gen_base, which):
    if which == "encoder":
        m, cin = _encoder(enc_base, None, 0, True), 3
        w = m.shape_encoder.encoder.conv_stem.weight
    else:
        m = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False).live_weights_(True)
        cin, w = GEN_CFG[0], m.decoder1.dec1conv1.weight
    x = _images(1, 600, cin).requires_grad_()
    loss = sum(o.sum() for o in _outputs(m(x)))
    with torch.no_grad():
        w.mul_(1.5)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()


def test_two_forwards_one_backward_refresh_again(gen_base):
    m = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False).live_weights_(True)
    host = copy.deepcopy(gen_base).to(DEV).eval().requires_grad_(False)
    m.precision = host.precision = 3
    a, b = _images(2, 700, 6).requires_grad_(), _images(2, 710, 6).requires_grad_()
    ga, gb = torch.autograd.grad(m(a).sum() + (2 * m(b)).sum(), [a, b])
    ar, br = a.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    ra, rb = torch.autograd.grad(host(ar).sum() + (2 * host(br)).sum(), [ar, br])
    assert torch.equal(ga, ra) and torch.equal(gb, rb)


def test_unrefreshed_live_handle_fails(native_lib):
    from smirk_b200 import _lib
    img = torch.zeros(1, 3, 224, 224, device=DEV)
    for kind, args in (("encoder", (7, 300, 50, 3)), ("generator", GEN_CFG + (1,))):
        h = C.c_void_p()
        _lib.call("smk_%s_live_create" % kind, DEV, *args, C.byref(h))
        h = _lib.NativeHandle(h, "smk_%s_destroy" % kind)
        ws = torch.empty(_lib.call("smk_%s_workspace_bytes" % kind, DEV, h, 1), dtype=torch.uint8, device=DEV)
        if kind == "encoder":
            outs = [torch.empty(1, n, device=DEV) for n in (6, 300, 55)]
            fwd = lambda: _lib.call("smk_encoder_forward", DEV, h, img, 1, *outs, ws, ws.numel())
        else:
            x, y = torch.zeros(1, 6, 224, 224, device=DEV), torch.empty(1, 3, 224, 224, device=DEV)
            fwd = lambda: _lib.call("smk_generator_forward", DEV, h, x, 1, y, ws, ws.numel())
        with pytest.raises(RuntimeError, match="never set: call smk_%s_refresh" % kind):
            fwd()
