"""GPU suite (-m gpu) for the backward passes: FLAME and Renderer gradients (smk_flame_backward,
smk_renderer_backward, smk_project_points_backward) through the reference-signature modules, against
torch autograd through the CPU oracle (oracle/flame_ref.py, oracle/grad_ref.py) on the same seeded
inputs.  Metric: rel_close of test_gpu_parity (max-abs error <= 1e-4 x max-abs of the oracle, per tensor).

Clamp-boundary rule: torch.clamp passes the gradient on [0, 1] inclusive, so a pixel whose n.l lies
within 1e-5 of 0 or 1 can switch sides between two correct fp32 implementations.  Such pixels get a
zero upstream gradient in both runs (the tolerance is not loosened instead)."""
import pytest
import torch
import torch.nn.functional as F

from smirk_b200 import synth_inputs

from test_gpu_parity import rel_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OUTS = {"vertices": 5023, "landmarks_fan": 68, "landmarks_fan_3d": 68, "landmarks_mp": 105}


@pytest.fixture(scope="module")
def mods(asset_root, native_lib):
    import smirk_b200
    from oracle import flame_ref, render_ref
    assert torch.cuda.is_available(), "GPU suite needs a CUDA device"
    return (smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV),
            flame_ref.FlameConstants(asset_root), render_ref.RenderConstants(asset_root))


def flame_inputs(B, seed, short=False, eyelid=True, zero_neck_eye=True):
    p = synth_inputs.flame_params(B, seed)
    p.pop("cam")
    if short:                                          # zero-padded by FLAME.forward (FLAME.py:244-248)
        p["shape_params"], p["expression_params"] = p["shape_params"][:, :100], p["expression_params"][:, :20]
    if not eyelid:
        p.pop("eyelid_params")
    if zero_neck_eye:                                  # r = 0: Rodrigues' gradient must stay finite there
        p["neck_pose_params"], p["eye_pose_params"] = torch.zeros(B, 3), torch.zeros(B, 6)
    return p


def upstream(B, seed, keys=tuple(OUTS)):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(B, OUTS[k], 3, generator=g) for k in keys}


def flame_grads(fwd, p, ups, dev):
    leaves = {k: v.clone().to(dev).requires_grad_() for k, v in p.items()}
    o = fwd(leaves)
    loss = sum((o[k] * ups[k].to(dev)).sum() for k in ups)
    return dict(zip(leaves, torch.autograd.grad(loss, list(leaves.values()))))


def check_flame(mods, p, ups):
    from oracle import flame_ref
    fl, _, c, _ = mods
    got = flame_grads(fl.forward, p, ups, DEV)
    ref = flame_grads(lambda q: flame_ref.flame_forward_ref(c, q), p, ups, "cpu")
    for k in ref:
        assert torch.isfinite(got[k]).all(), k
        rel_close(got[k], ref[k])
    return got


@pytest.mark.parametrize("B", [1, 3, 32, 100])
def test_flame_grad_vs_oracle(mods, B):
    check_flame(mods, flame_inputs(B, 4000 + B), upstream(B, 5000 + B))


def test_grad_vs_reference_golden(mods, golden):
    """FLAME and Renderer gradients against torch autograd through the reference's own classes (grad.npz)."""
    from oracle import make_golden_grad as mg
    fl, rd, _, rc = mods
    g = golden("grad")
    p, ups = mg.flame_inputs()
    for k, v in flame_grads(fl.forward, p, ups, DEV).items():
        print("grad flame/%s rel %.2e" % (k, rel_close(v, g["flame/" + k]) / abs(g["flame/" + k]).max()))
    T = torch.from_numpy
    x, ups = mg.render_inputs(T(g["render/input_vertices"]),
                              {k: T(g["render/input_" + k]) for k in ("landmarks_fan", "landmarks_mp")}, rc)
    got, _ = render_grads(rd.forward, x, ups, DEV)
    for k, v in got.items():
        print("grad render/%s rel %.2e" % (k, rel_close(v, g["render/" + k]) / abs(g["render/" + k]).max()))


def test_flame_grad_variants(mods):
    B = 3
    check_flame(mods, flame_inputs(B, 4101, short=True, eyelid=False), upstream(B, 5101))
    check_flame(mods, flame_inputs(B, 4102, zero_neck_eye=False), upstream(B, 5102))
    for i, k in enumerate(OUTS):                       # each upstream gradient alone (the others are NULL)
        check_flame(mods, flame_inputs(B, 4110 + i), upstream(B, 5110 + i, (k,)))


def render_case(mods, B, seed):
    """Seeded FLAME meshes + cam, the oracle's differentiable render, and the upstream gradients with the
    clamp-boundary pixels zeroed."""
    from oracle import flame_ref, grad_ref
    _, _, c, rc = mods
    p = synth_inputs.flame_params(B, seed)
    fo = flame_ref.flame_forward_ref(c, p)
    x = {"vertices": fo["vertices"].detach(), "cam": p["cam"], "landmarks_fan": fo["landmarks_fan"].detach(),
         "landmarks_mp": fo["landmarks_mp"].detach()}
    with torch.no_grad():
        ndl = grad_ref.render_forward_grad_ref(rc, x["vertices"], x["cam"])["ndl"]
    keep = ~(((ndl.abs() < 1e-5) | ((ndl - 1).abs() < 1e-5)).any(1))
    g = torch.Generator().manual_seed(seed + 1)
    ups = {"rendered_img": torch.randn(B, 3, 224, 224, generator=g) * keep[:, None],
           "transformed_vertices": torch.randn(B, 5023, 3, generator=g),
           "landmarks_fan": torch.randn(B, 68, 2, generator=g), "landmarks_mp": torch.randn(B, 105, 2, generator=g)}
    return x, ups


def render_grads(fwd, x, ups, dev):
    leaves = {k: v.clone().to(dev).requires_grad_() for k, v in x.items()}
    o = fwd(leaves["vertices"], leaves["cam"], landmarks_fan=leaves["landmarks_fan"], landmarks_mp=leaves["landmarks_mp"])
    loss = sum((o[k] * ups[k].to(dev)).sum() for k in ups)
    gs = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    return {k: torch.zeros_like(v) if g is None else g for (k, v), g in zip(leaves.items(), gs)}, o


@pytest.mark.parametrize("B,seed", [(1, 6100), (5, 6200), (32, 6300)])
def test_renderer_grad_vs_oracle(mods, B, seed):
    from oracle import grad_ref
    _, rd, _, rc = mods
    x, ups = render_case(mods, B, seed)
    ref, ro = render_grads(lambda *a, **k: grad_ref.render_forward_grad_ref(rc, *a, **k), x, ups, "cpu")
    o = rd.render_full(x["vertices"].to(DEV), x["cam"].to(DEV))
    assert torch.equal(o["pix_to_face"].cpu(), ro["pix_to_face"])                   # coverage first, bit-exact
    assert torch.equal(ro["bary"].detach(), ro["bary_c"])                            # differentiable bary == C raster
    got, _ = render_grads(rd.forward, x, ups, DEV)
    for k in ref:
        rel_close(got[k], ref[k])


def test_renderer_grad_paths_alone(mods):
    from oracle import grad_ref
    _, rd, _, rc = mods
    x, ups = render_case(mods, 2, 6400)
    for k in ups:
        one = {k: ups[k]}
        ref, _ = render_grads(lambda *a, **kw: grad_ref.render_forward_grad_ref(rc, *a, **kw), x, one, "cpu")
        got, _ = render_grads(rd.forward, x, one, DEV)
        for q in ref:
            rel_close(got[q], ref[q], atol=1e-30)


def trainer_step(fl, rd, leaves, tgt, keep):
    """smirk_trainer.py:57-60 landmark losses + an L1 photometric term, FLAME -> Renderer."""
    fo = fl(leaves)
    ro = rd(fo["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
    return (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])
            + F.l1_loss(ro["rendered_img"] * keep, tgt["img"] * keep))


def test_trainer_shaped_step(mods):
    from oracle import flame_ref, grad_ref
    fl, rd, c, rc = mods
    B = 4
    p = synth_inputs.flame_params(B, 7000)
    g = torch.Generator().manual_seed(7001)
    tgt = {"fan": torch.randn(B, 68, 2, generator=g) * 0.5, "mp": torch.randn(B, 105, 2, generator=g) * 0.5,
           "img": torch.rand(B, 3, 224, 224, generator=g)}
    with torch.no_grad():
        fo = flame_ref.flame_forward_ref(c, p)
        ndl = grad_ref.render_forward_grad_ref(rc, fo["vertices"], p["cam"])["ndl"]
    keep = (~(((ndl.abs() < 1e-5) | ((ndl - 1).abs() < 1e-5)).any(1))).float()[:, None]
    ref_fl = lambda q: flame_ref.flame_forward_ref(c, q)
    ref_rd = lambda v, cam, **lm: grad_ref.render_forward_grad_ref(rc, v, cam, **lm)
    out = {}
    for dev, f, r in (("cpu", ref_fl, ref_rd), (DEV, fl, rd)):
        leaves = {k: v.clone().to(dev).requires_grad_() for k, v in p.items()}
        trainer_step(f, r, leaves, {k: v.to(dev) for k, v in tgt.items()}, keep.to(dev)).backward()
        out[dev] = {k: v.grad for k, v in leaves.items()}
    for k in p:
        rel_close(out[DEV][k], out["cpu"][k])


def test_backward_is_deterministic(mods):
    fl, rd, _, _ = mods
    B = 32
    p = synth_inputs.flame_params(B, 7100)
    tgt = {"fan": torch.zeros(B, 68, 2, device=DEV), "mp": torch.zeros(B, 105, 2, device=DEV),
           "img": torch.full((B, 3, 224, 224), 0.5, device=DEV)}
    runs = []
    for _ in range(2):
        leaves = {k: v.clone().to(DEV).requires_grad_() for k, v in p.items()}
        trainer_step(fl, rd, leaves, tgt, 1.0).backward()
        runs.append({k: v.grad.clone() for k, v in leaves.items()})
    for k in p:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_batch_independence_full_batch(mods):
    fl, rd, _, _ = mods
    B = 256
    p = {k: v.to(DEV) for k, v in synth_inputs.flame_params(B, 7200).items()}
    g = torch.Generator().manual_seed(7201)
    ups = {"img": torch.randn(B, 3, 224, 224, generator=g).to(DEV), "tv": torch.randn(B, 5023, 3, generator=g).to(DEV)}

    def grads(rows):
        leaves = {k: v[rows].clone().requires_grad_() for k, v in p.items()}
        fo = fl(leaves)
        ro = rd(fo["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"])
        loss = ((ro["rendered_img"] * ups["img"][rows]).sum() + (ro["transformed_vertices"] * ups["tv"][rows]).sum()
                + ro["landmarks_fan"].square().sum())
        return torch.autograd.grad(loss, list(leaves.values()))
    full, sub = grads(slice(None)), grads(slice(100, 103))
    for a, b in zip(full, sub):
        assert torch.equal(a[100:103], b)


def test_no_grad_path_unchanged(mods):
    """Without an input that requires grad (or under no_grad) the modules launch exactly what the forward-only
    modules do: FLAME 3 kernels (+ the dyn_idx copy, not a launch), Renderer 4 + 1 per landmark set."""
    from smirk_b200 import _lib
    fl, rd, _, _ = mods
    L = _lib.lib()
    p = {k: v.to(DEV) for k, v in synth_inputs.flame_params(2, 7300).items()}
    n0 = L.smk_launch_count()
    fo = fl(p)
    ro = rd(fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"])
    assert L.smk_launch_count() - n0 == 3 + 5
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    with torch.no_grad():
        n0 = L.smk_launch_count()
        fo2 = fl(leaves)
        ro2 = rd(fo2["vertices"], leaves["cam"], landmarks_fan=fo2["landmarks_fan"])
        assert L.smk_launch_count() - n0 == 3 + 5
    fo3 = fl(leaves)
    ro3 = rd(fo3["vertices"], leaves["cam"], landmarks_fan=fo3["landmarks_fan"])
    assert fo3["vertices"].requires_grad and ro3["rendered_img"].requires_grad
    for a, b, c in ((fo, fo2, fo3), (ro, ro2, ro3)):
        for k in a:
            assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k].detach()), k


def test_cuda_graph_forward_backward(mods):
    fl, rd, _, _ = mods
    B = 4
    static = {k: v.to(DEV).requires_grad_() for k, v in synth_inputs.flame_params(B, 7400).items()}
    tgt = {"fan": torch.zeros(B, 68, 2, device=DEV), "mp": torch.zeros(B, 105, 2, device=DEV),
           "img": torch.full((B, 3, 224, 224), 0.5, device=DEV)}

    def step():
        for v in static.values():
            v.grad = None
        trainer_step(fl, rd, static, tgt, 1.0).backward()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    for v in static.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fo = fl(static)
        ro = rd(fo["vertices"], static["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
        loss = (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])
                + F.l1_loss(ro["rendered_img"], tgt["img"]))
        gs = torch.autograd.grad(loss, list(static.values()))
    new = synth_inputs.flame_params(B, 7401)
    with torch.no_grad():
        for k, v in static.items():
            v.copy_(new[k].to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    leaves = {k: v.to(DEV).requires_grad_() for k, v in new.items()}
    trainer_step(fl, rd, leaves, tgt, 1.0).backward()
    for (k, v), g in zip(leaves.items(), gs):
        assert torch.equal(v.grad, g), k


def test_fitting_trajectory(mods):
    """10 steps of plain SGD fitting shape/expression/pose/cam to seeded target landmarks, against the oracle."""
    from oracle import flame_ref, render_ref
    fl, rd, c, _ = mods
    B, keys = 2, ("landmarks_fan", "landmarks_mp")
    tp = synth_inputs.flame_params(B, 7500)
    with torch.no_grad():
        fo = flame_ref.flame_forward_ref(c, tp)
        tgt = {k: render_ref.orth_proj_ref(fo[k], tp["cam"])[..., :2] for k in keys}
    s0 = synth_inputs.flame_params(B, 7501)
    start = {"shape_params": s0["shape_params"] * 0.1, "expression_params": s0["expression_params"] * 0.1,
             "pose_params": s0["pose_params"] * 0.1, "jaw_params": torch.zeros(B, 3), "cam": tp["cam"] + 0.1}

    def project(dev, fo, cam):
        if dev == "cpu":
            return {k: render_ref.orth_proj_ref(fo[k], cam)[..., :2] for k in keys}
        return rd(fo["vertices"], cam, landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])

    runs = {}
    for dev, f in (("cpu", lambda q: flame_ref.flame_forward_ref(c, q)), (DEV, fl)):
        x = {k: v.clone().to(dev).requires_grad_() for k, v in start.items()}
        opt = torch.optim.SGD(list(x.values()), lr=1e-3)
        traj, losses = [], []
        for _ in range(10):
            opt.zero_grad()
            xy = project(dev, f({k: v for k, v in x.items() if k != "cam"}), x["cam"])
            loss = sum(F.mse_loss(xy[k], tgt[k].to(dev)) for k in keys)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
            traj.append({k: v.detach().cpu().clone() for k, v in x.items()})
        runs[dev] = (traj, losses)
    (tr_ref, _), (tr, l_gpu) = runs["cpu"], runs[DEV]
    assert l_gpu[-1] < l_gpu[0]
    for a, b in zip(tr, tr_ref):
        for k in a:
            rel_close(a[k], b[k])
