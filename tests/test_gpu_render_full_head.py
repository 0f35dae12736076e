"""GPU suite (-m gpu) of ``Renderer(render_full_head=True)``: the whole FLAME mesh (5023 vertices, 9976 triangles) through
smk_renderer_forward / smk_renderer_backward, against the full-head CPU restatement (tests/render_full_head_ref.py) and
the reference class's outputs and autograd (tests/golden/render_full_head.npz).

Forward: pix_to_face, bary and zbuf bit-exact against the C rasteriser (oracle/raster_ref.c) on the device's own
transformed vertices; transformed_vertices, with the reference's leaked z + 10, bitwise equal to the oracle.
Backward: max-abs error <= 1e-4 x max-abs of the oracle, per tensor (rel_close of test_gpu_parity), with the
clamp-boundary rule of test_gpu_grad (pixels whose n.l lies within 1e-5 of 0 or 1 get a zero upstream gradient)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import render_full_head_ref as fh
from smirk_b200 import _lib, synth_inputs

from test_gpu_parity import rel_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NV, NF = fh.N_VERTS, fh.N_FACES
SUB = (slice(None), slice(None, None, 2), slice(None, None, 2))


@pytest.fixture(scope="module")
def mods(asset_root, native_lib):
    import smirk_b200
    from oracle import flame_ref
    assert torch.cuda.is_available(), "GPU suite needs a CUDA device"
    return (smirk_b200.FLAME().to(DEV), smirk_b200.Renderer(render_full_head=True).to(DEV),
            flame_ref.FlameConstants(asset_root), fh.FullHeadConstants(asset_root))


def meshes(mods, B, seed):
    from oracle import flame_ref
    p = synth_inputs.flame_params(B, seed)
    with torch.no_grad():
        fo = flame_ref.flame_forward_ref(mods[2], p)
    return {"vertices": fo["vertices"], "cam": p["cam"], "landmarks_fan": fo["landmarks_fan"],
            "landmarks_mp": fo["landmarks_mp"]}


def upstream(rc, x, seed):
    B = x["vertices"].shape[0]
    keep = fh.clamp_keep(rc, x["vertices"], x["cam"])
    g = torch.Generator().manual_seed(seed)
    return {"rendered_img": torch.randn(B, 3, 224, 224, generator=g) * keep[:, None],
            "transformed_vertices": torch.randn(B, NV, 3, generator=g),
            "landmarks_fan": torch.randn(B, 68, 2, generator=g), "landmarks_mp": torch.randn(B, 105, 2, generator=g)}


def render_grads(fwd, x, ups, dev):
    leaves = {k: v.clone().to(dev).requires_grad_() for k, v in x.items()}
    o = fwd(leaves["vertices"], leaves["cam"], landmarks_fan=leaves["landmarks_fan"], landmarks_mp=leaves["landmarks_mp"])
    loss = sum((o[k] * ups[k].to(dev)).sum() for k in ups)
    gs = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    return {k: torch.zeros_like(v) if g is None else g for (k, v), g in zip(leaves.items(), gs)}, o


def oracle(rc):
    return lambda *a, **k: fh.render_forward_grad_ref(rc, *a, **k)


# ---------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("B", [32, 256])
def test_raster_bit_exact_on_device_vertices(mods, B):
    """The rasteriser at full size against raster_ref.c, fed the device's own transformed vertices."""
    from oracle import render_ref
    fl, rd, _, rc = mods
    p = {k: v.to(DEV) for k, v in synth_inputs.flame_params(B, 9000 + B).items()}
    o = rd.render_full(fl(p)["vertices"], p["cam"])
    fixed = o["transformed_vertices"].cpu()                     # z already carries the + 10 the rasteriser sees
    fixed[..., :2] = -fixed[..., :2]
    fv = fixed.reshape(B * NV, 3)[rc.faces + (torch.arange(B) * NV)[:, None, None]].reshape(-1, 3, 3)
    p2f, zbuf, bary, _ = render_ref.rasterize_ref(fv, B, NF)
    assert torch.equal(o["pix_to_face"].cpu(), p2f[..., 0]), "%d pixels differ" % int((o["pix_to_face"].cpu() != p2f[..., 0]).sum())
    assert torch.equal(o["bary"].cpu(), bary[:, :, :, 0])
    assert torch.equal(o["zbuf"].cpu(), zbuf[..., 0])
    assert (o["pix_to_face"] >= 0).float().mean() > 0.1
    lo = torch.arange(B, device=DEV).view(B, 1, 1) * NF
    assert ((o["pix_to_face"] < 0) | ((o["pix_to_face"] >= lo) & (o["pix_to_face"] < lo + NF))).all()


@pytest.mark.parametrize("B,seed", [(1, 9100), (5, 9200), (32, 9300)])
def test_forward_vs_oracle(mods, B, seed):
    _, rd, _, rc = mods
    x = meshes(mods, B, seed)
    ref = fh.render_forward_ref(rc, x["vertices"], x["cam"], landmarks_fan=x["landmarks_fan"], landmarks_mp=x["landmarks_mp"])
    o = rd.render_full(*(x[k].to(DEV) for k in ("vertices", "cam")), landmarks_fan=x["landmarks_fan"].to(DEV),
                       landmarks_mp=x["landmarks_mp"].to(DEV))
    for k in ("pix_to_face", "bary", "zbuf", "transformed_vertices", "landmarks_fan", "landmarks_mp"):
        assert torch.equal(o[k].cpu(), ref[k]), k
    rel_close(o["normals"], ref["normals"], 1e-5, 1e-6)
    rel_close(o["rendered_img"], ref["rendered_img"])
    out = rd(x["vertices"].to(DEV), x["cam"].to(DEV))
    assert set(out) == {"rendered_img", "transformed_vertices"}
    assert torch.equal(out["transformed_vertices"], o["transformed_vertices"]) and torch.equal(out["rendered_img"], o["rendered_img"])


def test_forward_and_grad_vs_reference_golden(mods, golden):
    """render_full_head.npz: the reference class's own outputs and autograd."""
    import make_golden_full_head as mgf
    _, rd, _, rc = mods
    g = golden("render_full_head")
    x, ups = mgf.inputs(golden("grad"), rc)
    o = rd.render_full(x["vertices"].to(DEV), x["cam"].to(DEV), landmarks_fan=x["landmarks_fan"].to(DEV),
                       landmarks_mp=x["landmarks_mp"].to(DEV))
    assert np.array_equal(o["pix_to_face"][SUB].cpu().numpy(), g["pix_to_face"].astype(np.int64))
    assert np.array_equal(o["zbuf"][SUB].cpu().numpy(), g["zbuf"])
    assert np.array_equal(o["transformed_vertices"][..., 2].cpu().numpy(), g["transformed_vertices_z"])
    for k in ("landmarks_fan", "landmarks_mp"):
        assert np.array_equal(o[k].cpu().numpy(), g[k])
    print("full head rendered_img vs golden: max abs %.2e" % rel_close(o["rendered_img"][:, 0][SUB], g["rendered_img"]))
    got, _ = render_grads(rd.forward, x, ups, DEV)
    for k, v in got.items():
        print("full head grad %s vs golden: rel %.2e" % (k, rel_close(v, g["grad/" + k]) / np.abs(g["grad/" + k]).max()))


# ---------------------------------------------------------------------------------------------- backward
@pytest.mark.parametrize("B,seed", [(1, 9400), (5, 9500), (32, 9600)])
def test_grad_vs_oracle(mods, B, seed):
    _, rd, _, rc = mods
    x = meshes(mods, B, seed)
    ups = upstream(rc, x, seed + 1)
    ref, ro = render_grads(oracle(rc), x, ups, "cpu")
    assert torch.equal(ro["bary"].detach(), ro["bary_c"])                       # differentiable bary == C raster
    got, o = render_grads(rd.forward, x, ups, DEV)
    assert torch.equal(o["transformed_vertices"].detach().cpu(), ro["transformed_vertices"].detach())
    for k in ref:
        assert torch.isfinite(got[k]).all(), k
        rel_close(got[k], ref[k])


def test_grad_paths_alone(mods):
    _, rd, _, rc = mods
    x = meshes(mods, 2, 9700)
    ups = upstream(rc, x, 9701)
    for k in ups:
        one = {k: ups[k]}
        ref, _ = render_grads(oracle(rc), x, one, "cpu")
        got, _ = render_grads(rd.forward, x, one, DEV)
        for q in ref:
            rel_close(got[q], ref[q], atol=1e-30)


def trainer_step(fl, rd, leaves, tgt, keep):
    """smirk_trainer.py:57-60 landmark losses + an L1 photometric term, FLAME -> full-head Renderer."""
    fo = fl(leaves)
    ro = rd(fo["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
    return (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])
            + F.l1_loss(ro["rendered_img"] * keep, tgt["img"] * keep))


def test_trainer_shaped_step(mods):
    from oracle import flame_ref
    fl, rd, c, rc = mods
    B = 4
    p = synth_inputs.flame_params(B, 9800)
    g = torch.Generator().manual_seed(9801)
    tgt = {"fan": torch.randn(B, 68, 2, generator=g) * 0.5, "mp": torch.randn(B, 105, 2, generator=g) * 0.5,
           "img": torch.rand(B, 3, 224, 224, generator=g)}
    with torch.no_grad():
        keep = fh.clamp_keep(rc, flame_ref.flame_forward_ref(c, p)["vertices"], p["cam"]).float()[:, None]
    ref_fl = lambda q: flame_ref.flame_forward_ref(c, q)
    out = {}
    for dev, f, r in (("cpu", ref_fl, oracle(rc)), (DEV, fl, rd)):
        leaves = {k: v.clone().to(dev).requires_grad_() for k, v in p.items()}
        trainer_step(f, r, leaves, {k: v.to(dev) for k, v in tgt.items()}, keep.to(dev)).backward()
        out[dev] = {k: v.grad for k, v in leaves.items()}
    for k in p:
        rel_close(out[DEV][k], out["cpu"][k])


def test_backward_is_deterministic(mods):
    fl, rd, _, _ = mods
    B = 32
    p = synth_inputs.flame_params(B, 9900)
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
    p = {k: v.to(DEV) for k, v in synth_inputs.flame_params(B, 9910).items()}
    g = torch.Generator().manual_seed(9911)
    ups = {"img": torch.randn(B, 3, 224, 224, generator=g).to(DEV), "tv": torch.randn(B, NV, 3, generator=g).to(DEV)}

    def run(rows):
        leaves = {k: v[rows].clone().requires_grad_() for k, v in p.items()}
        fo = fl(leaves)
        ro = rd(fo["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"])
        loss = ((ro["rendered_img"] * ups["img"][rows]).sum() + (ro["transformed_vertices"] * ups["tv"][rows]).sum()
                + ro["landmarks_fan"].square().sum())
        return [ro["rendered_img"].detach(), ro["transformed_vertices"].detach()] + list(torch.autograd.grad(loss, list(leaves.values())))
    full, sub = run(slice(None)), run(slice(100, 103))
    for a, b in zip(full, sub):
        assert torch.equal(a[100:103], b)


def test_no_grad_path_launches(mods):
    """The z offset costs no launch: FLAME 3 kernels, Renderer 4 + 1 per landmark set, as with the face mask; the
    autograd path's forward computes the same outputs."""
    fl, rd, _, _ = mods
    L = _lib.lib()
    p = {k: v.to(DEV) for k, v in synth_inputs.flame_params(2, 9920).items()}
    n0 = L.smk_launch_count()
    fo = fl(p)
    ro = rd(fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"])
    assert L.smk_launch_count() - n0 == 3 + 5
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    with torch.no_grad():
        n0 = L.smk_launch_count()
        ro2 = rd(fl(leaves)["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"])
        assert L.smk_launch_count() - n0 == 3 + 5
    fo3 = fl(leaves)
    ro3 = rd(fo3["vertices"], leaves["cam"], landmarks_fan=fo3["landmarks_fan"])
    assert ro3["rendered_img"].requires_grad and ro3["transformed_vertices"].requires_grad
    for k in ro:
        assert torch.equal(ro[k], ro2[k]) and torch.equal(ro[k], ro3[k].detach()), k


def test_cuda_graph_forward_backward(mods):
    fl, rd, _, _ = mods
    B = 4
    static = {k: v.to(DEV).requires_grad_() for k, v in synth_inputs.flame_params(B, 9930).items()}
    tgt = {"fan": torch.zeros(B, 68, 2, device=DEV), "mp": torch.zeros(B, 105, 2, device=DEV),
           "img": torch.full((B, 3, 224, 224), 0.5, device=DEV), "tv": torch.randn(B, NV, 3, device=DEV)}

    def loss_of(leaves):
        fo = fl(leaves)
        ro = rd(fo["vertices"], leaves["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
        return (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])
                + F.l1_loss(ro["rendered_img"], tgt["img"]) + (ro["transformed_vertices"] * tgt["tv"]).mean())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            torch.autograd.grad(loss_of(static), list(static.values()))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gs = torch.autograd.grad(loss_of(static), list(static.values()))
    new = synth_inputs.flame_params(B, 9931)
    with torch.no_grad():
        for k, v in static.items():
            v.copy_(new[k].to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    leaves = {k: v.to(DEV).requires_grad_() for k, v in new.items()}
    want = torch.autograd.grad(loss_of(leaves), list(leaves.values()))
    for k, a, b in zip(leaves, gs, want):
        assert torch.equal(a, b), k


# ---------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def encoder_generator(native_lib):
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
    return enc.eval().to(DEV), gen.eval().to(DEV)


def test_pipeline_replay_equals_eager(mods, encoder_generator):
    """SmirkPipeline with a full-head renderer: without a generator, and with the generator fed a ready-made masked
    image, graph replay equals the eager run bit for bit; with MaskingStage + generator the deterministic outputs do,
    and the reconstruction is the generator applied to the replay's own masked image."""
    from smirk_b200.masking import MaskingStage
    from smirk_b200.pipeline import SmirkPipeline
    fl, rd, _, _ = mods
    enc, gen = encoder_generator
    B = 3
    img, masked, hull = (synth_inputs.images(B, 9940).to(DEV), synth_inputs.masked_images(B, 9941).to(DEV),
                         synth_inputs.hull_masks(B, 9942).to(DEV))
    for g, aux in ((None, None), (gen, masked)):
        pipe = SmirkPipeline(enc, fl, rd, g, device=DEV, slots=1)
        eager = {k: v.clone() for k, v in pipe.forward(img, aux).items()}
        assert eager["transformed_vertices"].shape == (B, NV, 3)
        out = pipe.replay(img, aux)
        for k in eager:
            assert torch.equal(out[k], eager[k]), (g is not None, k)
    ro = rd.render_full(eager["vertices"], eager["params"][:, 3:6])
    assert torch.equal(ro["rendered_img"], eager["rendered_img"])
    assert torch.equal(ro["transformed_vertices"], eager["transformed_vertices"])
    st = MaskingStage(fl.faces_tensor, synth_inputs.face_probabilities(fl.faces_tensor.shape[0]), seed=5)
    pipe = SmirkPipeline(enc, fl, rd, gen, device=DEV, slots=1, masking=st)
    a = {k: v.clone() for k, v in pipe.forward(img, hull).items()}
    b = {k: v.clone() for k, v in pipe.replay(img, hull).items()}
    for k in SmirkPipeline.OUT_KEYS:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], eager[k]), k
    assert torch.equal(b["reconstructed_img"], gen(torch.cat([b["rendered_img"], b["masked_img"]], 1)))


def test_video_stage_grid(mods, encoder_generator):
    """VideoStage with a full-head renderer: the grid is the compose oracle of the pipeline's own crop and render, the
    render is the plain full-head pipeline's on that crop, and replay equals eager."""
    import video_ref
    from smirk_b200 import crop, video
    from smirk_b200.pipeline import SmirkPipeline
    fl, rd, _, _ = mods
    enc, _ = encoder_generator
    rng = np.random.default_rng(9950)
    B, H, W = 3, 360, 640
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    c = np.stack([rng.uniform(0.3 * W, 0.7 * W, B), rng.uniform(0.3 * H, 0.7 * H, B)], 1)[:, None]
    lm = c + rng.normal(0, 1, (B, 64, 2)) * 0.1 * H
    stage = video.VideoStage((H, W), render_orig=True, n_landmarks=64)
    pipe = SmirkPipeline(enc, fl, rd, device=DEV, slots=1, video=stage)
    batch = stage.prepare(lm)
    f = torch.from_numpy(frames).to(DEV)
    out = {k: v.clone() for k, v in pipe.forward(f, batch).items()}
    rep = pipe.replay(f, batch)
    for k in out:
        assert torch.equal(rep[k], out[k]), k
    T = batch["back_m"].numpy().reshape(B, 3, 3)
    ref_crop = crop.crop_to_tensor(f, [crop.SimilarityTransform(T[b]) for b in range(B)], 224)
    assert torch.equal(out["cropped_img"], ref_crop)
    plain = SmirkPipeline(enc, fl, rd, device=DEV, slots=1).forward(ref_crop)
    for k in SmirkPipeline.OUT_KEYS:
        assert torch.equal(out[k], plain[k]), k
    want = video_ref.compose_ref(frames, out["cropped_img"].cpu().numpy(), [out["rendered_img"].cpu().numpy()], T, True)
    assert np.array_equal(out["grid"].cpu().numpy(), want)
