"""GPU suite (-m gpu): the CUDA path, called through the C ABI via the reference-signature modules,
against the CPU oracle on the same seeded inputs, against the committed golden fixtures (outputs of
the reference's own Python), and — at BASELINE.json's full batch sizes — through size-independent
properties.  Tolerances: vertices / landmarks / rendered pixels 1e-4 relative (north_star); face
indices and coverage bit-exact; encoder / generator in fp32 mode 1e-4 relative."""
import numpy as np
import pytest
import torch

from smirk_b200 import synth_inputs

pytestmark = pytest.mark.gpu
T = torch.from_numpy
DEV = "cuda:0"


def rel_close(a, b, rtol=1e-4, atol=0.0):
    a = a.detach().cpu().double().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
    b = b.detach().cpu().double().numpy() if torch.is_tensor(b) else np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() if a.size else 0.0
    ref = np.abs(b).max() if b.size else 0.0
    assert err <= atol + rtol * ref, "max abs err %.3g vs ref max %.3g (rel %.3g)" % (err, ref, err / max(ref, 1e-30))
    return err


def cuda(d):
    return {k: v.to(DEV) for k, v in d.items()}


@pytest.fixture(scope="module")
def mods(asset_root, native_lib):
    import smirk_b200
    assert torch.cuda.is_available(), "GPU suite needs a CUDA device"
    return smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV)


# ---------------------------------------------------------------------------------------------- FLAME
def test_flame_vs_reference_golden(mods, golden):
    fl, _ = mods
    g = golden("flame")
    o = fl.forward(cuda(synth_inputs.flame_params(4, 101)))
    for k in ("vertices", "landmarks_fan", "landmarks_fan_3d", "landmarks_mp"):
        rel_close(o[k], g["full/" + k])
    p2 = synth_inputs.flame_params(2, 102)
    short = {"shape_params": p2["shape_params"][:, :100], "expression_params": p2["expression_params"][:, :20],
             "pose_params": p2["pose_params"], "jaw_params": p2["jaw_params"]}
    o = fl.forward(cuda(short))                                    # padding + no-eyelid path (FLAME.py:244-248)
    rel_close(o["vertices"], g["short/vertices"])
    rel_close(o["landmarks_mp"], g["short/landmarks_mp"])
    o = fl.forward(cuda(p2), zero_expression=True, zero_shape=True, zero_pose=True)
    rel_close(o["vertices"], g["zero/vertices"])
    rel_close(o["landmarks_fan"], g["zero/landmarks_fan"])


def test_flame_contour_lut_sweep(mods, golden):
    fl, _ = mods
    ps = synth_inputs.flame_params(8, 103)
    ps["pose_params"] = torch.tensor([[0.1, y, 0.05] for y in (-1.2, -0.69, -0.3, -0.01, 0.0, 0.2, 0.68, 1.3)])
    o = fl.forward(cuda(ps))
    rel_close(o["landmarks_fan"], golden("flame")["sweep/landmarks_fan"])


def test_lbs_config1_and_joints(mods, golden, asset_root):
    from oracle import flame_ref
    fl, _ = mods
    g = golden("flame")
    p1 = synth_inputs.flame_params(1, 1001)
    betas = torch.cat([p1["shape_params"], p1["expression_params"]], 1)
    pose = torch.cat([p1["pose_params"], torch.zeros(1, 3), p1["jaw_params"], torch.zeros(1, 6)], 1)
    r = fl.run_lbs(betas.to(DEV), pose.to(DEV), None)
    rel_close(r["vertices"], g["c1/verts"])
    rel_close(r["joints"], g["c1/joints"])


@pytest.mark.parametrize("B", [1, 2, 3, 7, 32, 100])
def test_flame_vs_oracle_batches(mods, asset_root, B):
    from oracle import flame_ref
    fl, _ = mods
    c = flame_ref.FlameConstants(asset_root)
    p = synth_inputs.flame_params(B, 2000 + B)
    ref = flame_ref.flame_forward_ref(c, p)
    o = fl.forward(cuda(p))
    for k in ("vertices", "landmarks_fan", "landmarks_fan_3d", "landmarks_mp"):
        rel_close(o[k], ref[k])
    r = fl.run_lbs(torch.cat([p["shape_params"], p["expression_params"]], 1).to(DEV),
                   torch.cat([p["pose_params"], torch.zeros(B, 3), p["jaw_params"], torch.zeros(B, 6)], 1).to(DEV),
                   p["eyelid_params"].to(DEV))
    assert torch.equal(r["dyn_idx"].cpu().long(), ref["_dyn_idx"])


def test_flame_properties_full_batch(mods):
    """B=256 (configs[2]): identity pose + zero betas returns the template; batch rows are independent."""
    fl, _ = mods
    B = 256
    z = lambda n: torch.zeros(B, n, device=DEV)
    o = fl.forward({"shape_params": z(300), "expression_params": z(50), "pose_params": z(3), "jaw_params": z(3)})
    assert (o["vertices"] - fl.v_template[None]).abs().max() < 1e-6
    p = cuda(synth_inputs.flame_params(B, 77))
    a = fl.forward(p)["vertices"]
    sub = {k: v[100:103] for k, v in p.items()}
    b = fl.forward(sub)["vertices"]
    rel_close(a[100:103], b, 1e-6)
    assert fl.forward({k: v[:0] for k, v in p.items()})["vertices"].shape == (0, 5023, 3)     # empty batch


# ------------------------------------------------------------------------------------------- Renderer
def test_renderer_vs_reference_golden(mods, golden):
    _, rd = mods
    g = golden("render")
    v, cam = T(g["vertices"]).to(DEV), T(g["cam"]).to(DEV)
    lm_fan, lm_mp = v[:, :68].contiguous(), v[:, 100:205].contiguous()
    o = rd.render_full(v, cam, landmarks_fan=lm_fan)
    assert np.array_equal(o["pix_to_face"].cpu().numpy(), g["pix_to_face"].astype(np.int64))        # bit-exact
    assert np.array_equal(o["bary"].cpu().numpy(), g["bary"])                                        # bit-exact
    assert np.array_equal(o["transformed_vertices"].cpu().numpy(), g["transformed_vertices"])
    rel_close(o["rendered_img"], g["rendered_img"])
    out = rd.forward(v, cam, landmarks_fan=T(g["vertices"][:, :68]).to(DEV))
    assert set(out) == {"rendered_img", "transformed_vertices", "landmarks_fan"} and out["landmarks_fan"].shape == (2, 68, 2)
    assert torch.equal(out["rendered_img"], o["rendered_img"])


@pytest.mark.parametrize("B,seed", [(1, 5), (5, 6), (32, 7)])
def test_renderer_vs_oracle(mods, asset_root, B, seed):
    from oracle import flame_ref, render_ref
    _, rd = mods
    c = flame_ref.FlameConstants(asset_root)
    rc = render_ref.RenderConstants(asset_root)
    p = synth_inputs.flame_params(B, 3000 + seed)
    fo = flame_ref.flame_forward_ref(c, p)
    ref = render_ref.render_forward_ref(rc, fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"],
                                        landmarks_mp=fo["landmarks_mp"])
    o = rd.render_full(fo["vertices"].to(DEV), p["cam"].to(DEV), landmarks_fan=fo["landmarks_fan"].to(DEV),
                       landmarks_mp=fo["landmarks_mp"].to(DEV))
    assert torch.equal(o["pix_to_face"].cpu(), ref["pix_to_face"]), \
        "%d pixels differ" % int((o["pix_to_face"].cpu() != ref["pix_to_face"]).sum())
    assert torch.equal(o["bary"].cpu(), ref["bary"])
    assert torch.equal(o["zbuf"].cpu(), ref["zbuf"])
    assert torch.equal(o["transformed_vertices"].cpu(), ref["transformed_vertices"])
    rel_close(o["normals"], ref["normals"], 1e-5, 1e-6)
    rel_close(o["rendered_img"], ref["rendered_img"])
    for k in ("landmarks_fan", "landmarks_mp"):
        assert torch.equal(o[k].cpu(), ref[k])


def test_renderer_edge_cases(mods, asset_root):
    from oracle import render_ref
    _, rd = mods
    rc = render_ref.RenderConstants(asset_root)
    base = T(np.load(asset_root + "/assets/l_eyelid.npy")).float() * 0        # [5023,3] zeros
    tmpl = torch.tensor(np.array([[float(x) for x in ln.split()[1:4]] for ln in open(asset_root + "/assets/head_template.obj")
                                  if ln.startswith("v ")], dtype=np.float32))
    tmpl = tmpl - tmpl.mean(0)
    verts = torch.stack([tmpl, base, tmpl, tmpl])                  # row 1: fully degenerate mesh (all zero-area)
    cam = torch.tensor([[7.0, 0, 0], [7.0, 0, 0], [60.0, 0.0, 0.0], [7.0, 3.0, -3.0]])   # zoomed-in; shifted off-screen
    ref = render_ref.render_forward_ref(rc, verts, cam)
    o = rd.render_full(verts.to(DEV), cam.to(DEV))
    assert torch.equal(o["pix_to_face"].cpu(), ref["pix_to_face"])
    assert (o["pix_to_face"][1] == -1).all() and (o["rendered_img"][1] == 0).all()
    assert (o["pix_to_face"][3] == -1).all()
    assert (o["pix_to_face"][2] >= 0).float().mean() > 0.5
    rel_close(o["rendered_img"], ref["rendered_img"])
    e = rd.forward(verts[:0].to(DEV), cam[:0].to(DEV))
    assert e["rendered_img"].shape == (0, 3, 224, 224)


def test_renderer_properties_full_batch(mods):
    """B=256: per-image independence, background exactly 0, grey image (3 equal channels),
    packed indices lie in their own image's range, barycentrics sum to 1."""
    fl, rd = mods
    B = 256
    p = cuda(synth_inputs.flame_params(B, 88))
    v = fl.forward(p)["vertices"]
    o = rd.render_full(v, p["cam"])
    img, p2f = o["rendered_img"], o["pix_to_face"]
    assert torch.equal(img[:, 0], img[:, 1]) and torch.equal(img[:, 0], img[:, 2])
    assert (img[:, 0][p2f < 0] == 0).all() and float(img.max()) <= 1.7 * 180 / 255 + 1e-5
    lo = torch.arange(B, device=DEV).view(B, 1, 1) * 3408
    ok = (p2f < 0) | ((p2f >= lo) & (p2f < lo + 3408))
    assert ok.all()
    s = o["bary"].sum(-1)[p2f >= 0]
    # w_i = e_i / (area + 1e-8): sub-pixel slivers deviate from 1 by ~1e-8/area (pytorch3d semantics)
    assert (s - 1).abs().max() < 0.2 and (s - 1).abs().median() < 1e-3
    o2 = rd.render_full(v[17:19].contiguous(), p["cam"][17:19].contiguous())
    assert torch.equal(o2["rendered_img"], img[17:19])
    assert torch.equal(o2["pix_to_face"] + 17 * 3408 * (o2["pix_to_face"] >= 0), p2f[17:19])


# -------------------------------------------------------------------------------------------- Encoder
@pytest.fixture(scope="module")
def encoder(native_lib):
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    return enc.eval().to(DEV)


def test_encoder_vs_golden_and_oracle(encoder, golden):
    from oracle import encoder_ref
    g = golden("encoder")
    o = encoder(synth_inputs.images(2, 401).to(DEV))
    assert set(o) == {"pose_params", "cam", "shape_params", "expression_params", "eyelid_params", "jaw_params"}
    for k in o:
        rel_close(o[k], g[k], 1e-4, 1e-5)
    img = synth_inputs.images(5, 402)
    ref = encoder_ref.encoder_forward_ref({k: v.cpu() for k, v in encoder.state_dict().items()}, img)
    o = encoder(img.to(DEV))
    for k in o:
        rel_close(o[k], ref[k], 1e-4, 1e-5)
    assert o["shape_params"].shape == (5, 300) and o["cam"].shape == (5, 3)


def test_encoder_repack_on_weight_change_and_properties(encoder):
    img = synth_inputs.images(32, 403).to(DEV)
    a = encoder(img)
    b = encoder(img[5:9].contiguous())
    for k in a:
        rel_close(b[k], a[k][5:9], 1e-5, 1e-6)                     # batch rows independent
    import copy
    e2 = copy.deepcopy(encoder)
    with torch.no_grad():
        e2.shape_encoder.shape_layers[0].bias += 1.0
    c = e2(img[:2].contiguous())
    rel_close(c["shape_params"], a["shape_params"][:2] + 1.0, 1e-5, 1e-5)
    assert (a["eyelid_params"] >= 0).all() and (a["eyelid_params"] <= 1).all()
    assert (a["jaw_params"][:, 0] >= 0).all() and (a["jaw_params"][:, 1:].abs() <= 0.2).all()


# ------------------------------------------------------------------------------------------ Generator
@pytest.fixture(scope="module")
def generator(native_lib):
    import smirk_b200
    gen = smirk_b200.SmirkGenerator(in_channels=6, out_channels=3, init_features=32, res_blocks=5)
    gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
    return gen.eval().to(DEV)


def test_generator_vs_golden_and_oracle(generator, golden):
    from oracle import generator_ref
    g, r = golden("generator"), golden("render")
    x = torch.cat([T(r["rendered_img"][:1]), synth_inputs.masked_images(1, 301)], 1)
    y = generator(x.to(DEV))
    rel_close(y[:, :, ::4, ::4], g["y_sub"], 1e-4, 1e-5)
    rel_close(y[:, :, 100:102], g["y_rows"], 1e-4, 1e-5)
    x2 = torch.cat([T(r["rendered_img"]), synth_inputs.masked_images(2, 302)], 1)
    ref = generator_ref.generator_forward_ref({k: v.cpu() for k, v in generator.state_dict().items()}, x2)
    y2 = generator(x2.to(DEV))
    rel_close(y2, ref, 1e-4, 1e-5)
    assert y2.shape == (2, 3, 224, 224) and float(y2.min()) > 0 and float(y2.max()) < 1


def test_generator_batch_independence(generator):
    x = torch.cat([synth_inputs.images(8, 303), synth_inputs.masked_images(8, 304)], 1).to(DEV)
    a = generator(x)
    b = generator(x[3:5].contiguous())
    rel_close(b, a[3:5], 1e-5, 1e-6)


# ------------------------------------------------------------------------- TF32 tensor-core precision
# precision = 1 runs the 1x1 / 3x3 / transposed convolutions on wgmma with TF32 operands (10-bit
# mantissa, fp32 accumulate) — the arithmetic the reference itself gets from cuDNN on Ampere+ GPUs
# (torch.backends.cudnn.allow_tf32 defaults to True).  Tolerance: 5e-3 of the output scale through
# the ~50-layer encoder and the 27-conv generator, stated here; the fp32 path above stays at 1e-4.
def test_generator_tf32_tensor_core_path(generator, golden):
    import copy
    from oracle import generator_ref
    gtc = copy.deepcopy(generator)
    gtc.precision = 1
    r = golden("render")
    x2 = torch.cat([T(r["rendered_img"]), synth_inputs.masked_images(2, 302)], 1)
    ref = generator_ref.generator_forward_ref({k: v.cpu() for k, v in generator.state_dict().items()}, x2)
    y = gtc(x2.to(DEV))
    assert torch.isfinite(y).all()
    err = rel_close(y, ref, 5e-3, 0)
    y32 = generator(x2.to(DEV))
    rel_close(y, y32, 5e-3, 0)
    x = torch.cat([synth_inputs.images(5, 305), synth_inputs.masked_images(5, 306)], 1).to(DEV)   # 5*196 rows: ragged tiles
    a = gtc(x)
    rel_close(gtc(x[1:3].contiguous()), a[1:3], 1e-6, 1e-7)        # tile boundaries do not leak across images
    rel_close(a, generator(x), 5e-3, 0)


def test_encoder_tf32_tensor_core_path(encoder):
    import copy
    from oracle import encoder_ref
    etc = copy.deepcopy(encoder)
    etc.precision = 1
    img = synth_inputs.images(5, 402)
    ref = encoder_ref.encoder_forward_ref({k: v.cpu() for k, v in encoder.state_dict().items()}, img)
    o = etc(img.to(DEV))
    for k in o:
        scale = max(float(ref[k].abs().max()), 1.0)
        assert float((o[k].cpu() - ref[k]).abs().max()) <= 5e-3 * scale, k
    o32 = encoder(img.to(DEV))
    assert float((o["shape_params"] - o32["shape_params"]).abs().max()) > 0      # really a different arithmetic path


def test_encoder_fused_blocks_path(encoder):
    """precision = 2: inverted-residual blocks run expand+depthwise as one wgmma kernel."""
    import copy
    from oracle import encoder_ref
    ef = copy.deepcopy(encoder)
    ef.precision = 2
    img = synth_inputs.images(5, 402)
    ref = encoder_ref.encoder_forward_ref({k: v.cpu() for k, v in encoder.state_dict().items()}, img)
    o = ef(img.to(DEV))
    for k in o:
        scale = max(float(ref[k].abs().max()), 1.0)
        assert float((o[k].cpu() - ref[k]).abs().max()) <= 5e-3 * scale, k
    a = ef(synth_inputs.images(32, 403).to(DEV))
    b = ef(synth_inputs.images(32, 403)[7:9].contiguous().to(DEV))
    for k in a:
        rel_close(b[k], a[k][7:9], 1e-5, 1e-6)


# -------------------------------------------------------------------------------------------- pipeline
def test_pipeline_graph_lanes_and_host_path(mods, encoder):
    """SmirkPipeline: eager forward == CUDA-graph replay == software-pipelined lanes == pinned host path,
    bit for bit (same kernels, same inputs), and the composed pipeline agrees with the oracle stage by stage."""
    from smirk_b200.pipeline import SmirkPipeline
    fl, rd = mods
    pipe = SmirkPipeline(encoder, fl, rd, None, device=DEV, slots=2)
    B = 4
    imgs = [synth_inputs.images(B, 700 + i) for i in range(4)]
    dimgs = [x.to(DEV) for x in imgs]
    eager = [{k: v.clone() for k, v in pipe.forward(x).items()} for x in dimgs]
    for i, x in enumerate(dimgs):
        out = pipe.replay(x)
        for k in eager[i]:
            assert torch.equal(out[k], eager[i][k]), k
    got = []
    for i, x in enumerate(dimgs):                      # lanes: batch i on lane i % 2; read back after join
        o = pipe.submit(i, x)
        pipe.join()
        got.append({k: v.clone() for k, v in o.items()})
    for i in range(4):
        for k in eager[i]:
            assert torch.equal(got[i][k], eager[i][k]), (i, k)
    keys = ("rendered_img", "vertices", "params")
    pinned = [x.pin_memory() for x in imgs]
    for i in range(4):
        ho = pipe.run_host(pinned[i], i, None, keys)
        pipe.lane_done(i).synchronize()
        for k in keys:
            assert torch.equal(ho[k], eager[i][k].cpu()), (i, k)
    assert eager[0]["params"].shape == (B, 361) and pipe.launches_per_step(B) > 50


# ----------------------------------------------------- parity of the BENCHED configuration (image -> pixels), B = 32 / 256
def _pipeline_outputs(enc, fl, rd, img):
    p = enc(img.to(DEV))
    fo = fl.forward(p)
    ro = rd.render_full(fo["vertices"], p["cam"])
    return {"params_dict": p, "vertices": fo["vertices"], "rendered_img": ro["rendered_img"],
            "transformed_vertices": ro["transformed_vertices"], "pix_to_face": ro["pix_to_face"]}


def _write_report(name, rep):
    import json, os
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, name), "w") as fh:
            json.dump(rep, fh, indent=1)
    except OSError:
        pass


@pytest.mark.parametrize("precision", [3, 2, 0])
def test_benched_pipeline_parity_configs1(mods, encoder, asset_root, precision):
    """configs[1] inputs (32 faces): encoder at the given precision -> FLAME -> renderer against the CPU oracle.
    precision 3 (3xTF32, the bench default) and 0 (fp32 CUDA cores) must meet the north_star: vertices 1e-4 relative,
    rendered pixels 1e-4 and face indices bit-exact for the rasteriser on the device's own vertices.  precision 2
    (plain TF32, cuDNN's default arithmetic) is measured and bounded at its stated 5e-3 parameter tolerance."""
    import copy
    from oracle import parity_check
    fl, rd = mods
    enc = copy.deepcopy(encoder)
    enc.precision = precision
    img = synth_inputs.images(32, 5000)
    rep = parity_check.pipeline_report(asset_root, encoder.state_dict(), img, _pipeline_outputs(enc, fl, rd, img))
    rep["precision"] = precision
    _write_report("parity_c1_b32_precision%d.json" % precision, rep)
    print("parity precision %d: %s" % (precision, rep))
    assert rep["p2f_stage_mismatch"] == 0
    assert rep["pixels_stage_abs"] <= 1e-4 * 1.7
    if precision in (0, 3):
        assert rep["params_rel"] <= 1e-4, rep
        assert rep["vertices_rel"] <= 1e-4, rep
        assert rep["tverts_rel"] <= 1e-4, rep
    else:
        assert rep["params_rel"] <= 5e-3, rep
        assert rep["vertices_rel"] <= 5e-3, rep


def test_encoder_and_generator_at_batch_256(mods, encoder, generator, asset_root):
    """configs[2] batch size: 256 faces through encoder (precision 3) -> FLAME -> renderer -> generator (TF32).  The CPU
    oracle checks a strided sample of 8 faces end to end (its generator costs ~1 s per face); the rest of the batch is
    covered by batch-row independence against the same faces run as a small batch."""
    import copy
    from oracle import parity_check, generator_ref
    fl, rd = mods
    enc = copy.deepcopy(encoder); enc.precision = 3
    gtc = copy.deepcopy(generator); gtc.precision = 1
    B = 256
    img = synth_inputs.images(B, 5100)
    mask = synth_inputs.masked_images(B, 5101)
    out = _pipeline_outputs(enc, fl, rd, img)
    y = gtc(torch.cat([out["rendered_img"], mask.to(DEV)], 1))
    assert y.shape == (B, 3, 224, 224) and bool(torch.isfinite(y).all())
    sel = torch.arange(5, B, 32)                                    # 8 faces
    sub = {k: (v[sel] if torch.is_tensor(v) else {kk: vv[sel] for kk, vv in v.items()}) for k, v in out.items()}
    sub["pix_to_face"] = None                                       # packed indices depend on the batch position
    rep = parity_check.pipeline_report(asset_root, encoder.state_dict(), img[sel], sub)
    _write_report("parity_c2_b256_sample8.json", rep)
    assert rep["vertices_rel"] <= 1e-4 and rep["pixels_stage_abs"] <= 1e-4 * 1.7, rep
    small = _pipeline_outputs(enc, fl, rd, img[sel])
    rel_close(small["vertices"], out["vertices"][sel], 1e-6, 1e-7)
    assert torch.equal(small["pix_to_face"] % 3408, out["pix_to_face"][sel] % 3408) or \
        torch.equal((small["pix_to_face"] >= 0), (out["pix_to_face"][sel] >= 0))
    x_sel = torch.cat([out["rendered_img"][sel].cpu(), mask[sel]], 1)
    ref = generator_ref.generator_forward_ref({k: v.cpu() for k, v in generator.state_dict().items()}, x_sel[:2])
    rel_close(y[sel[:2]], ref, 5e-3, 0)                              # TF32 generator: stated tolerance
    rel_close(gtc(x_sel.to(DEV)), y[sel], 1e-6, 1e-7)                # batch rows independent at B = 256


# ----------------------------------------------------------------------- graph lifetime, sub-encoders, masking in the pipeline
def test_graphs_of_different_batch_sizes_keep_their_workspaces_alive(mods, encoder):
    """ADVICE r1 (medium): capture B = 2, then B = 8 (the module workspaces grow -> new buffers), then re-pack the
    encoder; the B = 2 graph must still replay correctly: it keeps the workspace and the packed weights it was recorded
    with alive (rec['keep'])."""
    import copy
    import gc
    from smirk_b200.pipeline import SmirkPipeline
    fl, rd = mods
    enc = copy.deepcopy(encoder)
    enc.precision = 3
    pipe = SmirkPipeline(enc, fl, rd, None, device=DEV, slots=1)
    x2, x8 = synth_inputs.images(2, 801).to(DEV), synth_inputs.images(8, 802).to(DEV)
    eager2 = {k: v.clone() for k, v in pipe.forward(x2).items()}
    pipe.capture(2)
    ws_before = enc.graph_keep_alive()[1].data_ptr()
    eager8 = {k: v.clone() for k, v in pipe.forward(x8).items()}
    pipe.capture(8)
    assert enc.graph_keep_alive()[1].data_ptr() != ws_before, "the workspace was expected to grow into a new buffer"
    with torch.no_grad():
        enc.shape_encoder.shape_layers[0].bias += 0.0           # bumps the version: the next eager forward re-packs the weights
    pipe.forward(x8)
    gc.collect()
    torch.cuda.empty_cache()
    scratch = torch.full((64 << 20,), float("nan"), device=DEV)  # would land in any freed workspace
    o2 = pipe.replay(x2)
    for k in eager2:
        assert torch.equal(o2[k], eager2[k]), k
    o8 = pipe.replay(x8)
    for k in eager8:
        assert torch.equal(o8[k], eager8[k]), k
    del scratch


def test_sub_encoders_have_the_reference_forward(encoder):
    """src/smirk_encoder.py:34-45,66-73,95-110: each sub-encoder is callable on its own and returns its own dict."""
    img = synth_inputs.images(3, 811).to(DEV)
    full = encoder(img)
    p = encoder.pose_encoder(img)
    s = encoder.shape_encoder(img)
    e = encoder.expression_encoder(img)
    assert set(p) == {"pose_params", "cam"} and set(s) == {"shape_params"} and set(e) == {"expression_params", "eyelid_params", "jaw_params"}
    for d in (p, s, e):
        for k, v in d.items():
            rel_close(v, full[k], 1e-6, 1e-7)
    encoder.train()
    try:
        with pytest.raises(RuntimeError, match="train-mode"):
            encoder(img)                                         # .train() after the first forward must not silently run eval BN
    finally:
        encoder.eval()


def test_full_cycle_pipeline_with_masking_stage(mods, encoder, generator):
    """The full cycle with the real masking step (demo.py:138-165) inside the CUDA graph: rendered image and vertices are
    identical from replay to replay, the masked image is redrawn (device RNG counter advances in-graph), and the
    generator's input is exactly cat(rendered, masked)."""
    import copy
    from smirk_b200.masking import MaskingStage
    from smirk_b200.pipeline import SmirkPipeline
    fl, rd = mods
    gtc = copy.deepcopy(generator); gtc.precision = 1
    st = MaskingStage(fl.faces_tensor, synth_inputs.face_probabilities(fl.faces_tensor.shape[0]), seed=5)
    pipe = SmirkPipeline(encoder, fl, rd, gtc, device=DEV, slots=1, masking=st)
    img, hull = synth_inputs.images(3, 821).to(DEV), synth_inputs.hull_masks(3, 822).to(DEV)
    a = {k: v.clone() for k, v in pipe.replay(img, hull).items()}
    b = {k: v.clone() for k, v in pipe.replay(img, hull).items()}
    assert torch.equal(a["rendered_img"], b["rendered_img"]) and torch.equal(a["vertices"], b["vertices"])
    assert not torch.equal(a["masked_img"], b["masked_img"]), "the device RNG did not advance between graph replays"
    m = a["masked_img"]
    outside = hull.expand(-1, 3, -1, -1) > 0
    far = torch.nn.functional.max_pool2d(1 - hull, 21, 1, 10) == 0          # pixels the dilated hull does not reach
    bg = (a["rendered_img"] == 0).all(1, keepdim=True)
    keep = (far & bg).expand(-1, 3, -1, -1)
    # outside the dilated hull and off the rendered mesh the image passes through, except at sampled points of mesh parts
    # the renderer does not draw (scalp, neck), which carry img * noise
    assert float((m[keep] == img[keep]).float().mean()) > 0.95
    assert float((m > 0).float().mean()) > 0.1 and outside.any()
    y = gtc(torch.cat([a["rendered_img"], a["masked_img"]], 1))
    rel_close(a["reconstructed_img"], y, 1e-6, 1e-7)
