"""GPU suite of the video stage: smk_hull_mask against cv2's create_mask on a corpus of ~4k landmark sets, smk_video_compose
against the numpy oracle (tests/video_ref.py), and SmirkPipeline with video= — the grid against the oracle applied to the
pipeline's own crop and render (and generator reconstruction), the crop and render against the stage-by-stage path, graph
replay and lanes against eager, batch independence at 1080p, launch counts, input errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import video_ref
from oracle import warp_ref
from smirk_b200 import _lib, crop, video

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _landmarks(rng, B, H, W, L=478):
    c = np.stack([rng.uniform(0.2 * W, 0.8 * W, B), rng.uniform(0.2 * H, 0.8 * H, B)], 1)[:, None]
    lm = c + rng.normal(0, 1, (B, L, 2)) * rng.uniform(0.03, 0.3, (B, 1, 1)) * min(H, W)
    lm[0] += np.array([0.45 * W, 0.0])                # frame 0's crop reaches past the right border
    return lm


def _compose(frames, crop_f, panels, m, render_orig):
    B, H, W, _ = frames.shape
    S = panels[0].shape[-1]
    Ho, Wo = (H, W) if render_orig else (S, S)
    grid = torch.full((B, Ho, (len(panels) + 1) * Wo, 3), 7, dtype=torch.uint8, device=DEV)
    ws = torch.empty(_lib.call("smk_video_workspace_bytes", DEV, B, len(panels)), dtype=torch.uint8, device=DEV)
    ptrs = (C.c_void_p * len(panels))(*[p.data_ptr() for p in panels])
    _lib.call("smk_video_compose", DEV, frames, B, H, W, crop_f, ptrs, len(panels), S, m, int(render_orig), grid, ws, ws.numel())
    return grid


@pytest.mark.parametrize("H,W", [(1080, 1920), (721, 1283)])
@pytest.mark.parametrize("n_panels", [1, 2])
@pytest.mark.parametrize("render_orig", [False, True])
def test_compose_matches_oracle(native_lib, H, W, n_panels, render_orig):
    rng = np.random.default_rng(H + n_panels + 10 * render_orig)
    B = 2
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    T = video.box_transforms(_landmarks(rng, B, H, W))
    crop_f = rng.integers(0, 256, (B, 3, 224, 224)).astype(np.float32) / np.float32(255.0)
    panels = [video_ref.special_renders(rng, B) for _ in range(n_panels)]
    if n_panels == 2:
        panels[1][1] = np.clip(panels[1][1], 0.1, 0.9)    # a panel without exact zeros: the clip to its minimum applies
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    got = _compose(t(frames), t(crop_f), [t(p) for p in panels], t(T.reshape(B, 9)), render_orig).cpu().numpy()
    want = video_ref.compose_ref(frames, crop_f, panels, T, render_orig)
    assert got.shape == want.shape
    for b in range(B):
        assert np.array_equal(got[b], want[b]), "frame %d: %d bytes differ" % (b, int((got[b] != want[b]).sum()))


def test_compose_row_pitch_and_empty_batch(native_lib):
    """A grid whose row pitch is not a multiple of 16 bytes, with its base off a 16-byte boundary."""
    rng = np.random.default_rng(5)
    B, H, W = 3, 37, 61
    frames = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).to(DEV)
    rend = torch.from_numpy(video_ref.special_renders(rng, B)).to(DEV)
    T = torch.from_numpy(np.stack([np.array([[3.0, 0.2, -20.0], [-0.2, 3.0, -10.0], [0, 0, 1]])] * B).reshape(B, 9)).to(DEV)
    pitch = 2 * W * 3
    store = torch.zeros(B * H * pitch + 5, dtype=torch.uint8, device=DEV)
    grid = store[5:].view(B, H, 2 * W, 3)
    ws = torch.empty(_lib.call("smk_video_workspace_bytes", DEV, B, 1), dtype=torch.uint8, device=DEV)
    ptrs = (C.c_void_p * 1)(rend.data_ptr())
    _lib.call("smk_video_compose", DEV, frames, B, H, W, None, ptrs, 1, 224, T, 1, grid, ws, ws.numel())
    want = video_ref.compose_ref(frames.cpu().numpy(), None, [rend.cpu().numpy()], T.cpu().numpy().reshape(B, 3, 3), True)
    assert np.array_equal(grid.cpu().numpy(), want) and not store[:5].any()
    _lib.call("smk_video_compose", DEV, None, 0, H, W, None, None, 0, 224, None, 1, None, None, 0)


# ---------------------------------------------------------------------------------------------- hull mask
def _create_mask(p, S=224):
    """datasets/base_dataset.py:9-15 with cv2 itself."""
    import cv2
    hull = cv2.convexHull(np.ascontiguousarray(p.astype(np.int32)[..., :2]))
    mask = np.ones((S, S), dtype=np.uint8)
    cv2.fillConvexPoly(mask, hull, 0)
    return mask


def _hull_corpus(rng, n, L=478):
    """Landmark sets of every kind create_mask meets, padded to L points by repeating their own points."""
    sets = []
    for t in range(n):
        k = t % 8
        if k == 0:
            p = rng.normal(112, rng.uniform(5, 60), (L, 2))                                   # mediapipe-like clouds
        elif k == 1:
            p = rng.uniform(-100, 330, (rng.integers(1, 30), 2))                              # touching / crossing the border
        elif k == 2:
            p = rng.integers(-3, 3, (rng.integers(1, 6), 2)) + rng.integers(0, 224, 2)       # 1-pixel and tiny hulls
        elif k == 3:
            a, b = rng.uniform(-300, 500, 2), rng.uniform(-300, 500, 2)
            p = np.round(a + rng.uniform(0, 1, (rng.integers(1, 20), 1)) * (b - a))          # collinear points
        elif k == 4:
            p = np.repeat(rng.uniform(-50, 270, (rng.integers(1, 4), 2)), rng.integers(1, 5), 0)   # 1 or 2 distinct points
        elif k == 5:
            p = rng.uniform(-2000, 2200, (rng.integers(3, 12), 2))                            # covering the whole crop
        elif k == 6:
            p = rng.normal(112, 200, (L, 2))
        else:
            p = rng.uniform(0, 224, (rng.integers(2, 8), 2)) * np.array([1, 0.02]) + np.array([0, rng.uniform(-10, 230)])
        p = p.astype(np.int32)
        sets.append(np.resize(p, (L, 2)))
    return np.stack(sets)


def test_hull_mask_matches_cv2(native_lib):
    rng = np.random.default_rng(61)
    pts = _hull_corpus(rng, 4096)
    mask = torch.empty(len(pts), 1, 224, 224, device=DEV)
    _lib.call("smk_hull_mask", DEV, torch.from_numpy(pts).to(DEV), len(pts), pts.shape[1], 224, mask)
    got = mask.cpu().numpy()
    bad = [i for i in range(len(pts)) if not np.array_equal(got[i, 0], _create_mask(pts[i]).astype(np.float32))]
    assert not bad, "%d of %d masks differ, first %d" % (len(bad), len(pts), bad[0])
    _lib.call("smk_hull_mask", DEV, None, 0, 478, 224, None)                             # empty batch: no-op
    with pytest.raises(RuntimeError):
        _lib.call("smk_hull_mask", DEV, torch.zeros(1, 1025, 2, dtype=torch.int32, device=DEV), 1, 1025, 224, mask)


# ---------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def modules(native_lib, asset_root):
    import smirk_b200
    from smirk_b200 import synth_inputs
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    enc = enc.eval().to(DEV)
    return enc, smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV)


def _pipe(modules, render_orig, hw=(1080, 1920), slots=2, generator=None, masking=None):
    from smirk_b200.pipeline import SmirkPipeline
    stage = video.VideoStage(hw, render_orig=render_orig, n_landmarks=64)
    return SmirkPipeline(*modules, generator, device=DEV, slots=slots, masking=masking, video=stage), stage


def _faces(rng, B, H, W):
    """Frames with a bright face-sized blob where the landmarks are, so the crops differ from frame to frame."""
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    lm = _landmarks(rng, B, H, W, L=64)
    lm[0] -= np.array([0.45 * W, 0.0])
    return frames, lm


@pytest.mark.parametrize("render_orig", [False, True])
def test_pipeline_grid_matches_the_stage_by_stage_path(modules, render_orig):
    rng = np.random.default_rng(21 + render_orig)
    B, H, W = 3, 1080, 1920
    frames, lm = _faces(rng, B, H, W)
    pipe, stage = _pipe(modules, render_orig)
    batch = stage.prepare(lm)
    f = torch.from_numpy(frames).to(DEV)
    out = pipe.forward(f, batch)
    torch.cuda.synchronize()
    T = batch["back_m"].numpy().reshape(B, 3, 3)
    # the crop is crop_to_tensor's; the render is the pipeline's without the video stage on that crop
    ref_crop = crop.crop_to_tensor(f, [crop.SimilarityTransform(T[b]) for b in range(B)], 224)
    assert torch.equal(out["cropped_img"], ref_crop)
    from smirk_b200.pipeline import SmirkPipeline
    plain = SmirkPipeline(*modules, device=DEV, slots=1).forward(ref_crop)
    for k in SmirkPipeline.OUT_KEYS:
        assert torch.equal(out[k], plain[k]), k
    want = video_ref.compose_ref(frames, out["cropped_img"].cpu().numpy(), [out["rendered_img"].cpu().numpy()], T, render_orig)
    assert np.array_equal(out["grid"].cpu().numpy(), want)
    # and row by row what the demo's per-frame loop writes, given the same crop and render
    cu8 = np.stack([warp_ref.warp_ref(frames[b], np.linalg.inv(T[b]), (224, 224)) for b in range(B)])
    for b in range(B):
        row = video_ref.demo_video_grid(frames[b], T[b], cu8[b], out["rendered_img"][b:b + 1].cpu(), render_orig)
        assert np.array_equal(out["grid"][b].cpu().numpy(), row)


def test_pipeline_graph_lanes_and_host_path_equal_eager(modules):
    rng = np.random.default_rng(31)
    B, H, W = 4, 721, 1283
    pipe, stage = _pipe(modules, True, (H, W))
    sets = []
    for _ in range(3):
        frames, lm = _faces(rng, B, H, W)
        sets.append((torch.from_numpy(frames), stage.prepare(lm)))
    eager = []
    for fr, bt in sets:
        o = pipe.forward(fr.to(DEV), bt)
        eager.append({k: v.clone() for k, v in o.items()})
    rep = pipe.replay(sets[0][0].to(DEV), sets[0][1])
    for k in eager[0]:
        assert torch.equal(rep[k], eager[0][k]), k
    dev_frames = [fr.to(DEV) for fr, _ in sets]
    for i in range(3):
        o = pipe.submit(i, dev_frames[i], sets[i][1])
        pipe.join()
        torch.cuda.synchronize()
        assert torch.equal(o["grid"], eager[i]["grid"]) and torch.equal(o["params"], eager[i]["params"]), i
    keys = ("grid", "params")
    for i in range(3):
        h = pipe.run_host(sets[i][0].pin_memory(), i, sets[i][1], keys)
        pipe.lane_done(i).synchronize()
        for k in keys:
            assert torch.equal(h[k], eager[i][k].cpu()), (i, k)
    h2d, d2h = pipe.bytes_per_step(B, keys)
    assert h2d == B * H * W * 3 + 2 * B * 9 * 8 and d2h == B * H * 2 * W * 3 + B * 361 * 4


@pytest.mark.parametrize("render_orig", [False, True])
def test_pipeline_launches_and_batch_independence_at_1080p(modules, render_orig):
    rng = np.random.default_rng(41)
    H, W = 1080, 1920
    frames, lm = _faces(rng, 64, H, W)
    pipe, stage = _pipe(modules, render_orig, slots=1)
    from smirk_b200.pipeline import SmirkPipeline
    base = SmirkPipeline(*modules, device=DEV, slots=1)
    for B in (1, 64):
        # crop = smk_crop_warp's three launches; compose = one, plus the clip-range reduction with render_orig
        assert pipe.launches_per_step(B) == base.launches_per_step(B) + 3 + (2 if render_orig else 1)
    f = torch.from_numpy(frames).to(DEV)
    big = {k: v.clone() for k, v in pipe.replay(f, stage.prepare(lm)).items()}
    for i in (0, 17, 63):
        one = pipe.replay(f[i:i + 1].contiguous(), stage.prepare(lm[i:i + 1]))
        assert torch.equal(one["grid"][0], big["grid"][i]), i
        assert torch.equal(one["params"][0], big["params"][i]), i


def test_video_inputs_are_checked(modules):
    rng = np.random.default_rng(51)
    pipe, stage = _pipe(modules, True, (64, 96))
    frames, lm = _faces(rng, 2, 64, 96)
    f, batch = torch.from_numpy(frames).to(DEV), stage.prepare(lm)
    for bad_f, bad_b in [(f.float(), batch), (f[..., :2], batch), (f[0], batch), (f[:, :32], batch),
                         (f[:1], batch), (f, stage.prepare(lm[:1])), (f, None)]:
        for call in (lambda: pipe.forward(bad_f, bad_b), lambda: pipe.submit(0, bad_f, bad_b),
                     lambda: pipe.run_host(bad_f.cpu(), 0, bad_b, ("grid",))):
            with pytest.raises(ValueError):
                call()
    from smirk_b200.pipeline import SmirkPipeline
    with pytest.raises(ValueError):
        SmirkPipeline(*modules, generator=torch.nn.Identity(), device=DEV, video=stage)


@pytest.fixture(scope="module")
def generator_stage(modules):
    import smirk_b200
    from smirk_b200 import synth_inputs
    from smirk_b200.masking import MaskingStage
    gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
    gen = gen.eval().to(DEV)
    fl = modules[1]
    return gen, MaskingStage(fl.faces_tensor, synth_inputs.face_probabilities(fl.faces_tensor.shape[0]), seed=5)


@pytest.mark.parametrize("render_orig", [False, True])
def test_pipeline_generator_panel(modules, generator_stage, render_orig):
    """--use_smirk_generator: the hull mask is create_mask of the batch's int32 crop landmarks; panel 2 is the oracle
    compose of the generator applied to the pipeline's own masked image; graph replay launches one hull-mask kernel more."""
    gen, stage_m = generator_stage
    rng = np.random.default_rng(71 + render_orig)
    B, H, W = 3, 721, 1283
    frames, lm = _faces(rng, B, H, W)
    pipe, stage = _pipe(modules, render_orig, (H, W), slots=1, generator=gen, masking=stage_m)
    batch = stage.prepare(lm)
    T = batch["back_m"].numpy().reshape(B, 3, 3)
    for b in range(B):                                               # demo_video.py:130-131, then create_mask's cast
        k = np.dot(T[b], np.hstack([lm[b, :, :2], np.ones([lm.shape[1], 1])]).T).T[:, :2]
        assert np.array_equal(batch["kpt"][b].numpy(), k.astype(np.int32))
    f = torch.from_numpy(frames).to(DEV)
    for out in (pipe.forward(f, batch), pipe.replay(f, batch)):
        torch.cuda.synchronize()
        for b in range(B):
            assert np.array_equal(out["hull_mask"][b, 0].cpu().numpy(), _create_mask(batch["kpt"][b].numpy()).astype(np.float32))
        rec = gen(torch.cat([out["rendered_img"], out["masked_img"]], 1))
        assert torch.equal(rec, out["reconstructed_img"])
        want = video_ref.compose_ref(frames, out["cropped_img"].cpu().numpy(),
                                     [out["rendered_img"].cpu().numpy(), rec.cpu().numpy()], T, render_orig)
        assert np.array_equal(out["grid"].cpu().numpy(), want)
    from smirk_b200.pipeline import SmirkPipeline
    base = SmirkPipeline(*modules, gen, device=DEV, slots=1, masking=stage_m)
    assert pipe.launches_per_step(B) == base.launches_per_step(B) + 3 + 1 + (2 if render_orig else 1)
