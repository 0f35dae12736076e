"""GPU suite of the video stage without --crop: smk_crop_warp without a matrix against cv2.resize, smk_video_compose mode 2
against the numpy oracle (tests/resize_ref.py) and torch's own CUDA F.interpolate, smk_hull_mask on landmarks in frame
pixels against cv2's create_mask, and SmirkPipeline with VideoStage(..., crop=False): the resize, the outputs against the
plain pipeline, the grid against the oracle, graph replay, lanes and the host path against eager, launch counts, batch
independence at 1080p, the H2D bytes and input errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import resize_ref
import video_ref
from resize_ref import SHAPES, frame_contents
from smirk_b200 import _lib, video

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cv2_input(frame):
    """demo_video.py:134-136 without --crop, with cv2 itself: the encoder's input [3,224,224]."""
    import cv2
    return torch.tensor(cv2.resize(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB), (224, 224))).permute(2, 0, 1).float() / 255


def _resize(frames):
    B, H, W, _ = frames.shape
    out = torch.full((B, 3, 224, 224), -1.0, device=DEV)
    n0 = _lib.call("smk_launch_count", DEV)
    _lib.call("smk_crop_warp", DEV, frames, B, H, W, None, 224, 1, out, None, 0)
    assert _lib.call("smk_launch_count", DEV) - n0 == 1
    return out


def test_resize_matches_cv2_on_the_corpus(native_lib):
    pytest.importorskip("cv2")
    rng = np.random.default_rng(81)
    for H, W in SHAPES:
        frames = np.stack(frame_contents(rng, H, W))
        got = _resize(torch.from_numpy(frames).to(DEV)).cpu()
        for b in range(len(frames)):
            assert torch.equal(got[b], _cv2_input(frames[b])), (H, W, b)


def test_resize_batch_of_64_at_1080p(native_lib):
    pytest.importorskip("cv2")
    rng = np.random.default_rng(82)
    frames = rng.integers(0, 256, (64, 1080, 1920, 3), dtype=np.uint8)
    frames[5:9] = frame_contents(rng, 1080, 1920)
    dev = torch.from_numpy(frames).to(DEV)
    got = _resize(dev).cpu()
    for b in range(64):
        assert torch.equal(got[b], _cv2_input(frames[b])), b
    one = _resize(dev[37:38].contiguous())                              # a frame on its own equals its row of the batch
    assert torch.equal(one.cpu()[0], got[37])


def _compose2(frames, panels):
    B, H, W, _ = frames.shape
    grid = torch.full((B, H, (len(panels) + 1) * W, 3), 7, dtype=torch.uint8, device=DEV)
    ptrs = (C.c_void_p * len(panels))(*[p.data_ptr() for p in panels])
    n0 = _lib.call("smk_launch_count", DEV)
    _lib.call("smk_video_compose", DEV, frames, B, H, W, None, ptrs, len(panels), 224, None, 2, grid, None, 0)
    assert _lib.call("smk_launch_count", DEV) - n0 == 1
    return grid


@pytest.mark.parametrize("H,W", [(1080, 1920), (721, 1283), (512, 512), (224, 224)])
@pytest.mark.parametrize("n_panels", [1, 2])
def test_compose_mode2_matches_oracle_and_torch(native_lib, H, W, n_panels):
    import torch.nn.functional as F
    rng = np.random.default_rng(H + W + n_panels)
    B = 2
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    panels = [video_ref.special_renders(rng, B) for _ in range(n_panels)]
    dp = [torch.from_numpy(p).to(DEV) for p in panels]
    got = _compose2(torch.from_numpy(frames).to(DEV), dp).cpu().numpy()
    want = resize_ref.compose_resize_ref(frames, panels)
    for b in range(B):
        assert np.array_equal(got[b], want[b]), "frame %d: %d bytes differ" % (b, int((got[b] != want[b]).sum()))
    # the reference's own op on this device: bytes differ only by one, where x * 255 lies near an integer
    tol = 255 * resize_ref.FUSED_INDEX_TOL
    x255 = torch.cat([dp[0].new_full((B, 3, H, W), 0.5)] + [F.interpolate(p, (H, W), mode='bilinear') * 255.0 for p in dp],
                     3).permute(0, 2, 3, 1).flip(3).cpu().numpy()                 # BGR; the frame panel gets no slack
    ref = x255.astype(np.uint8)
    ref[:, :, :W] = frames
    bad = got != ref
    assert (np.abs(got[bad].astype(int) - ref[bad]) == 1).all() and (np.abs(x255[bad] - np.rint(x255[bad])) <= tol).all()
    dist = np.abs(x255[bad] - np.rint(x255[bad]))
    print("%dx%d, %d panel(s): %d bytes off by one against torch's CUDA F.interpolate, %d of them farther than 1e-4 from an "
          "integer" % (H, W, n_panels, int(bad.sum()), int((dist > 1e-4).sum())))


def test_compose_mode2_row_pitch_and_empty_batch(native_lib):
    """A grid whose row pitch is not a multiple of 16 bytes, with its base off a 16-byte boundary."""
    rng = np.random.default_rng(6)
    B, H, W = 3, 37, 61
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    for n_panels in (1, 2):
        panels = [video_ref.special_renders(rng, B) for _ in range(n_panels)]
        dp = [torch.from_numpy(p).to(DEV) for p in panels]
        pitch = (n_panels + 1) * W * 3
        store = torch.zeros(B * H * pitch + 5, dtype=torch.uint8, device=DEV)
        grid = store[5:].view(B, H, (n_panels + 1) * W, 3)
        ptrs = (C.c_void_p * n_panels)(*[p.data_ptr() for p in dp])
        _lib.call("smk_video_compose", DEV, torch.from_numpy(frames).to(DEV), B, H, W, None, ptrs, n_panels, 224, None, 2,
                  grid, None, 0)
        assert np.array_equal(grid.cpu().numpy(), resize_ref.compose_resize_ref(frames, panels)) and not store[:5].any()
    _lib.call("smk_video_compose", DEV, None, 0, H, W, None, None, 0, 224, None, 2, None, None, 0)


# ---------------------------------------------------------------------------------------------- hull mask
def _create_mask(p, S=224):
    """datasets/base_dataset.py:9-15 with cv2 itself, on landmarks in frame pixels (float, cast as the reference does)."""
    import cv2
    hull = cv2.convexHull(np.ascontiguousarray(p.astype(np.int32)[..., :2]))
    mask = np.ones((S, S), dtype=np.uint8)
    cv2.fillConvexPoly(mask, hull, 0)
    return mask


def _frame_landmark_corpus(rng, n, L=478):
    """Landmark sets in frame pixels: 1080p and 4K clouds anywhere, hulls wholly right of or below the mask, hulls
    straddling the origin, sets with negative fractional coordinates."""
    sets = []
    for t in range(n):
        k = t % 6
        if k == 0:
            H, W = (1080, 1920) if t % 12 == 0 else (2160, 3840)
            p = np.array([rng.uniform(0, W), rng.uniform(0, H)]) + rng.normal(0, 1, (L, 2)) * rng.uniform(5, 400)
        elif k == 1:
            p = rng.uniform(0, 1, (L, 2)) * rng.uniform(10, 400) + np.array([rng.uniform(224, 3600), rng.uniform(-50, 200)])
        elif k == 2:
            p = rng.uniform(0, 1, (L, 2)) * rng.uniform(10, 400) + np.array([rng.uniform(-50, 200), rng.uniform(224, 2000)])
        elif k == 3:
            p = rng.normal(0, rng.uniform(2, 300), (L, 2))
        elif k == 4:
            p = rng.uniform(-1, 1, (L, 2)) * rng.uniform(0.5, 3) + rng.uniform(0, 224, 2)
            p[:L // 4] = -rng.uniform(0, 1, (L // 4, 2))                                      # truncate to 0
        else:
            p = rng.uniform(-3840, 3840, (rng.integers(3, 12), 2))
            p = np.resize(p, (L, 2))
        sets.append(p)
    return np.stack(sets)


def test_hull_mask_from_frame_landmarks_matches_cv2(native_lib):
    pytest.importorskip("cv2")
    rng = np.random.default_rng(62)
    lm = _frame_landmark_corpus(rng, 1536)
    stage = video.VideoStage((2160, 3840), crop=False)
    kpt = stage.prepare(lm)["kpt"]
    mask = torch.empty(len(lm), 1, 224, 224, device=DEV)
    _lib.call("smk_hull_mask", DEV, kpt.to(DEV), len(lm), lm.shape[1], 224, mask)
    got = mask.cpu().numpy()
    bad = [i for i in range(len(lm)) if not np.array_equal(got[i, 0], _create_mask(lm[i]).astype(np.float32))]
    assert not bad, "%d of %d masks differ, first %d" % (len(bad), len(lm), bad[0])
    assert (got == 1).all(axis=(1, 2, 3))[1::6].any() and (got == 0).any(axis=(1, 2, 3))[3::6].all()


# ---------------------------------------------------------------------------------------------- pipeline
@pytest.fixture(scope="module")
def modules(native_lib, asset_root):
    import smirk_b200
    from smirk_b200 import synth_inputs
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    enc = enc.eval().to(DEV)
    return enc, smirk_b200.FLAME().to(DEV), smirk_b200.Renderer().to(DEV)


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


def _pipe(modules, render_orig, hw, slots=2, gen=None):
    from smirk_b200.pipeline import SmirkPipeline
    stage = video.VideoStage(hw, render_orig=render_orig, n_landmarks=64, crop=False)
    g, m = gen if gen is not None else (None, None)
    return SmirkPipeline(*modules, g, device=DEV, slots=slots, masking=m, video=stage), stage


def _frames(rng, B, H, W):
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    c = np.stack([rng.uniform(0, W, B), rng.uniform(0, H, B)], 1)[:, None]
    lm = c + rng.normal(0, 1, (B, 64, 2)) * rng.uniform(0.03, 0.3, (B, 1, 1)) * min(H, W)
    return frames, lm


@pytest.mark.parametrize("generator", [False, True])
@pytest.mark.parametrize("render_orig", [False, True])
def test_pipeline_without_crop(modules, generator_stage, render_orig, generator):
    from smirk_b200.pipeline import SmirkPipeline
    rng = np.random.default_rng(91 + render_orig + 2 * generator)
    B, H, W = 3, 721, 1283
    frames, lm = _frames(rng, B, H, W)
    gen, stage_m = generator_stage if generator else (None, None)
    pipe, stage = _pipe(modules, render_orig, (H, W), gen=generator_stage if generator else None)
    batch = stage.prepare(lm) if generator else stage.prepare(batch_size=B)
    f = torch.from_numpy(frames).to(DEV)
    pipe.capture(B)
    if generator:                                   # the masking step's draws restart from the same counter below
        stage_m.reseed(5)
    eager = {k: v.clone() for k, v in pipe.forward(f, batch).items()}
    torch.cuda.synchronize()
    assert torch.equal(eager["cropped_img"].cpu(), torch.stack([_cv2_input(fr) for fr in frames]))
    plain = SmirkPipeline(*modules, device=DEV, slots=1).forward(eager["cropped_img"])
    for k in SmirkPipeline.OUT_KEYS:
        assert torch.equal(eager[k], plain[k]), k
    panels = [eager["rendered_img"].cpu().numpy()]
    if generator:
        for b in range(B):                          # create_mask(kpt_mediapipe, (224, 224)) on frame pixels
            assert np.array_equal(eager["hull_mask"][b, 0].cpu().numpy(), _create_mask(lm[b]).astype(np.float32)), b
        rec = gen(torch.cat([eager["rendered_img"], eager["masked_img"]], 1))
        assert torch.equal(rec, eager["reconstructed_img"])
        panels.append(rec.cpu().numpy())
    if render_orig:
        want = resize_ref.compose_resize_ref(frames, panels)
    else:
        want = video_ref.compose_ref(frames, eager["cropped_img"].cpu().numpy(), panels, None, False)
    assert np.array_equal(eager["grid"].cpu().numpy(), want)
    # graph replay, lanes and the host path equal eager
    if generator:
        stage_m.reseed(5)
    rep = pipe.replay(f, batch)
    for k in eager:
        assert torch.equal(rep[k], eager[k]), k
    base = SmirkPipeline(*modules, gen, device=DEV, slots=1, masking=stage_m)
    # launches: the base pipeline + the resize + the compose (+ the hull mask with the generator)
    assert pipe.launches_per_step(B) == base.launches_per_step(B) + 2 + (1 if generator else 0)
    h2d, d2h = pipe.bytes_per_step(B, ("grid", "params"))
    assert h2d == B * H * W * 3 + (B * 64 * 2 * 4 if generator else 0)
    assert d2h == eager["grid"].numel() + B * 361 * 4
    if generator:                                   # lanes draw their own masks; without a generator they must agree
        return
    for i in range(3):
        o = pipe.submit(i, f, batch)
        pipe.join()
        torch.cuda.synchronize()
        assert torch.equal(o["grid"], eager["grid"]) and torch.equal(o["params"], eager["params"]), i
    keys = ("grid", "params")
    host = torch.from_numpy(frames).pin_memory()
    for i in range(3):
        h = pipe.run_host(host, i, batch, keys)
        pipe.lane_done(i).synchronize()
        for k in keys:
            assert torch.equal(h[k], eager[k].cpu()), (i, k)


@pytest.mark.parametrize("render_orig", [False, True])
def test_pipeline_without_crop_batch_independence_at_1080p(modules, render_orig):
    rng = np.random.default_rng(43)
    H, W = 1080, 1920
    frames, _ = _frames(rng, 64, H, W)
    pipe, stage = _pipe(modules, render_orig, (H, W), slots=1)
    f = torch.from_numpy(frames).to(DEV)
    big = {k: v.clone() for k, v in pipe.replay(f, stage.prepare(batch_size=64)).items()}
    for i in (0, 17, 63):
        one = pipe.replay(f[i:i + 1].contiguous(), stage.prepare(batch_size=1))
        assert torch.equal(one["grid"][0], big["grid"][i]), i
        assert torch.equal(one["params"][0], big["params"][i]), i


def test_video_inputs_without_crop_are_checked(modules, generator_stage):
    rng = np.random.default_rng(52)
    pipe, stage = _pipe(modules, True, (64, 96))
    frames, lm = _frames(rng, 2, 64, 96)
    f, batch = torch.from_numpy(frames).to(DEV), stage.prepare(batch_size=2)
    for bad_f, bad_b in [(f.float(), batch), (f[..., :2], batch), (f[0], batch), (f[:, :32], batch),
                         (f[:1], batch), (f, stage.prepare(batch_size=1)), (f, None), (f, {})]:
        for call in (lambda: pipe.forward(bad_f, bad_b), lambda: pipe.submit(0, bad_f, bad_b),
                     lambda: pipe.run_host(bad_f.cpu(), 0, bad_b, ("grid",))):
            with pytest.raises(ValueError):
                call()
    gpipe, gstage = _pipe(modules, True, (64, 96), gen=generator_stage)
    for call in (lambda: gpipe.forward(f, batch), lambda: gpipe.replay(f, batch), lambda: gpipe.submit(0, f, batch),
                 lambda: gpipe.run_host(f.cpu(), 0, batch, ("grid",))):
        with pytest.raises(ValueError, match="lacks kpt"):                 # a generator needs the landmarks
            call()
