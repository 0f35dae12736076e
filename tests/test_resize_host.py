"""CPU suite of the video stage without --crop: the resize oracle (tests/resize_ref.py) against cv2.resize, the compose
oracle of mode 2 against a literal restatement of the demo's per-frame grid with cv2 and torch's CPU F.interpolate,
VideoStage.prepare with crop=False, and the argument checks of the two extended entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

import resize_ref
import video_ref
from smirk_b200 import video


@pytest.mark.parametrize("H,W", resize_ref.SHAPES)
def test_resize_oracle_equals_cv2(H, W):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(H * 7 + W)
    for k, img in enumerate(resize_ref.frame_contents(rng, H, W)):
        want = cv2.resize(img, (224, 224))
        got = resize_ref.cv2_resize_ref(img)
        assert np.array_equal(got, want), "content %d: %d bytes differ" % (k, int((got != want).sum()))


CPU_TOL = resize_ref.FUSED_INDEX_TOL


@pytest.mark.parametrize("H,W", [(97, 131), (224, 224), (512, 512), (300, 533)])
@pytest.mark.parametrize("n_panels", [1, 2])
@pytest.mark.parametrize("render_orig", [False, True])
def test_resize_compose_oracle_equals_the_demo_video_restatement(H, W, n_panels, render_orig):
    pytest.importorskip("cv2")
    import torch.nn.functional as F
    rng = np.random.default_rng(H + W + n_panels + 10 * render_orig)
    B = 2
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    panels = [video_ref.special_renders(rng, B) for _ in range(n_panels)]
    crop_f = np.stack([resize_ref.cv2_resize_ref(f[..., ::-1]).transpose(2, 0, 1) for f in frames]).astype(np.float32) / np.float32(255.0)
    if render_orig:
        for p in panels:
            err = np.abs(resize_ref.torch_bilinear_ref(p, H, W) - F.interpolate(torch.from_numpy(p), (H, W), mode='bilinear').numpy())
            assert err.max() <= CPU_TOL
        got = resize_ref.compose_resize_ref(frames, panels)
    else:
        got = video_ref.compose_ref(frames, crop_f, panels, None, False)
    near = 0
    for b in range(B):
        t = [torch.from_numpy(p[b:b + 1]) for p in panels]
        cropped, want = resize_ref.demo_video_grid_nocrop(frames[b], t[0], render_orig, t[1] if n_panels == 2 else None)
        assert torch.equal(cropped[0], torch.from_numpy(crop_f[b]))
        assert got[b].shape == want.shape
        diff = got[b].astype(np.int16) - want.astype(np.int16)
        if not render_orig:
            assert not diff.any()
            continue
        # a byte may differ by one only where torch's x * 255 lies within 255 * CPU_TOL of an integer
        x255 = torch.cat([F.interpolate(u, (H, W), mode='bilinear') for u in t], 3)[0].permute(1, 2, 0).numpy()[..., ::-1] * np.float32(255.0)
        x255 = np.concatenate([np.full((H, W, 3), 0.5, np.float32), x255], 1)              # the frame panel: no slack
        bad = diff != 0
        assert (np.abs(diff[bad]) == 1).all() and (np.abs(x255[bad] - np.rint(x255[bad])) <= 255 * CPU_TOL).all()
        near += int(bad.sum())
    print("%dx%d, %d panel(s): %d bytes off by one at a near-integer x * 255" % (H, W, n_panels, near))


def test_prepare_without_crop():
    stage = video.VideoStage((512, 512), crop=False, n_landmarks=478)
    rng = np.random.default_rng(4)
    lm = rng.uniform(-40.0, 560.0, (5, 478, 3))
    lm[0, :3, :2] = [[-0.7, -3.9], [2.9, -0.2], [511.99, 0.5]]                         # negative fractions truncate to 0
    batch = stage.prepare(lm)
    assert batch.size == 5 and list(batch) == ["kpt"] and batch["kpt"].dtype == torch.int32
    assert np.array_equal(batch["kpt"].numpy(), lm.astype(np.int32)[..., :2])
    assert batch["kpt"].is_pinned() == torch.cuda.is_available()
    assert np.array_equal(batch["kpt"][0, :3].numpy(), [[0, -3], [2, 0], [511, 0]])
    empty = stage.prepare(batch_size=7)
    assert empty.size == 7 and not empty
    assert stage.prepare(batch_size=0).size == 0
    for bad in (lambda: stage.prepare(), lambda: stage.prepare(batch_size=-1), lambda: stage.prepare(np.zeros((5, 2))),
                lambda: stage.prepare(np.zeros((2, 10, 2))), lambda: stage.prepare(lm, batch_size=4),
                lambda: video.VideoStage((512, 512)).prepare(batch_size=3), lambda: video.VideoStage((512, 512)).prepare()):
        with pytest.raises(ValueError):
            bad()


def test_extended_entry_points_check_their_arguments(native_lib):
    L = native_lib
    vp, nul = C.c_void_p, C.c_void_p(0)
    buf = vp(16)                                      # never dereferenced: the checks fail first
    # smk_crop_warp: a NULL matrix is the resize; NULL frames or output still fail
    assert L.smk_crop_warp(nul, 2, 8, 8, nul, 224, 1, buf, nul, 0, nul) < 0 and b"null argument" in L.smk_last_error()
    assert L.smk_crop_warp(buf, 2, 8, 8, nul, 224, 1, nul, nul, 0, nul) < 0 and b"null argument" in L.smk_last_error()
    assert L.smk_crop_warp(buf, 2, 0, 8, nul, 224, 1, buf, nul, 0, nul) < 0 and b"bad sizes" in L.smk_last_error()
    assert L.smk_crop_warp(buf, 70000, 8, 8, nul, 224, 1, buf, nul, 0, nul) < 0 and b"too many frames" in L.smk_last_error()
    # smk_video_compose mode 2: frames needed, no workspace, crop and m unused
    ptrs = (vp * 2)(16, 16)
    rc = L.smk_video_compose(nul, 2, 8, 8, buf, ptrs, 1, 224, buf, 2, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"needs frames" in L.smk_last_error()
    rc = L.smk_video_compose(buf, 2, 70000, 8, nul, ptrs, 2, 224, nul, 2, buf, nul, 0, nul)
    assert rc < 0 and b"too many rows" in L.smk_last_error()                               # past the workspace check
    for mode in (3, -1):
        rc = L.smk_video_compose(buf, 2, 8, 8, buf, ptrs, 1, 224, buf, mode, buf, buf, 1 << 20, nul)
        assert rc < 0 and b"must be 0, 1 or 2" in L.smk_last_error()
