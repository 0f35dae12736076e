"""CPU suite of the video stage (smirk_b200/video.py, smk_hull_mask / smk_video_* in include/smirk_b200.h): argument
checking of the entry points, the byte round trip of the frame panel, the batched crop transforms against the one-frame
helper, and the compose oracle (tests/video_ref.py) against a literal restatement of the video demo's per-frame grid."""
import ctypes as C

import numpy as np
import pytest
import torch

from smirk_b200 import crop, video
import video_ref


def _landmarks(rng, B, H=1080, W=1920, L=478):
    c = np.stack([rng.uniform(0.1 * W, 0.9 * W, B), rng.uniform(0.1 * H, 0.9 * H, B)], 1)[:, None]
    lm = c + rng.normal(0, 1, (B, L, 2)) * rng.uniform(10, 250, (B, 1, 1))
    return np.concatenate([lm, rng.normal(0, 1, (B, L, 1))], 2)                          # mediapipe's third (z) column


def test_video_compose_rejects_bad_arguments(native_lib):
    L = native_lib
    vp, nul = C.c_void_p, C.c_void_p(0)
    buf = vp(16)                                      # never dereferenced: the checks fail first
    ptrs = (vp * 2)(16, 16)
    rc = L.smk_video_compose(buf, -1, 8, 8, buf, ptrs, 1, 224, buf, 1, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_video_compose(buf, 2, 8, 8, buf, ptrs, 3, 224, buf, 1, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"bad sizes" in L.smk_last_error()
    rc = L.smk_video_compose(buf, 2, 8, 8, buf, ptrs, 1, 224, buf, 1, nul, buf, 1 << 20, nul)
    assert rc < 0 and b"null argument" in L.smk_last_error()
    rc = L.smk_video_compose(buf, 2, 8, 8, nul, ptrs, 1, 224, nul, 0, buf, nul, 0, nul)
    assert rc < 0 and b"crop is needed" in L.smk_last_error()
    rc = L.smk_video_compose(buf, 2, 8, 8, nul, ptrs, 1, 224, buf, 1, buf, buf, 0, nul)
    assert rc < 0 and b"workspace too small" in L.smk_last_error()
    assert L.smk_video_compose(nul, 0, 0, 0, nul, nul, 0, 0, nul, 0, nul, nul, 0, nul) == 0      # empty batch: no-op
    assert L.smk_video_workspace_bytes(64, 2) >= 64 * 2 * 8


def test_frame_panel_round_trip_is_the_identity():
    """u8 -> BGR2RGB -> /255 (float32) -> x255 -> astype(uint8) -> RGB2BGR gives back every one of the 256 values, so
    the frame panel of --render_orig is a copy of the frame's bytes (and a rendered panel's /255 -> x255 likewise)."""
    v = np.arange(256, dtype=np.uint8)
    t = torch.tensor(v).float() / 255.0                                                     # demo_video.py:150,156
    assert np.array_equal((t.numpy() * 255.0).astype(np.uint8), v)                           # demo_video.py:211-212
    cv2 = pytest.importorskip("cv2")
    img = np.stack(list(np.meshgrid(v, v[::-1], indexing="ij")) + [np.roll(np.broadcast_to(v, (256, 256)), 7, 1)], -1).astype(np.uint8)
    chain = torch.Tensor(cv2.cvtColor(img, cv2.COLOR_BGR2RGB)).permute(2, 0, 1).unsqueeze(0).float() / 255.0
    out = cv2.cvtColor((chain.squeeze(0).permute(1, 2, 0).numpy() * 255.0).astype(np.uint8), cv2.COLOR_BGR2RGB)
    assert np.array_equal(out, img)


def test_prepare_equals_the_one_frame_transform_bitwise():
    rng = np.random.default_rng(3)
    stage = video.VideoStage((1080, 1920), render_orig=True)
    for B in (1, 7, 64):
        lm = _landmarks(rng, B)
        batch = stage.prepare(lm)
        assert batch.size == B and batch["back_m"].dtype == torch.float64
        assert batch["crop_m"].is_pinned() == torch.cuda.is_available()
        for b in range(B):
            t = crop.landmark_box_transform(lm[b], 1.4, 224)
            assert np.array_equal(batch["back_m"][b].numpy().reshape(3, 3), t.params)
            assert np.array_equal(batch["crop_m"][b].numpy().reshape(3, 3), t.inverse.params)
            kpt = np.dot(t.params, np.hstack([lm[b, :, :2], np.ones([lm.shape[1], 1])]).T).T[:, :2]     # demo_video.py:130-131
            assert np.array_equal(batch["kpt"][b].numpy(), kpt.astype(np.int32))
    # degenerate boxes (one point, one line) take the one-frame path and still agree
    lm = np.zeros((3, 5, 2))
    lm[1, :, 0] = np.arange(5) * 10.0
    lm[2] = 100.0
    lm[2, 0] = 160.0
    T = video.box_transforms(lm)
    for b in range(3):
        assert np.array_equal(T[b], crop.landmark_box_transform(lm[b], 1.4, 224).params, equal_nan=True)


def test_prepare_rejects_bad_landmarks():
    stage = video.VideoStage((64, 64))
    with pytest.raises(ValueError):
        stage.prepare(np.zeros((5, 2)))
    with pytest.raises(ValueError):
        video.VideoStage((0, 64))


@pytest.mark.parametrize("render_orig", [False, True])
def test_compose_oracle_equals_the_demo_video_restatement(render_orig):
    pytest.importorskip("cv2")
    from oracle import warp_ref
    rng = np.random.default_rng(11 + render_orig)
    B, H, W = 3, 97, 131
    frames = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    lm = _landmarks(rng, B, H, W, L=40) * 0.3 + np.array([W * 0.35, H * 0.35, 0.0])
    T = video.box_transforms(lm)
    crops_u8 = np.stack([warp_ref.warp_ref(frames[b], np.linalg.inv(T[b]), (224, 224)) for b in range(B)])
    crop_f = np.ascontiguousarray(crops_u8[..., ::-1].transpose(0, 3, 1, 2)).astype(np.float32) / np.float32(255.0)
    rend = video_ref.special_renders(rng, B)
    got = video_ref.compose_ref(frames, crop_f, [rend], T, render_orig)
    for b in range(B):
        want = video_ref.demo_video_grid(frames[b], T[b], crops_u8[b], torch.from_numpy(rend[b:b + 1]), render_orig)
        assert got[b].shape == want.shape and np.array_equal(got[b], want), b
