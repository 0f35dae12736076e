"""TEST INFRASTRUCTURE — CPU oracles of the video demo without ``--crop`` (``demo_video.py:130-160,198-213``).

``cv2_resize_ref`` restates ``cv2.resize(img, (S, S))`` (INTER_LINEAR, uint8, 3 channels) as integer numpy, the rule
``smk_crop_warp`` with a NULL matrix claims to compute; ``torch_bilinear_ref`` restates torch's
``upsample_bilinear2d`` (align_corners=False, no scale factor) in float32 numpy, one rounding per operation, the rule
of ``smk_video_compose``'s mode 2; ``compose_resize_ref`` is that mode's grid on a batch.  ``demo_video_grid_nocrop``
restates the script's per-frame steps literally with cv2 and torch.  tests/test_resize_host.py shows each oracle equals
what it restates; the GPU suite compares the kernels with the oracles.
"""
import numpy as np

from video_ref import to_u8

F32 = np.float32

# frame-sized, pre-cropped, 2x (cv2's area fast path), non-square, upscales, degenerate and identity shapes
SHAPES = [(1080, 1920), (720, 1280), (480, 640), (512, 512), (448, 448), (896, 896), (672, 672), (300, 400), (1000, 999),
          (225, 224), (224, 448), (448, 224), (100, 100), (112, 112), (160, 120), (223, 225), (50, 300), (1, 1), (2, 3),
          (7, 500), (500, 7), (224, 224)]


def frame_contents(rng, H, W):
    """Random, constant, 0 / 255 extremes and gradient frames."""
    grad = (np.arange(H)[:, None, None] * 7 + np.arange(W)[None, :, None] * 3 + np.arange(3) * 50) % 256
    return [rng.integers(0, 256, (H, W, 3), dtype=np.uint8), np.full((H, W, 3), 173, np.uint8),
            (rng.integers(0, 2, (H, W, 3)) * 255).astype(np.uint8), grad.astype(np.uint8)]


def _linear_taps(src, dst, clamp):
    """cv2's fixed-point INTER_LINEAR taps along one axis: first source index (unclamped), weights a0, a1 (sum 2048)."""
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * (np.float64(src) / dst) - 0.5).astype(F32)
    s = np.floor(f)
    f = (f - s).astype(F32)
    s = s.astype(np.int64)
    if clamp:                                   # horizontal taps only: cv2 leaves the vertical weights as computed
        lo, hi = s < 0, s >= src - 1
        f[lo | hi] = 0
        s[lo] = 0
        s[hi] = src - 1
    a0 = np.rint((F32(1) - f) * F32(2048)).astype(np.int64)
    a1 = np.rint(f * F32(2048)).astype(np.int64)
    return s, a0, a1


def cv2_resize_ref(img, S=224):
    """``cv2.resize(img, (S, S))`` of a uint8 [H,W,3] image, bit for bit (OpenCV 4.x, INTER_LINEAR)."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[:2]
    if (H, W) == (S, S):
        return img.copy()
    x = img.astype(np.int64)
    if (H, W) == (2 * S, 2 * S):                # cv2 switches an exact 2x on both axes to its INTER_AREA fast path
        return ((x[0::2, 0::2] + x[0::2, 1::2] + x[1::2, 0::2] + x[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    sx, a0, a1 = _linear_taps(W, S, True)
    h = x[:, sx] * a0[None, :, None] + x[:, np.minimum(sx + 1, W - 1)] * a1[None, :, None]        # [H,S,3]
    sy, b0, b1 = _linear_taps(H, S, False)
    h0 = h[np.clip(sy, 0, H - 1)] >> 4
    h1 = h[np.clip(sy + 1, 0, H - 1)] >> 4
    v = (((h0 * b0[:, None, None]) >> 16) + ((h1 * b1[:, None, None]) >> 16) + 2) >> 2     # cv2's SIMD rounding
    return np.clip(v, 0, 255).astype(np.uint8)


# torch's own kernels may fuse the source-index arithmetic scale * (d + 0.5) - 0.5 into one rounding, so their sample
# positions may differ from this rule's by one float32 ulp of an index below 256 (2^-16): a resized value then differs by
# at most 2^-16 times the step between its taps, which are in [0, 1].
FUSED_INDEX_TOL = 2.0 ** -16


def _bilinear_index(src, dst):
    """torch's area_pixel_compute_source_index (align_corners=False) in float32: i0, i1, lambda0, lambda1."""
    scale = F32(src) / F32(dst)
    r = np.maximum(scale * (np.arange(dst).astype(F32) + F32(0.5)) - F32(0.5), F32(0))
    i0 = r.astype(np.int64)
    l1 = r - i0.astype(F32)
    return i0, i0 + (i0 < src - 1), F32(1) - l1, l1


def torch_bilinear_ref(x, H, W):
    """``F.interpolate(x, (H, W), mode='bilinear')`` of float32 [..., 3, S, S] as torch's CUDA kernel writes it, with
    every product and sum rounded to float32 (no fused multiply-add)."""
    x = np.asarray(x, F32)
    h0, h1, hl0, hl1 = _bilinear_index(x.shape[-2], H)
    w0, w1, wl0, wl1 = _bilinear_index(x.shape[-1], W)
    r0, r1 = x[..., h0, :], x[..., h1, :]
    top = wl0 * r0[..., w0] + wl1 * r0[..., w1]
    bot = wl0 * r1[..., w0] + wl1 * r1[..., w1]
    return hl0[:, None] * top + hl1[:, None] * bot


def compose_resize_ref(frames, panels):
    """``smk_video_compose`` mode 2: frames uint8 [B,H,W,3] BGR; panels: list of float32 [B,3,S,S] RGB in [0,1].
    Returns uint8 [B,H,(len(panels)+1)*W,3] BGR: the frame, then each panel resized to the frame."""
    H, W = frames.shape[1:3]
    cols = [frames] + [to_u8(torch_bilinear_ref(p, H, W).transpose(0, 2, 3, 1))[..., ::-1] for p in panels]
    return np.ascontiguousarray(np.concatenate(cols, 2))


def demo_video_grid_nocrop(image, rendered_img, render_orig, reconstructed_img=None):
    """One frame of demo_video.py without --crop: image uint8 [H,W,3] BGR (cap.read()), rendered_img (and
    reconstructed_img) float32 torch [1,3,224,224].  Returns the cropped_image tensor the encoder reads and the uint8
    array the script passes to cap_out.write."""
    import cv2
    import torch
    import torch.nn.functional as F
    video_height, video_width = image.shape[:2]
    cropped_image = cv2.cvtColor(image, cv2.COLOR_BGR2RGB)                                # demo_video.py:130,134-136
    cropped_image = cv2.resize(cropped_image, (224, 224))
    cropped_image = torch.tensor(cropped_image).permute(2, 0, 1).unsqueeze(0).float() / 255.0
    if render_orig:                                                                       # demo_video.py:153-157
        rendered_img_orig = F.interpolate(rendered_img, (video_height, video_width), mode='bilinear').cpu()
        full_image = torch.Tensor(cv2.cvtColor(image, cv2.COLOR_BGR2RGB)).permute(2, 0, 1).unsqueeze(0).float() / 255.0
        grid = torch.cat([full_image, rendered_img_orig], dim=3)
    else:
        grid = torch.cat([cropped_image, rendered_img], dim=3)
    if reconstructed_img is not None:                                                     # demo_video.py:198-209
        if render_orig:
            reconstructed_img_orig = F.interpolate(reconstructed_img, (video_height, video_width), mode='bilinear').cpu()
            grid = torch.cat([grid, reconstructed_img_orig], dim=3)
        else:
            grid = torch.cat([grid, reconstructed_img], dim=3)
    grid_numpy = grid.squeeze(0).permute(1, 2, 0).detach().cpu().numpy() * 255.0          # demo_video.py:211-213
    grid_numpy = grid_numpy.astype(np.uint8)
    return cropped_image, cv2.cvtColor(grid_numpy, cv2.COLOR_BGR2RGB)
