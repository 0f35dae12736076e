"""TEST INFRASTRUCTURE — CPU oracles of the video demo's output grid (``demo_video.py:139-150,171,211-213`` with ``--crop``).

``demo_video_grid`` restates the script's per-frame steps literally (torch tensors, cv2 colour conversion, scikit-image's
``warp`` through its restatement ``oracle.warp_ref``); ``compose_ref`` is what ``smk_video_compose`` claims to compute, in
numpy, on a batch.  tests/test_video_host.py shows the two agree; the GPU suite compares the kernel with ``compose_ref``.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import warp_ref  # noqa: E402


def to_u8(x):
    """(x * 255).astype(np.uint8) on a float32 array, as numpy does it."""
    return (np.asarray(x, np.float32) * np.float32(255.0)).astype(np.uint8)


def compose_ref(frames, crop, panels, back_m, render_orig):
    """frames uint8 [B,H,W,3] BGR; crop float32 [B,3,S,S] RGB; panels: list of float32 [B,3,S,S] RGB in [0,1];
    back_m float64 [B,3,3] (frame -> crop, tform.params).  Returns uint8 [B,Hout,(len(panels)+1)*Wout,3] BGR."""
    rows = []
    H, W = frames.shape[1:3]
    for b in range(frames.shape[0]):
        cols = [frames[b] if render_orig else to_u8(crop[b].transpose(1, 2, 0))[..., ::-1]]
        for p in panels:
            u8 = to_u8(p[b].transpose(1, 2, 0))                                          # RGB HWC
            cols.append((warp_ref.warp_ref(u8, back_m[b], (H, W)) if render_orig else u8)[..., ::-1])
        rows.append(np.concatenate(cols, 1))
    return np.ascontiguousarray(np.stack(rows))


def demo_video_grid(image, tform_params, cropped_u8, rendered_img, render_orig):
    """One frame of demo_video.py with --crop: image uint8 [H,W,3] BGR (cap.read()), tform_params 3x3 (crop_face),
    cropped_u8 uint8 [224,224,3] BGR (the warp of line 128), rendered_img float32 torch [1,3,224,224].  Returns the
    uint8 array the script passes to cap_out.write."""
    import cv2
    video_height, video_width = image.shape[:2]
    cropped_image = cv2.cvtColor(cropped_u8, cv2.COLOR_BGR2RGB)                           # demo_video.py:134-136
    cropped_image = cv2.resize(cropped_image, (224, 224))
    cropped_image = torch.tensor(cropped_image).permute(2, 0, 1).unsqueeze(0).float() / 255.0
    if render_orig:                                                                       # demo_video.py:146-157
        rendered_img_numpy = (rendered_img.squeeze(0).permute(1, 2, 0).detach().cpu().numpy() * 255.0).astype(np.uint8)
        rendered_img_orig = warp_ref.warp_ref(rendered_img_numpy, tform_params, (video_height, video_width))
        rendered_img_orig = torch.Tensor(rendered_img_orig).permute(2, 0, 1).unsqueeze(0).float() / 255.0
        full_image = torch.Tensor(cv2.cvtColor(image, cv2.COLOR_BGR2RGB)).permute(2, 0, 1).unsqueeze(0).float() / 255.0
        grid = torch.cat([full_image, rendered_img_orig], dim=3)
    else:
        grid = torch.cat([cropped_image, rendered_img], dim=3)                            # demo_video.py:160
    grid_numpy = grid.squeeze(0).permute(1, 2, 0).detach().cpu().numpy() * 255.0          # demo_video.py:211-213
    grid_numpy = grid_numpy.astype(np.uint8)
    return cv2.cvtColor(grid_numpy, cv2.COLOR_BGR2RGB)


def special_renders(rng, B, S=224):
    """Renders with a background of exact zeros and values at and within one float32 ulp of k / 255."""
    x = rng.random((B, 3, S, S), dtype=np.float32)
    k = rng.integers(0, 256, size=x.shape).astype(np.float32) / np.float32(255.0)
    pick = rng.integers(0, 5, size=x.shape)
    x = np.where(pick == 1, k, x)
    x = np.where(pick == 2, np.nextafter(k, np.float32(0)), x)
    x = np.where(pick == 3, np.nextafter(k, np.float32(2)), x)
    x = np.clip(x, 0, 1).astype(np.float32)
    x[:, :, :30] = 0.0
    x[:, :, -3:] = 1.0
    return x
