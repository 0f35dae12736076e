"""Crop / warp around the per-frame path for frames that live on the GPU (SURVEY.md §8f #2).

Mirrors the helpers the reference's entry scripts use (``demo.py:16-34,84-105``, ``demo_video.py:116-137,147-150``):

    tform = landmark_box_transform(landmarks, scale=1.4, image_size=224) # the crop transform of demo.py:16-34 (.params)
    img   = crop_to_tensor(frames_u8, [tform, ...])                      # warp(image, tform.inverse) + BGR2RGB + /255
    back  = warp_back(rendered, [tform, ...], (H, W))                    # warp(rendered_uint8, tform, (H, W))

``estimate_transform('similarity', src, dst)`` (skimage, Umeyama's method) is host-side numpy on three points;
the per-pixel work — skimage's ``_warp_fast`` bilinear gather in float64 with ``mode='constant'``, ``cval=0``,
clipping to the source range and truncation to uint8 — runs in ``csrc/warp.cu`` (``smk_crop_warp``, ``smk_warp_u8``).
The landmark detector (mediapipe) stays what it is in the reference: third-party, on the CPU.
"""
import numpy as np
import torch

from . import _lib


class SimilarityTransform:
    """The part of skimage.transform.SimilarityTransform the reference touches: ``params``, ``inverse``, call."""

    def __init__(self, matrix=None):
        self.params = np.eye(3) if matrix is None else np.asarray(matrix, np.float64)

    @property
    def inverse(self):
        return SimilarityTransform(np.linalg.inv(self.params))

    def __call__(self, coords):
        coords = np.asarray(coords, np.float64)
        h = np.hstack([coords, np.ones((coords.shape[0], 1))]) @ self.params.T
        return h[:, :2] / h[:, 2:3]


def _umeyama(src, dst, estimate_scale):
    # skimage/transform/_geometric.py::_umeyama (Umeyama 1991, eq. 34-43)
    num, dim = src.shape
    src_mean, dst_mean = src.mean(axis=0), dst.mean(axis=0)
    src_demean, dst_demean = src - src_mean, dst - dst_mean
    A = dst_demean.T @ src_demean / num
    d = np.ones((dim,), dtype=np.float64)
    if np.linalg.det(A) < 0:
        d[dim - 1] = -1
    T = np.eye(dim + 1, dtype=np.float64)
    U, S, V = np.linalg.svd(A)
    rank = np.linalg.matrix_rank(A)
    if rank == 0:
        return np.nan * T
    if rank == dim - 1:
        if np.linalg.det(U) * np.linalg.det(V) > 0:
            T[:dim, :dim] = U @ V
        else:
            s = d[dim - 1]
            d[dim - 1] = -1
            T[:dim, :dim] = U @ np.diag(d) @ V
            d[dim - 1] = s
    else:
        T[:dim, :dim] = U @ np.diag(d) @ V
    scale = 1.0 / src_demean.var(axis=0).sum() * (S @ d) if estimate_scale else 1.0
    T[:dim, dim] = dst_mean - scale * (T[:dim, :dim] @ src_mean.T)
    T[:dim, :dim] *= scale
    return T


def estimate_transform(ttype, src, dst):
    if ttype != "similarity":
        raise NotImplementedError("smirk_b200.crop.estimate_transform: only 'similarity' is on the reference's path")
    return SimilarityTransform(_umeyama(np.asarray(src, np.float64), np.asarray(dst, np.float64), True))


def landmark_box_transform(landmarks, scale=1.0, image_size=224):
    """Similarity transform frame -> crop for the square that bounds ``landmarks`` [L,2], grown by ``scale``.

    Produces the transform the reference's entry scripts build for their crops (``demo.py:16-34``: landmark bounding
    box -> square of side int(mean extent * scale) around the box centre -> three corners mapped onto the crop); the
    scripts keep their own helper, this one exists for callers that batch frames on the GPU (``crop_to_tensor``)."""
    pts = np.asarray(landmarks, np.float64)[:, :2]
    lo, hi = pts.min(axis=0), pts.max(axis=0)
    half = int(0.5 * float((hi - lo).sum()) * scale) / 2.0
    centre = hi - (hi - lo) / 2.0
    corners = centre + half * np.array([[-1.0, -1.0], [-1.0, 1.0], [1.0, -1.0]])
    target = (image_size - 1) * np.array([[0.0, 0.0], [0.0, 1.0], [1.0, 0.0]])
    return estimate_transform("similarity", corners, target)


def _matrices(tforms, invert, device):
    mats = []
    for t in tforms:
        p = np.asarray(t.params if hasattr(t, "params") else t, np.float64)
        if p.shape != (3, 3):
            raise ValueError("expected 3x3 transform parameters, got %s" % (p.shape,))
        if not (p[2, 0] == 0.0 and p[2, 1] == 0.0 and p[2, 2] == 1.0):
            raise ValueError("only affine transforms (last row 0 0 1) are supported")
        mats.append(np.linalg.inv(p) if invert else p)
    # pinned staging + asynchronous upload on the caller's stream: a pageable copy would stall the pipeline on every call
    host = torch.from_numpy(np.ascontiguousarray(np.stack(mats))).pin_memory()
    return host.to(device, non_blocking=True), host


def _workspace(B, device):
    return torch.empty(_lib.call("smk_warp_workspace_bytes", device, B), dtype=torch.uint8, device=device)


def crop_to_tensor(frames, tforms, image_size=224, bgr=True):
    """frames: uint8 CUDA tensor [B,H,W,3] (cv2 / BGR order when ``bgr``); tforms: B transforms frame -> crop (as
    returned by ``landmark_box_transform`` or the scripts' own ``crop_face``).  Returns float32 [B,3,S,S] in [0,1], RGB — what ``demo.py:97,103-105`` feeds the encoder."""
    _lib.require_cuda(frames, "frames")
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError("frames must be uint8 [B,H,W,3]")
    frames = frames.contiguous()
    B, H, W, _ = frames.shape
    if len(tforms) != B:
        raise ValueError("one transform per frame expected")
    out = torch.empty(B, 3, image_size, image_size, dtype=torch.float32, device=frames.device)
    if B == 0:
        return out
    m, _pinned = _matrices(tforms, True, frames.device)
    ws = _workspace(B, frames.device)
    _lib.call("smk_crop_warp", frames.device, frames, B, H, W, m, image_size, 1 if bgr else 0, out, ws, ws.numel())
    return out


def warp_back(rendered, tforms, out_hw):
    """rendered: float32 CUDA tensor [B,3,S,S] in [0,1]; returns uint8 [B,H,W,3] in frame coordinates
    (``demo_video.py:147-149``: ``warp((rendered*255).astype(uint8), tform, output_shape=(H, W))``)."""
    _lib.require_cuda(rendered, "rendered")
    if rendered.dtype != torch.float32 or rendered.dim() != 4 or rendered.shape[1] != 3 or rendered.shape[2] != rendered.shape[3]:
        raise ValueError("rendered must be float32 [B,3,S,S]")
    rendered = rendered.contiguous()
    B, _, S, _ = rendered.shape
    H, W = int(out_hw[0]), int(out_hw[1])
    if len(tforms) != B:
        raise ValueError("one transform per frame expected")
    dev = rendered.device
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
    if B == 0:
        return out
    u8 = torch.empty(B, S, S, 3, dtype=torch.uint8, device=dev)
    _lib.call("smk_f32chw_to_u8hwc", dev, rendered, B, S, u8)
    m, _pinned = _matrices(tforms, False, dev)
    ws = _workspace(B, dev)
    _lib.call("smk_warp_u8", dev, u8, B, S, S, m, H, W, out, ws, ws.numel())
    return out
