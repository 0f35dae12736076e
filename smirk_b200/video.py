"""The frame loop of the reference's video demo (``demo_video.py:107-214``) as a stage of ``SmirkPipeline``.

    stage = VideoStage(frame_hw=(1080, 1920), render_orig=True)        # demo_video.py --crop [--render_orig]
    pipe  = SmirkPipeline(enc, flame, renderer, video=stage, slots=2)
    batch = stage.prepare(landmarks)          # host: [B,L,2|3] landmarks -> the B crop transforms, in pinned memory
    out   = pipe.forward(frames_u8_cuda, batch)            # eager
    out   = pipe.submit(i, frames_u8_cuda, batch)          # graph replay on lane i % slots
    out   = pipe.run_host(frames_pinned, i, batch, keys=("grid",))

    stage = VideoStage((512, 512), render_orig=True, crop=False)       # demo_video.py [--render_orig] without --crop
    batch = stage.prepare(batch_size=B)       # or stage.prepare(landmarks) with a generator (the hull mask's points)

Per batch of uint8 BGR frames [B,H,W,3] on the device the pipeline crops (``smk_crop_warp``: ``warp(image,
tform.inverse, (224, 224))`` + BGR2RGB + /255), runs encoder -> FLAME -> renderer, and writes ``out["grid"]``, uint8 BGR
[B, Hout, k * Wout, 3]: row i is the image ``demo_video.py:211-214`` passes to ``cap_out.write`` for frame i
(``smk_video_compose``; Hout x Wout = H x W with ``render_orig``, 224 x 224 without; k = 2, or 3 with the generator).
With a generator (``--use_smirk_generator``, which needs ``masking=MaskingStage(...)``) the landmark hull mask of
``datasets/base_dataset.py:9-15`` is drawn on the device (``smk_hull_mask``) from the int32 crop landmarks, goes through
the masking step into the generator, and the reconstruction is the third panel.  The crop transforms and landmarks are
graph inputs, so one captured graph per (B, H, W) serves every batch.  The landmark detector and the video decode /
encode stay on the host, as in the reference.

Without ``--crop`` (``crop=False``; the reference's branch for face-aligned clips) the encoder reads
``cv2.resize(frame, (224, 224))`` (``smk_crop_warp`` without a matrix, bit for bit), and with ``render_orig`` each render
panel is ``F.interpolate(x, (H, W), mode='bilinear')`` of the reference (``smk_video_compose`` mode 2).  The hull mask
is drawn from the landmarks in frame pixels as the reference does (``create_mask(kpt, (224, 224))``: points outside the
224 x 224 mask are clipped there, not rescaled), and the batch holds no transforms.
"""
import numpy as np
import torch

from . import _lib

_CORNERS = np.array([[-1.0, -1.0], [-1.0, 1.0], [1.0, -1.0]])


def box_transforms(landmarks, scale=1.4, image_size=224):
    """[B,L,2|3] landmarks -> [B,3,3] float64 similarity transforms frame -> crop: ``crop.landmark_box_transform`` (the
    transform of ``demo_video.py:16-34``) for every frame at once, bitwise equal to it frame by frame."""
    pts = np.asarray(landmarks, np.float64)[..., :2]
    if pts.ndim != 3 or pts.shape[1] == 0:
        raise ValueError("landmarks must be [B,L,2] or [B,L,3] with L > 0")
    lo, hi = pts.min(axis=1), pts.max(axis=1)
    half = np.trunc(0.5 * (hi - lo).sum(axis=1) * scale) / 2.0                      # int(mean extent * scale) / 2
    centre = hi - (hi - lo) / 2.0
    src = centre[:, None, :] + half[:, None, None] * _CORNERS                         # [B,3,2]
    dst = (image_size - 1) * np.array([[0.0, 0.0], [0.0, 1.0], [1.0, 0.0]])
    # skimage's _umeyama (crop._umeyama), stacked over the batch
    B, num, dim = src.shape
    src_mean, dst_mean = src.mean(axis=1), dst.mean(axis=0)
    src_demean, dst_demean = src - src_mean[:, None, :], dst - dst_mean
    A = np.matmul(dst_demean.T, src_demean) / num
    d = np.ones((B, dim))
    d[np.linalg.det(A) < 0, dim - 1] = -1
    U, S, V = np.linalg.svd(A)
    rank = np.linalg.matrix_rank(A)
    if (rank != dim).any():
        # a degenerate box (all landmarks on one point or line): the rare case keeps the one-frame code
        from . import crop
        return np.stack([crop.landmark_box_transform(p, scale, image_size).params for p in pts])
    T = np.tile(np.eye(dim + 1), (B, 1, 1))
    D = np.zeros((B, dim, dim))
    D[:, range(dim), range(dim)] = d
    T[:, :dim, :dim] = np.matmul(np.matmul(U, D), V)
    sc = np.array([1.0 / src_demean[b].var(axis=0).sum() * (S[b] @ d[b]) for b in range(B)])
    T[:, :dim, dim] = dst_mean - sc[:, None] * np.matmul(T[:, :dim, :dim], src_mean[:, :, None])[..., 0]
    T[:, :dim, :dim] *= sc[:, None, None]
    return T


def crop_landmarks(landmarks, T):
    """demo_video.py:130-131 + create_mask's cast: the landmarks in crop pixels, ``(tform.params @ [kpt; 1])[:, :2]`` in
    float64 with numpy's ``dot`` frame by frame (as the script computes it), then ``astype(np.int32)``."""
    pts = np.asarray(landmarks, np.float64)[..., :2]
    out = np.empty(pts.shape, np.int32)
    for b in range(pts.shape[0]):
        k = np.dot(T[b], np.hstack([pts[b], np.ones([pts.shape[1], 1])]).T).T
        out[b] = k[:, :2].astype(np.int32)
    return out


class VideoBatch(dict):
    """The host side of one batch of ``size`` frames (``VideoStage.prepare``): ``crop_m`` / ``back_m``, pinned float64
    [B,9], the maps crop -> frame (inverse of the transform; what the crop warp samples with) and frame -> crop
    (``tform.params``; what the warp back to the frame samples with); ``kpt``, pinned int32 [B,L,2], the landmarks in
    crop pixels (the hull mask's input).  Without the crop only ``kpt`` (in frame pixels), or nothing."""

    def __init__(self, size, **tensors):
        super().__init__(**tensors)
        self.size = int(size)


class VideoStage:
    """Configuration and workspaces of the video stage; attach it with ``SmirkPipeline(..., video=stage)``.
    ``crop=False``: the reference's branch without ``--crop``, the whole frame resized to the encoder's input."""

    def __init__(self, frame_hw, render_orig=False, scale=1.4, image_size=224, n_landmarks=478, crop=True):
        self.frame_hw = (int(frame_hw[0]), int(frame_hw[1]))
        if min(self.frame_hw) <= 0:
            raise ValueError("frame_hw must be positive")
        self.render_orig, self.scale, self.S, self.L = bool(render_orig), float(scale), int(image_size), int(n_landmarks)
        self.use_crop = bool(crop)
        if not 1 <= self.L <= 1024:
            raise ValueError("n_landmarks must be in [1, 1024]")
        self._ws = {}

    def __deepcopy__(self, memo):
        new = VideoStage(self.frame_hw, self.render_orig, self.scale, self.S, self.L, self.use_crop)
        memo[id(self)] = new
        return new

    @property
    def out_hw(self):
        return self.frame_hw if self.render_orig else (self.S, self.S)

    def grid_shape(self, B, n_panels=1):
        Ho, Wo = self.out_hw
        return (B, Ho, (n_panels + 1) * Wo, 3)

    # ---- host ------------------------------------------------------------------------------------------------------------
    def prepare(self, landmarks=None, batch_size=None):
        """[B,L,2|3] landmarks (mediapipe's, in frame pixels) -> ``VideoBatch`` of pinned host tensors.  Without the crop
        the landmarks are only the hull mask's input (``kpt = landmarks.astype(np.int32)[..., :2]``, demo_video.py:131,171);
        a pipeline without a generator needs none: ``prepare(batch_size=B)`` gives an empty batch of B frames."""
        if landmarks is None:
            if self.use_crop:
                raise ValueError("VideoStage: the crop needs landmarks")
            if batch_size is None or int(batch_size) < 0:
                raise ValueError("VideoStage: without landmarks give batch_size >= 0")
            return VideoBatch(batch_size)
        lm = np.asarray(landmarks)
        if lm.ndim != 3 or lm.shape[1] != self.L:
            raise ValueError("VideoStage: expected landmarks [B,%d,2|3], got %s" % (self.L, lm.shape))
        if batch_size is not None and int(batch_size) != lm.shape[0]:
            raise ValueError("VideoStage: batch_size %d but %d landmark sets" % (batch_size, lm.shape[0]))
        cuda = torch.cuda.is_available()             # page-locked memory needs the driver; a host without one gets plain tensors
        pin = lambda a: (lambda t: t.pin_memory() if cuda else t)(torch.from_numpy(np.ascontiguousarray(a)))
        if not self.use_crop:
            return VideoBatch(lm.shape[0], kpt=pin(lm.astype(np.int32)[..., :2]))
        T = box_transforms(lm, self.scale, self.S)
        return VideoBatch(lm.shape[0], crop_m=pin(np.linalg.inv(T).reshape(-1, 9)), back_m=pin(T.reshape(-1, 9)),
                          kpt=pin(crop_landmarks(lm, T)))

    def check(self, frames, batch):
        if not (torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3):
            raise ValueError("VideoStage: frames must be a uint8 tensor [B,H,W,3] (BGR)")
        if tuple(frames.shape[1:3]) != self.frame_hw:
            raise ValueError("VideoStage: frames are %dx%d, the stage was made for %dx%d"
                             % (frames.shape[1], frames.shape[2], self.frame_hw[0], self.frame_hw[1]))
        if not isinstance(batch, VideoBatch):
            raise ValueError("VideoStage: the second input must be the VideoBatch of VideoStage.prepare")
        if batch.size != frames.shape[0]:
            raise ValueError("VideoStage: %d frames but %d landmark sets" % (frames.shape[0], batch.size))

    # ---- device ----------------------------------------------------------------------------------------------------------
    def _workspace(self, name, nbytes, device):
        return self._ws.setdefault(name, _lib.Workspace()).get(nbytes, device)

    def crop(self, frames, crop_m):
        """frames uint8 [B,H,W,3] BGR, crop_m float64 [B,9] on the device -> the encoder's input, float32 [B,3,S,S] RGB.
        Without the crop (crop_m unused) the input is cv2.resize of the whole frame."""
        dev = frames.device
        B, H, W, _ = frames.shape
        out = torch.empty(B, 3, self.S, self.S, dtype=torch.float32, device=dev)
        if B and not self.use_crop:
            _lib.call("smk_crop_warp", dev, frames, B, H, W, None, self.S, 1, out, None, 0)
        elif B:
            ws = self._workspace("crop", _lib.call("smk_warp_workspace_bytes", dev, B), dev)
            _lib.call("smk_crop_warp", dev, frames, B, H, W, crop_m, self.S, 1, out, ws, ws.numel())
        return out

    def hull_mask(self, kpt):
        """kpt int32 [B,L,2] crop landmarks (frame landmarks without the crop) on the device -> create_mask(kpt, (S, S))
        as float [B,1,S,S]."""
        dev = kpt.device
        B = kpt.shape[0]
        mask = torch.empty(B, 1, self.S, self.S, dtype=torch.float32, device=dev)
        if B:
            _lib.call("smk_hull_mask", dev, kpt, B, kpt.shape[1], self.S, mask)
        return mask

    def compose(self, frames, crop, panels, back_m):
        """The output grid: panel 0 = the frame (render_orig) or the crop, then each of ``panels`` ([B,3,S,S] in [0,1])
        warped back (or, without the crop, resized) to the frame with render_orig."""
        import ctypes as C
        dev = frames.device
        B, H, W, _ = frames.shape
        panels = [p.contiguous() for p in panels]
        grid = torch.empty(self.grid_shape(B, len(panels)), dtype=torch.uint8, device=dev)
        if not B:
            return grid
        ptrs = (C.c_void_p * len(panels))(*[p.data_ptr() for p in panels])
        if self.render_orig and not self.use_crop:              # mode 2: the panels resized to the frame, no workspace
            _lib.call("smk_video_compose", dev, frames, B, H, W, None, ptrs, len(panels), self.S, None, 2, grid, None, 0)
        else:
            ws = self._workspace("compose", _lib.call("smk_video_workspace_bytes", dev, B, len(panels)), dev)
            _lib.call("smk_video_compose", dev, frames, B, H, W, None if self.render_orig else crop, ptrs, len(panels),
                      self.S, back_m if self.render_orig else None, 1 if self.render_orig else 0, grid, ws, ws.numel())
        return grid

    def graph_keep_alive(self):
        return [w.buf for w in self._ws.values()]
