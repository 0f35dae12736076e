"""Masking between Renderer and SmirkGenerator on the GPU (SURVEY.md §8f #1).

Mirrors ``src/utils/masking.py``: ``mesh_based_mask_uniform_faces`` and ``masking`` keep the reference's names,
arguments and return values.  Random draws (multinomial, rand, randn, bernoulli) are made with torch on the tensors'
device, exactly where the reference makes them; the deterministic parts run in ``csrc/masking.cu``.
"""
import torch

from . import _lib


class MaskingContext:
    """Native handle for one mesh topology on one device (the reference passes ``flame.faces_tensor`` on every call)."""

    def __init__(self, faces, n_verts, device):
        f, fp = _lib.i32(faces)
        self.n_verts, self.n_faces = int(n_verts), int(f.shape[0])
        self.handle = _lib.create("masking", _lib.SmkMaskingDesc(self.n_verts, self.n_faces, fp), device)

    def workspace(self, B, S, device):
        n = _lib.call("smk_masking_workspace_bytes", device, self.handle, B, S)
        return torch.empty(n, dtype=torch.uint8, device=device)


_CTX = {}


def _context(flame_faces, n_verts, device):
    key = (flame_faces.data_ptr(), int(flame_faces.shape[0]), int(n_verts), device)
    if key not in _CTX:
        _CTX[key] = MaskingContext(flame_faces, n_verts, device)
    return _CTX[key]


def random_barycentric(num=1, device="cpu"):
    """masking.py:55-68 (drawn on ``device``)."""
    u, v = torch.rand(num, device=device), torch.rand(num, device=device)
    outside = u + v > 1
    u[outside], v[outside] = 1 - u[outside], 1 - v[outside]
    return torch.stack((1 - (u + v), u, v), dim=1)


def face_weights(flame_trans_verts, flame_faces, face_probabilities):
    """masking.py:146-160: sampling weight of every face, [B,F]."""
    _lib.require_cuda(flame_trans_verts, "flame_trans_verts")
    tv = flame_trans_verts.float().contiguous()
    B, V = tv.shape[:2]
    ctx = _context(flame_faces, V, tv.device)
    w = torch.empty(B, ctx.n_faces, dtype=torch.float32, device=tv.device)
    if B == 0:
        return w
    ws = ctx.workspace(B, 224, tv.device)
    bp = face_probabilities.to(tv.device, torch.float32).contiguous()
    _lib.call("smk_masking_face_weights", tv.device, ctx.handle, tv, bp, B, w, ws, ws.numel())
    return w


def mesh_based_mask_uniform_faces(flame_trans_verts, flame_faces, face_probabilities, mask_ratio=0.1, coords=None, IMAGE_SIZE=224):
    """masking.py:132-181 — same arguments and return value ``(npoints, coords)``."""
    _lib.require_cuda(flame_trans_verts, "flame_trans_verts")
    tv = flame_trans_verts.float().contiguous()
    B, V = tv.shape[:2]
    num = int(mask_ratio * IMAGE_SIZE * IMAGE_SIZE)
    if coords is None:
        w = face_weights(tv, flame_faces, face_probabilities)
        idx = torch.multinomial(w, num, replacement=True)
        bary = random_barycentric(B * num, tv.device).view(B, num, 3)
    else:
        idx, bary = coords["sampled_faces_indices"], coords["barycentric_coords"]
    idx = idx.to(tv.device, torch.int64).contiguous()
    bary = bary.to(tv.device, torch.float32).contiguous()
    ctx = _context(flame_faces, V, tv.device)
    npoints = torch.empty(B, idx.shape[1], 2, dtype=torch.int64, device=tv.device)
    if B and idx.shape[1]:
        _lib.call("smk_masking_points", tv.device, ctx.handle, tv, idx, bary, B, idx.shape[1], IMAGE_SIZE, npoints)
    return npoints, {"sampled_faces_indices": idx, "barycentric_coords": bary}


def masking_from_points(img, mask, npoints, rbound, wr=15, rendered_mask=None, noise_mult=None, random_centres=None, flame_faces=None, n_verts=5023):
    """demo.py:154-163 + masking.py:71-102 fused: point mask of the first ``rbound[b]`` points, dilation, noise, random
    patches, composite.  ``noise_mult`` / ``random_centres`` are the two random tensors of ``masking()`` (None = off)."""
    _lib.require_cuda(img, "img")
    img = img.float().contiguous()
    B, _, S, _ = img.shape
    ctx = _context(flame_faces, n_verts, img.device) if flame_faces is not None else next(iter(_CTX.values()))
    out = torch.empty_like(img)
    if B == 0:
        return out
    hull, rmask, noise, centres = [t.to(img.device, torch.float32).contiguous() if t is not None else None
                                   for t in (mask, rendered_mask, noise_mult, random_centres)]
    npts = npoints[..., :2].to(img.device, torch.int64).contiguous()      # the reference's npoints may carry a third (z) column
    rb = rbound.to(img.device, torch.int64).contiguous()
    ws = ctx.workspace(B, S, img.device)
    _lib.call("smk_masking_compose", img.device, ctx.handle, img, hull, npts, rb, npts.shape[1], None, rmask, noise, centres,
              int(wr), B, S, out, ws, ws.numel())
    return out


def transfer_pixels(img, points1, points2, rbound=None):
    """masking.py:116-129 — same arguments and result.  With duplicate targets the last pair in index order wins."""
    _lib.require_cuda(img, "img")
    img = img.float().contiguous()
    B, _, S, _ = img.shape
    p1 = points1[..., :2].to(img.device, torch.int64).contiguous()
    p2 = points2[..., :2].to(img.device, torch.int64).contiguous()
    rb = rbound.to(img.device, torch.int64).contiguous() if rbound is not None else None
    out = torch.empty_like(img)
    if B == 0:
        return out
    ws = torch.empty(B * S * S, dtype=torch.int32, device=img.device)
    _lib.call("smk_masking_transfer_pixels", img.device, img, p1, p2, rb, B, p1.shape[1], S, out, ws, ws.numel() * 4)
    return out


def masking(img, mask, extra_points, wr=15, rendered_mask=None, extra_noise=True, random_mask=0.01, flame_faces=None, n_verts=5023):
    """masking.py:71-102 — same arguments and result; the two random draws are made with torch on the image's device
    (as the reference does), the dilation / composite runs in ``csrc/masking.cu``."""
    _lib.require_cuda(img, "img")
    img = img.float().contiguous()
    B, _, S, _ = img.shape
    ctx = _context(flame_faces, n_verts, img.device) if flame_faces is not None else (next(iter(_CTX.values())) if _CTX else MaskingContext(torch.tensor([[0, 1, 2]]), 3, img.device))
    noise = (torch.randn_like(img) * 0.05 + 1) if extra_noise else None
    centres = torch.bernoulli(torch.ones((B, 1, S, S), device=img.device) * random_mask) if random_mask > 0 else None
    f = lambda t: None if t is None else t.to(img.device, torch.float32).contiguous()
    hull, extra, rmask = f(mask), f(extra_points), f(rendered_mask)
    out = torch.empty_like(img)
    if B == 0:
        return out
    ws = ctx.workspace(B, S, img.device)
    _lib.call("smk_masking_compose", img.device, ctx.handle, img, hull, None, None, 0, extra, rmask, noise, centres,
              int(wr), B, S, out, ws, ws.numel())
    return out


class MaskingStage(_lib.NativeModule):
    """The masking step of the full cycle (``demo.py:138-165``) as one capturable device call:
    ``rendered_img, transformed_vertices, img, hull_mask -> masked_img`` with every random draw made on the device by a
    counter-based generator (``csrc/masking.cu``, Philox4x32-10).  ``rng_state`` = (seed, call counter) lives in device
    memory; each call advances the counter on the stream, so a CUDA-graph replay draws fresh samples.

    Parameters follow the script: ``mask_ratio = 0.01``, ``mask_ratio_mul = 5`` (upper bound on the sampled points),
    ``mask_dilation_radius = 10``; ``extra_noise`` / ``random_mask`` are ``masking()``'s defaults (masking.py:71)."""

    def __init__(self, flame_faces, face_probabilities, n_verts=5023, mask_ratio=0.01, mask_ratio_mul=5, mask_dilation_radius=10,
                 extra_noise=True, random_mask=0.01, image_size=224, seed=0):
        self.faces = flame_faces.detach().to("cpu", torch.int64)
        self.n_verts, self.S = int(n_verts), int(image_size)
        self.base_prob_host = face_probabilities.detach().to("cpu", torch.float32).contiguous()
        self.ratio_mul, self.wr = float(mask_ratio_mul), int(mask_dilation_radius)
        self.N = int(mask_ratio * mask_ratio_mul * image_size * image_size)
        self.extra_noise, self.p_centre, self.seed = bool(extra_noise), float(random_mask), int(seed)

    def _native_key(self, device):              # one topology handle, made on the device of the first call
        return ()

    def _native_create(self, device):
        return MaskingContext(self.faces, self.n_verts, device)

    def _state(self, device):
        ctx, per_device = self._native_handle(device), self._native.per_device
        if device not in per_device:
            rng = torch.tensor([self.seed, 0], dtype=torch.int64, device=device)
            per_device[device] = (self.base_prob_host.to(device), rng)
        return (ctx,) + per_device[device]

    def reseed(self, seed, counter=0):
        self.seed = int(seed)
        for _, rng in self._native.per_device.values():
            rng.copy_(torch.tensor([self.seed, int(counter)], dtype=torch.int64))

    @torch.no_grad()
    def forward(self, img, hull_mask, transformed_vertices, rendered_img, debug=False):
        _lib.require_cuda(img, "img")
        dev = img.device
        img, hull = _lib.dev_f32(img, "img"), _lib.dev_f32(hull_mask, "hull_mask")
        tv, rend = _lib.dev_f32(transformed_vertices, "transformed_vertices"), _lib.dev_f32(rendered_img, "rendered_img")
        B, S, N = img.shape[0], self.S, self.N
        if tuple(img.shape[1:]) != (3, S, S) or tuple(rend.shape) != tuple(img.shape) or hull.numel() != B * S * S or tuple(tv.shape) != (B, self.n_verts, 3):
            raise RuntimeError("smirk_b200.MaskingStage: expected img/rendered [B,3,%d,%d], hull [B,1,%d,%d], transformed_vertices [B,%d,3]" % (S, S, S, S, self.n_verts))
        ctx, base_prob, rng = self._state(dev)
        out = torch.empty_like(img)
        dbg = {}
        if debug:
            i64 = lambda *s: torch.empty(*s, dtype=torch.int64, device=dev)
            f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            dbg = dict(sampled_faces_indices=i64(B, N), barycentric_coords=f32(B, N, 3), npoints=i64(B, N, 2), rbound=i64(B),
                       noise_mult=f32(B, 3, S, S), random_centres=f32(B, 1, S, S))
        ws = self._native_workspace("forward", _lib.call("smk_masking_forward_workspace_bytes", dev, ctx.handle, B, S, N), dev)
        _lib.call("smk_masking_forward", dev, ctx.handle, img, hull, tv, rend, base_prob, B, S, N, self.wr, self.ratio_mul,
                  self.p_centre, 1 if self.extra_noise else 0, rng, out,
                  *[dbg.get(k) for k in ("sampled_faces_indices", "barycentric_coords", "npoints", "rbound", "noise_mult", "random_centres")],
                  ws, ws.numel())
        return (out, dbg) if debug else out

    __call__ = forward


class TrainMaskingStage(_lib.NativeModule):
    """The reference trainer's masking (``src/smirk_trainer.py``: step1 at :76-92, step2 at :262-293) as one capturable
    device call per path, every random draw made on the device by the counter-based generator of ``MaskingStage``
    (``include/smirk_b200.h``).  Unlike the demo's step it keeps all ``int(mask_ratio * S^2)`` sampled points, and
    the second path moves the pixels under points sampled on the first path's mesh onto the augmented mesh.

    ``first_path(img, hull_mask, transformed_vertices, rendered_img)``: ``masking(img, hull, transfer_pixels(img, p, p),
    wr, rendered_mask = 1 - all(rendered == 0), random_mask = 0.01)``.
    ``second_path(img, hull_mask, transformed_vertices, transformed_vertices_2nd, rendered_img_2nd, Ke)``: points sampled on
    ``transformed_vertices`` [B] and placed on ``transformed_vertices_2nd`` [Ke*B]; ``transfer_pixels(img.repeat(Ke),
    points1.repeat(Ke), points2)``, ``rendered_mask = all(rendered_2nd > 0)``, ``random_mask = 0.005``; [Ke*B,3,S,S] out.
    ``rng_state`` = (seed, call counter) lives in device memory and each call advances the counter on the stream."""

    FIRST_RANDOM_MASK, SECOND_RANDOM_MASK = 0.01, 0.005          # smirk_trainer.py:90 (masking()'s default), :293
    DEBUG_KEYS = ("sampled_faces_indices", "barycentric_coords", "points1", "points2", "noise_mult", "random_centres")

    def __init__(self, flame_faces, face_probabilities, mask_ratio=0.01, mask_dilation_radius=10, image_size=224, seed=0, n_verts=5023):
        self.faces = flame_faces.detach().to("cpu", torch.int64)
        self.n_verts, self.S, self.wr = int(n_verts), int(image_size), int(mask_dilation_radius)
        self.base_prob_host = face_probabilities.detach().to("cpu", torch.float32).contiguous()
        self.N = int(mask_ratio * image_size * image_size)                   # masking.py:140
        self.seed = int(seed)

    def _native_key(self, device):
        return ()

    def _native_create(self, device):
        return MaskingContext(self.faces, self.n_verts, device)

    _state = MaskingStage._state
    reseed = MaskingStage.reseed

    def graph_keep_alive(self):
        return (self._native.handle,) + tuple(w.buf for w in self._native.workspaces.values())

    def _check(self, name, t, shape):
        if tuple(t.shape) != tuple(shape):
            raise RuntimeError("smirk_b200.TrainMaskingStage: %s must be %s, got %s" % (name, list(shape), list(t.shape)))

    @torch.no_grad()
    def _run(self, step, img, hull_mask, tv, tv2, rendered, Ke, debug):
        _lib.require_cuda(img, "img")
        dev = img.device
        img, hull, tv, rend = (_lib.dev_f32(t, n) for t, n in ((img, "img"), (hull_mask, "hull_mask"), (tv, "transformed_vertices"),
                                                                (rendered, "rendered_img")))
        B, S, N, R = img.shape[0], self.S, self.N, img.shape[0] * Ke
        self._check("img", img, (B, 3, S, S))
        self._check("hull_mask", hull, (B, 1, S, S))
        self._check("transformed_vertices", tv, (B, self.n_verts, 3))
        self._check("rendered_img", rend, (R, 3, S, S))
        if tv2 is not None:
            tv2 = _lib.dev_f32(tv2, "transformed_vertices_2nd")
            self._check("transformed_vertices_2nd", tv2, (R, self.n_verts, 3))
        ctx, base_prob, rng = self._state(dev)
        out = torch.empty(R, 3, S, S, dtype=torch.float32, device=dev)
        dbg = {}
        if debug:
            i64 = lambda *s: torch.empty(*s, dtype=torch.int64, device=dev)
            f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            dbg = dict(sampled_faces_indices=i64(B, N), barycentric_coords=f32(B, N, 3), points1=i64(B, N, 2),
                       noise_mult=f32(R, 3, S, S), random_centres=f32(R, 1, S, S))
            if step == 2:
                dbg["points2"] = i64(R, N, 2)
        p = self.FIRST_RANDOM_MASK if step == 1 else self.SECOND_RANDOM_MASK
        nbytes = _lib.call("smk_masking_train_workspace_bytes", dev, ctx.handle, B, Ke, S, N)
        ws = self._native_workspace("step%d" % step, nbytes, dev)
        _lib.call("smk_masking_train_forward", dev, ctx.handle, step, img, hull, tv, tv2, rend, base_prob, B, Ke, S, N, self.wr, p,
                  rng, out, *[dbg.get(k) for k in self.DEBUG_KEYS], ws, ws.numel())
        return (out, dbg) if debug else out

    def first_path(self, img, hull_mask, transformed_vertices, rendered_img, debug=False):
        return self._run(1, img, hull_mask, transformed_vertices, None, rendered_img, 1, debug)

    def second_path(self, img, hull_mask, transformed_vertices, transformed_vertices_2nd, rendered_img_2nd, Ke=1, debug=False):
        if int(Ke) < 1:
            raise RuntimeError("smirk_b200.TrainMaskingStage: Ke must be >= 1")
        return self._run(2, img, hull_mask, transformed_vertices, transformed_vertices_2nd, rendered_img_2nd, int(Ke), debug)
