"""``Renderer`` — drop-in for the reference class ``src/renderer/renderer.py:49-207``.

Same constructor arguments, registered buffers (``state_dict`` keys: faces, face_colors, raw_uvcoords,
uvcoords, uvfaces, face_uvcoords, constant_factor) and ``forward`` output dict; the vertex stage,
normals, rasterisation (pytorch3d's ``rasterize_meshes`` in the reference) and shading run in
``csrc/render.cu`` through ``smk_renderer_forward``.  When grad mode is on and an input requires grad,
``forward`` is differentiable for the vertices, the camera and the landmark sets (``smk_renderer_backward``,
``smk_project_points_backward``); otherwise it is the plain forward.
"""
import pickle

import numpy as np
import torch
import torch.nn as nn

from . import _lib


def load_obj(path):
    """Minimal OBJ reader for what renderer.py:54-57 takes from pytorch3d.io.load_obj."""
    v, vt, f, ft = [], [], [], []
    with open(path) as fh:
        for ln in fh:
            if ln.startswith("v "):
                v.append(ln.split()[1:4])
            elif ln.startswith("vt "):
                vt.append(ln.split()[1:3])
            elif ln.startswith("f "):
                corners = [c.split("/") for c in ln.split()[1:]]
                for k in range(1, len(corners) - 1):          # fan-triangulate polygons
                    tri = (corners[0], corners[k], corners[k + 1])
                    f.append([int(c[0]) - 1 for c in tri])
                    ft.append([int(c[1]) - 1 if len(c) > 1 and c[1] else -1 for c in tri])
    return (torch.tensor(np.array(v, dtype=np.float32)), torch.tensor(np.array(f, dtype=np.int64)),
            torch.tensor(np.array(ft, dtype=np.int64)), torch.tensor(np.array(vt, dtype=np.float32)))


def keep_vertices_and_update_faces(faces, vertices_to_keep):
    """renderer.py:11-47: drop faces touching removed vertices, renumber the rest."""
    keep = torch.unique(torch.as_tensor(vertices_to_keep, dtype=torch.long))
    n = int(faces.max()) + 1
    remap = torch.full((n,), -1, dtype=torch.long)
    remap[keep] = torch.arange(len(keep))
    return remap[faces[(remap[faces] != -1).all(1)]]


def _face_vertices(vertices, faces):
    bs, nv = vertices.shape[:2]
    return vertices.reshape(bs * nv, -1)[(faces + (torch.arange(bs) * nv)[:, None, None]).long()]


class Renderer(_lib.NativeModule, nn.Module):
    def __init__(self, render_full_head=False, obj_filename="assets/head_template.obj"):
        super().__init__()
        self.image_size = 224
        verts, faces, uvfaces, uvcoords = load_obj(obj_filename)
        uvcoords, uvfaces, faces = uvcoords[None], uvfaces[None], faces[None]
        self.render_full_head = render_full_head
        self.n_verts = verts.shape[0]
        colors = torch.tensor([180, 180, 180])[None, None, :].repeat(1, int(faces.max()) + 1, 1).float() / 255.
        with open("assets/FLAME_masks/FLAME_masks.pkl", "rb") as fh:
            self.flame_masks = pickle.load(fh, encoding="latin1")
        if not render_full_head:
            self.final_mask = self.flame_masks["face"].tolist()
            faces = keep_vertices_and_update_faces(faces[0], self.final_mask).unsqueeze(0)
            colors = colors[:, self.final_mask, :]
        else:
            self.final_mask = list(range(self.n_verts))
        self.register_buffer("faces", faces)
        self.register_buffer("face_colors", _face_vertices(colors, faces))
        self.register_buffer("raw_uvcoords", uvcoords)
        uvcoords = torch.cat([uvcoords, uvcoords[:, :, 0:1] * 0. + 1.], -1)
        uvcoords = uvcoords * 2 - 1
        uvcoords[..., 1] = -uvcoords[..., 1]
        self.register_buffer("uvcoords", uvcoords)
        self.register_buffer("uvfaces", uvfaces)
        self.register_buffer("face_uvcoords", _face_vertices(uvcoords, uvfaces))
        pi = np.pi
        self.register_buffer("constant_factor", torch.tensor(
            [1 / np.sqrt(4 * pi), ((2 * pi) / 3) * (np.sqrt(3 / (4 * pi))), ((2 * pi) / 3) * (np.sqrt(3 / (4 * pi))),
             ((2 * pi) / 3) * (np.sqrt(3 / (4 * pi))), (pi / 4) * (3) * (np.sqrt(5 / (12 * pi))),
             (pi / 4) * (3) * (np.sqrt(5 / (12 * pi))), (pi / 4) * (3) * (np.sqrt(5 / (12 * pi))),
             (pi / 4) * (3 / 2) * (np.sqrt(5 / (12 * pi))), (pi / 4) * (1 / 2) * (np.sqrt(5 / (4 * pi)))]).float())

    def _native_key(self, device):              # the handle packs only the topology and the image size
        return str(device), self.faces._version, self.faces.data_ptr(), self.image_size

    def _native_create(self, device):
        mask_np, mask_p = _lib.i32(np.asarray(self.final_mask))
        faces_np, faces_p = _lib.i32(self.faces[0])
        d = _lib.SmkRendererDesc()
        d.n_verts, d.n_mask, d.mask_ids = self.n_verts, len(self.final_mask), mask_p
        d.n_faces, d.faces, d.image_size = faces_np.shape[0], faces_p, self.image_size
        # renderer.py:140-144: with the full head the fancy-index is skipped, so the in-place `z + 10` of render()
        # also lands in the tensor the reference returns as `transformed_vertices`
        d.z_offset = 10.0 if self.render_full_head else 0.0
        return _lib.create("renderer", d, device)

    def forward(self, vertices, cam_params, **landmarks):
        if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad
                                           for t in (vertices, cam_params, *landmarks.values())):
            return self._forward_autograd(vertices, cam_params, **landmarks)
        return self.render_full(vertices, cam_params, raw=False, **landmarks)

    def _forward_autograd(self, vertices, cam_params, **landmarks):
        """forward() with gradients for vertices, cam_params and every landmark set (smk_renderer_backward,
        smk_project_points_backward).  Saves the rasteriser's pix_to_face, bary and the vertex normals."""
        rendered, tverts = _RenderFunction.apply(self, vertices, cam_params)
        out = {"rendered_img": rendered, "transformed_vertices": tverts}
        for k, pts in landmarks.items():
            out[k] = _ProjectFunction.apply(pts, cam_params)
        return out

    @torch.no_grad()
    def render_full(self, vertices, cam_params, raw=True, **landmarks):
        """forward() plus, with ``raw=True``, the rasteriser's own outputs (pix_to_face int64 [B,S,S]
        packed like pytorch3d, bary [B,S,S,3], zbuf [B,S,S]) and the vertex normals [B,n_mask,3]."""
        _lib.require_cuda(vertices, "vertices")
        dev = vertices.device
        h = self._native_handle(dev)
        verts, cam = _lib.dev_f32(vertices, "vertices"), _lib.dev_f32(cam_params, "cam_params")
        B, S = verts.shape[0], self.image_size
        if verts.shape[1] != self.n_verts or cam.shape != (B, 3):
            raise RuntimeError("smirk_b200.Renderer: expected vertices [B,%d,3] and cam [B,3]" % self.n_verts)
        o = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        rendered, tverts = o(B, 3, S, S), o(B, self.n_verts, 3)
        p2f = torch.empty(B, S, S, dtype=torch.int64, device=dev) if raw else None
        bary, zbuf = (o(B, S, S, 3), o(B, S, S)) if raw else (None, None)
        normals = o(B, len(self.final_mask), 3) if raw else None
        out = {"rendered_img": rendered, "transformed_vertices": tverts}
        ws = self._native_workspace("forward", _lib.call("smk_renderer_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_renderer_forward", dev, h, verts, cam, B, rendered, tverts, p2f, bary, zbuf, normals, ws, ws.numel())
        for k, pts in landmarks.items():                                         # renderer.py:104-108
            pts = _lib.dev_f32(pts, k)
            xy = o(B, pts.shape[1], 2)
            _lib.call("smk_project_points", dev, pts, cam, B, pts.shape[1], xy)
            out[k] = xy
        if raw:
            out.update(pix_to_face=p2f, bary=bary, zbuf=zbuf, normals=normals)
        return out


def _grad_f32(g):
    return None if g is None else g.to(torch.float32).contiguous()


class _RenderFunction(torch.autograd.Function):
    """vertices, cam -> (rendered_img, transformed_vertices) through ``render_full(raw=True)``; the backward is
    ``smk_renderer_backward`` from the saved pix_to_face / bary / normals.  Serves the face mask and the full head;
    the full head's z offset on transformed_vertices is a constant, so its gradient passes through unchanged."""

    @staticmethod
    def forward(ctx, module, vertices, cam):
        r = module.render_full(vertices, cam, raw=True)
        ctx.module, ctx.dtypes = module, (vertices.dtype, cam.dtype)
        ctx.save_for_backward(_lib.dev_f32(vertices, "vertices"), _lib.dev_f32(cam, "cam_params"),
                              r["pix_to_face"], r["bary"], r["normals"])
        return r["rendered_img"], r["transformed_vertices"]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rendered, g_tverts):
        verts, cam, p2f, bary, normals = ctx.saved_tensors
        m, dev, B = ctx.module, verts.device, verts.shape[0]
        h = m._native_handle(dev)
        g_verts, g_cam = torch.empty_like(verts), torch.empty_like(cam)
        g_rendered, g_tverts = _grad_f32(g_rendered), _grad_f32(g_tverts)
        ws = m._native_workspace("backward", _lib.call("smk_renderer_backward_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_renderer_backward", dev, h, verts, cam, B, p2f, bary, normals, g_rendered, g_tverts, g_verts, g_cam,
                  ws, ws.numel())
        return None, g_verts.to(ctx.dtypes[0]), g_cam.to(ctx.dtypes[1])


class _ProjectFunction(torch.autograd.Function):
    """Landmark projection (renderer.py:104-108): pts [B,L,3], cam [B,3] -> [B,L,2]."""

    @staticmethod
    def forward(ctx, pts, cam):
        p, c = _lib.dev_f32(pts, "landmarks"), _lib.dev_f32(cam, "cam_params")
        B, n = p.shape[0], p.shape[1]
        xy = torch.empty(B, n, 2, dtype=torch.float32, device=p.device)
        _lib.call("smk_project_points", p.device, p, c, B, n, xy)
        ctx.dtypes = (pts.dtype, cam.dtype)
        ctx.save_for_backward(p, c)
        return xy

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_xy):
        p, c = ctx.saved_tensors
        B, n = p.shape[0], p.shape[1]
        g_pts, g_cam, g_xy = torch.empty_like(p), torch.empty_like(c), _grad_f32(g_xy)
        _lib.call("smk_project_points_backward", p.device, p, c, B, n, g_xy, g_pts, g_cam)
        return g_pts.to(ctx.dtypes[0]), g_cam.to(ctx.dtypes[1])
