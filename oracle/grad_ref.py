"""ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Differentiable CPU fp32 restatements for the backward passes.  FLAME (``flame_ref.flame_forward_ref``)
is already plain torch, so autograd through it is the reference gradient (Tier A).  The renderer's
rasteriser is the C restatement in ``raster_ref.c``, which carries no gradient; here its barycentrics
are recomputed in torch from the face vertices and the C rasteriser's ``pix_to_face``, in the forward's
exact fp32 operation order (so they equal the C rasteriser's bitwise), and autograd through them is
pytorch3d's ``rasterize_meshes`` backward for blur 0, K = 1, no perspective correction (Tier B).
"""
import torch
import torch.nn.functional as F

from . import render_ref


def bary_from_p2f(face_verts, p2f, H=224, W=224):
    """face_verts [N*F,3,3] (NDC, differentiable), p2f i64 [N,H,W] -> bary [N,H,W,3] (-1 on background).

    Same arithmetic as the rasteriser: pixel centre xf = -1 + (2 i + 1) / S with i = S-1-x (pytorch3d's
    +X-left convention), w_k = edge_k(p) / (edge(v2; v0, v1) + 1e-8), edge(p; a, b) = (px-ax)(by-ay) - (py-ay)(bx-ax)."""
    N = p2f.shape[0]
    xi = torch.arange(W, dtype=torch.float32)
    yi = torch.arange(H, dtype=torch.float32)
    xf = (2.0 * (W - 1 - xi) + 1.0) / W + -1.0          # __fadd_rn(-1, __fdiv_rn(2 i + 1, S))
    yf = (2.0 * (H - 1 - yi) + 1.0) / H + -1.0
    px = xf[None, None, :].expand(N, H, W)
    py = yf[None, :, None].expand(N, H, W)
    cov = p2f >= 0
    fv = face_verts[p2f.clamp(min=0).reshape(-1)].reshape(N, H, W, 3, 3)
    x0, y0, x1, y1, x2, y2 = fv[..., 0, 0], fv[..., 0, 1], fv[..., 1, 0], fv[..., 1, 1], fv[..., 2, 0], fv[..., 2, 1]

    def edge(px_, py_, ax, ay, bx, by):
        return (px_ - ax) * (by - ay) - (py_ - ay) * (bx - ax)
    den = edge(x2, y2, x0, y0, x1, y1) + 1e-8
    w = torch.stack([edge(px, py, x1, y1, x2, y2) / den, edge(px, py, x2, y2, x0, y0) / den,
                     edge(px, py, x0, y0, x1, y1) / den], -1)
    return torch.where(cov[..., None], w, torch.full_like(w, -1.0))


def render_forward_grad_ref(rc, vertices, cam, **landmarks):
    """``render_ref.render_forward_ref`` with differentiable barycentrics: gradients reach ``vertices``,
    ``cam`` and the landmark sets through every path torch autograd takes in the reference."""
    B = vertices.shape[0]
    tv = render_ref.orth_proj_ref(vertices, cam)
    out = {k: render_ref.orth_proj_ref(v, cam)[..., :2] for k, v in landmarks.items()}
    tvm = tv[:, rc.final_mask, :].clone()
    vm = vertices[:, rc.final_mask, :]
    tvm[:, :, 2] = tvm[:, :, 2] + 10
    faces = rc.faces.expand(B, -1, -1)
    normals = render_ref.vertex_normals_ref(vm, faces)
    nv = vm.shape[1]
    fl = faces + (torch.arange(B) * nv)[:, None, None]
    face_normals = normals.reshape(B * nv, 3)[fl]
    fixed = tvm.clone()
    fixed[..., :2] = -fixed[..., :2]
    face_verts = fixed.reshape(B * nv, 3)[fl].reshape(-1, 3, 3)
    Fm, S = faces.shape[1], rc.image_size
    p2f, zbuf, bary_c, _ = render_ref.rasterize_ref(face_verts, B, Fm, S, S)
    p2f = p2f[..., 0]
    bary = bary_from_p2f(face_verts, p2f, S, S)
    attr = torch.cat([torch.full((B * Fm, 3, 3), 180.0 / 255.0), face_normals.reshape(B * Fm, 3, 3)], -1)
    mask = p2f == -1
    vals = attr[p2f.clamp(min=0).reshape(-1)].view(B, S, S, 3, 6)
    pix = (bary[..., None] * vals).sum(-2)
    pix = torch.where(mask[..., None], torch.zeros_like(pix), pix)
    pix = pix.permute(0, 3, 1, 2)
    albedo, nimg = pix[:, :3], pix[:, 3:6]
    nrm = nimg.permute(0, 2, 3, 1).reshape(B, -1, 3)
    ld = F.normalize(render_ref.LIGHT_DIRS[None, :, None, :].expand(B, -1, nrm.shape[1], -1), dim=3)
    ndl_raw = (nrm[:, None] * ld).sum(3)
    ndl = torch.clamp(ndl_raw, 0., 1.)
    shading = (ndl[..., None] * 1.7).expand(-1, -1, -1, 3).mean(1)
    shading = shading.reshape(B, S, S, 3).permute(0, 3, 1, 2)
    out.update(rendered_img=albedo * shading, transformed_vertices=tv, pix_to_face=p2f,
               bary=bary, bary_c=bary_c[:, :, :, 0], normals=normals,
               ndl=ndl_raw.detach().reshape(B, 5, S, S))
    return out
