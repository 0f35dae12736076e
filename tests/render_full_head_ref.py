"""CPU restatement of ``Renderer(render_full_head=True).forward`` (src/renderer/renderer.py:50-74,100-207): the
face-mask restatement of ``oracle/render_ref.py`` and ``oracle/grad_ref.py`` on the whole FLAME topology (5023
vertices, 9976 triangles, no subset and no renumbering), plus the leaked depth offset.

With the full head ``render()`` skips the fancy-index (renderer.py:140-142), so its ``transformed_vertices[:, :, 2] =
transformed_vertices[:, :, 2] + 10`` writes into the tensor ``forward`` returns: the reference's
``transformed_vertices`` carry z + 10 (fp32).  x and y are untouched, and the offset is a constant, so the gradient
through ``transformed_vertices`` is unchanged.
"""
import os

import torch

from oracle import grad_ref, render_ref

Z_OFFSET = 10.0
N_VERTS, N_FACES = 5023, 9976


class FullHeadConstants:
    """renderer.py:50-74 with render_full_head=True: every vertex, every face of head_template.obj."""

    def __init__(self, root="."):
        _, faces, _, _ = render_ref.parse_obj(os.path.join(root, "assets", "head_template.obj"))
        n = int(faces.max()) + 1
        self.final_mask = list(range(n))
        self.faces = faces[None]                                       # [1,9976,3]
        self.image_size = 224


def _leak_offset(out):
    tv = out["transformed_vertices"].clone()
    tv[:, :, 2] = tv[:, :, 2] + Z_OFFSET                             # renderer.py:144 on the returned tensor
    out["transformed_vertices"] = tv
    return out


def render_forward_ref(rc, vertices, cam, brute=False, **landmarks):
    """``render_ref.render_forward_ref`` on the full head, with the offset on transformed_vertices."""
    return _leak_offset(render_ref.render_forward_ref(rc, vertices, cam, brute=brute, **landmarks))


def render_forward_grad_ref(rc, vertices, cam, **landmarks):
    """``grad_ref.render_forward_grad_ref`` on the full head (differentiable barycentrics), with the offset."""
    return _leak_offset(grad_ref.render_forward_grad_ref(rc, vertices, cam, **landmarks))


def clamp_keep(rc, vertices, cam):
    """[B,S,S] bool: pixels whose n.l lies at least 1e-5 from both clamp boundaries for every light (the clamp-boundary
    rule of tests/test_gpu_grad.py; the other pixels get a zero upstream gradient)."""
    with torch.no_grad():
        ndl = grad_ref.render_forward_grad_ref(rc, vertices, cam)["ndl"]
    return ~(((ndl.abs() < 1e-5) | ((ndl - 1).abs() < 1e-5)).any(1))
