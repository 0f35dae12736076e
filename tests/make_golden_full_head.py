"""Generates tests/golden/render_full_head.npz: the REFERENCE's own ``Renderer(render_full_head=True)`` (through
oracle/ref_harness.py, so it needs the reference checkout) at B = 2, forward outputs and torch autograd (CPU fp32).
Re-run: ``python tests/make_golden_full_head.py``.

As in oracle/make_golden_grad.py, the reference renderer's ``rasterize_meshes`` is swapped for one that recomputes
the barycentrics in torch from the face vertices and the C rasteriser's pix_to_face (asserted bitwise equal to the C
rasteriser's), so autograd yields pytorch3d's rasterize_meshes backward (blur 0, K = 1).

The inputs are those of grad.npz's renderer case: the meshes and landmarks stored there as ``render/input_*`` (the
reference FLAME's outputs for seed 211), ``cam`` from seed 211, and the upstream gradients of
``make_golden_grad.render_inputs`` with the clamp-boundary mask of the full head.  Stored: every output of the
forward (the image, pix_to_face and zbuf subsampled 2x in x and y, one channel of the grey image; the z of
transformed_vertices, which carries the offset) and the gradients for vertices, cam and both landmark sets.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from smirk_b200 import synth_assets  # noqa: E402
from oracle import make_golden_grad as mg, ref_harness  # noqa: E402
import render_full_head_ref as fh  # noqa: E402

GOLD = os.path.join(HERE, "golden")
N = lambda t: t.detach().cpu().numpy()
SUB = (slice(None), slice(None, None, 2), slice(None, None, 2))         # [B, ::2, ::2]


def inputs(grad_npz, rc):
    """(x, ups) of grad.npz's renderer case, with the full head's clamp-boundary mask on rendered_img's upstream."""
    T = torch.from_numpy
    return mg.render_inputs(T(grad_npz["render/input_vertices"]),
                            {k: T(grad_npz["render/input_" + k]) for k in ("landmarks_fan", "landmarks_mp")}, rc)


def main():
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))
    g = np.load(os.path.join(GOLD, "grad.npz"))
    x, ups = inputs(g, fh.FullHeadConstants(root))
    out = {}
    with ref_harness.reference(root) as R:
        sys.modules["src.renderer.renderer"].rasterize_meshes = mg._diff_rasterize
        rend = R.Renderer(render_full_head=True)
        assert rend.faces.shape == (1, fh.N_FACES, 3)
        leaves = {k: v.clone().requires_grad_() for k, v in x.items()}
        ro = rend.forward(leaves["vertices"], leaves["cam"], landmarks_fan=leaves["landmarks_fan"],
                          landmarks_mp=leaves["landmarks_mp"])
        loss = sum((ro[k] * ups[k]).sum() for k in ups)
        for k, gr in zip(leaves, torch.autograd.grad(loss, list(leaves.values()))):
            out["grad/" + k] = N(gr)
        out["rendered_img"] = N(ro["rendered_img"][:, 0][SUB])
        out["transformed_vertices_z"] = N(ro["transformed_vertices"][:, :, 2])      # x, y as with the face mask
        for k in ("landmarks_fan", "landmarks_mp"):
            out[k] = N(ro[k])
        with torch.no_grad():                       # the raw rasteriser outputs, from the reference's own call
            tv = ro["transformed_vertices"].detach().clone()
            fixed = tv.clone()
            fixed[..., :2] = -fixed[..., :2]        # renderer.py:172-173 (the +10 is already in tv)
            p2f, zbuf, bary, _ = mg._diff_rasterize(types.SimpleNamespace(verts=fixed, faces=rend.faces.expand(2, -1, -1)))
        out["pix_to_face"] = p2f[..., 0][SUB].numpy().astype(np.int32)
        out["zbuf"] = zbuf[..., 0][SUB].numpy()
    path = os.path.join(GOLD, "render_full_head.npz")
    np.savez_compressed(path, **out)
    for k, v in out.items():
        print(k, v.shape, v.dtype, float(np.abs(v).max()))
    print("render_full_head.npz", os.path.getsize(path))


if __name__ == "__main__":
    main()
