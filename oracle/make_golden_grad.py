"""ORACLE — TEST INFRASTRUCTURE ONLY.  Generates tests/golden/grad.npz: torch autograd (CPU fp32) through the
REFERENCE's own FLAME and Renderer classes (via oracle/ref_harness.py) in the build container.
Re-run: ``python -m oracle.make_golden_grad``.

The harness's pytorch3d stub returns barycentrics without a gradient; here the reference renderer's
``rasterize_meshes`` is swapped for one that recomputes them in torch from the face vertices and the C
rasteriser's pix_to_face (oracle/grad_ref.py, asserted bitwise equal to the C rasteriser's), so autograd
yields pytorch3d's rasterize_meshes backward (blur 0, K = 1): that part is Tier B.  The tests regenerate the
parameters and upstream gradients from the seeds in ``flame_inputs`` / ``render_inputs``; stored are the
gradients and the renderer's input meshes and landmarks (the reference FLAME's outputs).
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from smirk_b200 import synth_assets, synth_inputs  # noqa: E402
from oracle import grad_ref, ref_harness, render_ref  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
N = lambda t: t.detach().cpu().numpy()
FLAME_OUTS = {"vertices": 5023, "landmarks_fan": 68, "landmarks_fan_3d": 68, "landmarks_mp": 105}


def flame_inputs():
    """B = 4, seeded parameters with eyelids and explicit zero neck / eye poses; seeded upstream gradients."""
    p = synth_inputs.flame_params(4, 111)
    p.pop("cam")
    p["neck_pose_params"], p["eye_pose_params"] = torch.zeros(4, 3), torch.zeros(4, 6)
    g = torch.Generator().manual_seed(112)
    return p, {k: torch.randn(4, n, 3, generator=g) for k, n in FLAME_OUTS.items()}


def render_inputs(vertices, landmarks, rc):
    """B = 2 meshes (the FLAME outputs of seed 211) + cam; seeded upstream gradients.  rendered_img's upstream is
    zeroed where a pixel's n.l lies within 1e-5 of a clamp boundary (see tests/test_gpu_grad.py)."""
    cam = synth_inputs.flame_params(2, 211)["cam"]
    with torch.no_grad():
        ndl = grad_ref.render_forward_grad_ref(rc, vertices, cam)["ndl"]
    keep = ~(((ndl.abs() < 1e-5) | ((ndl - 1).abs() < 1e-5)).any(1))
    g = torch.Generator().manual_seed(212)
    ups = {"rendered_img": torch.randn(2, 3, 224, 224, generator=g) * keep[:, None],
           "transformed_vertices": torch.randn(2, 5023, 3, generator=g),
           "landmarks_fan": torch.randn(2, 68, 2, generator=g), "landmarks_mp": torch.randn(2, 105, 2, generator=g)}
    x = {"vertices": vertices, "cam": cam, **landmarks}
    return x, ups


def _diff_rasterize(meshes, image_size=224, blur_radius=0.0, faces_per_pixel=1, bin_size=None,
                    max_faces_per_bin=None, perspective_correct=False, **kw):
    assert blur_radius == 0.0 and faces_per_pixel == 1 and not perspective_correct
    B, V = meshes.verts.shape[:2]
    Fm = meshes.faces.shape[1]
    fl = meshes.faces + (torch.arange(B) * V)[:, None, None]
    fv = meshes.verts.reshape(B * V, 3)[fl].reshape(-1, 3, 3)
    p2f, zbuf, bary_c, dists = render_ref.rasterize_ref(fv, B, Fm, image_size, image_size)
    bary = grad_ref.bary_from_p2f(fv, p2f[..., 0], image_size, image_size)
    assert torch.equal(bary.detach(), bary_c[:, :, :, 0]), "differentiable bary differs from the C rasteriser"
    return p2f, zbuf, bary[:, :, :, None, :], dists


def main():
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))
    out = {}
    with ref_harness.reference(root) as R:
        sys.modules["src.renderer.renderer"].rasterize_meshes = _diff_rasterize
        flame, rend = R.FLAME(), R.Renderer()
        # ---- FLAME ------------------------------------------------------------------------------
        p, ups = flame_inputs()
        leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
        fo = flame.forward(leaves)
        loss = sum((fo[k] * ups[k]).sum() for k in ups)
        for k, g in zip(leaves, torch.autograd.grad(loss, list(leaves.values()))):
            out["flame/" + k] = N(g)
        # ---- Renderer ---------------------------------------------------------------------------
        with torch.no_grad():
            fr = flame.forward(synth_inputs.flame_params(2, 211))
        x, ups = render_inputs(fr["vertices"], {k: fr[k] for k in ("landmarks_fan", "landmarks_mp")},
                               render_ref.RenderConstants(root))
        leaves = {k: v.clone().requires_grad_() for k, v in x.items()}
        ro = rend.forward(leaves["vertices"], leaves["cam"], landmarks_fan=leaves["landmarks_fan"],
                          landmarks_mp=leaves["landmarks_mp"])
        loss = sum((ro[k] * ups[k]).sum() for k in ups)
        for k, g in zip(leaves, torch.autograd.grad(loss, list(leaves.values()))):
            out["render/" + k] = N(g)
        for k in ("vertices", "landmarks_fan", "landmarks_mp"):
            out["render/input_" + k] = N(fr[k])
    np.savez_compressed(os.path.join(GOLD, "grad.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))
    print("grad.npz", os.path.getsize(os.path.join(GOLD, "grad.npz")))


if __name__ == "__main__":
    main()
