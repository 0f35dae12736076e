"""CPU suite for the backward passes: the differentiable oracle's barycentrics equal the C rasteriser's
bitwise, and the backward entry points reject bad arguments with a negative return and a message
(checked before any device work, so no GPU is needed)."""
import ctypes as C

import torch

from smirk_b200 import synth_inputs


def test_differentiable_bary_equals_c_raster(asset_root):
    from oracle import flame_ref, grad_ref, render_ref
    c, rc = flame_ref.FlameConstants(asset_root), render_ref.RenderConstants(asset_root)
    p = synth_inputs.flame_params(3, 8000)
    with torch.no_grad():
        o = grad_ref.render_forward_grad_ref(rc, flame_ref.flame_forward_ref(c, p)["vertices"], p["cam"])
        ref = render_ref.render_forward_ref(rc, flame_ref.flame_forward_ref(c, p)["vertices"], p["cam"])
    assert (o["pix_to_face"] >= 0).float().mean() > 0.1
    assert torch.equal(o["bary"], o["bary_c"]) and torch.equal(o["bary"], ref["bary"])
    assert torch.equal(o["rendered_img"], ref["rendered_img"])


def test_differentiable_oracle_reaches_every_input(asset_root):
    from oracle import flame_ref, grad_ref, render_ref
    c, rc = flame_ref.FlameConstants(asset_root), render_ref.RenderConstants(asset_root)
    p = synth_inputs.flame_params(1, 8001)
    v = flame_ref.flame_forward_ref(c, p)["vertices"].detach().requires_grad_()
    cam = p["cam"].clone().requires_grad_()
    o = grad_ref.render_forward_grad_ref(rc, v, cam)
    gv, gc = torch.autograd.grad(o["rendered_img"].sum(), [v, cam])
    mask = torch.zeros(5023, dtype=torch.bool)
    mask[rc.final_mask] = True
    assert gv[0, mask].abs().sum() > 0 and gv[0, ~mask].abs().sum() == 0 and gc.abs().sum() > 0


def test_backward_entry_points_reject_bad_arguments(native_lib):
    L = native_lib
    vp = C.c_void_p
    fake, buf = vp(16), vp(16)                       # never dereferenced: the checks fail first
    nul = vp(0)
    rc = L.smk_flame_backward(nul, buf, buf, nul, 2, buf, nul, nul, nul, nul, buf, buf, nul, buf, 1 << 20, nul)
    assert rc < 0 and b"smk_flame_backward: null argument" in L.smk_last_error()
    rc = L.smk_flame_backward(fake, buf, buf, nul, 2, nul, nul, nul, nul, nul, buf, buf, nul, buf, 1 << 20, nul)
    assert rc < 0 and b"null argument" in L.smk_last_error()           # dyn_idx is required
    rc = L.smk_flame_backward(fake, buf, buf, nul, 2, buf, nul, nul, nul, nul, buf, buf, nul, nul, 0, nul)
    assert rc < 0 and b"workspace too small" in L.smk_last_error()
    rc = L.smk_flame_backward(fake, buf, buf, nul, -1, buf, nul, nul, nul, nul, buf, buf, nul, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_renderer_backward(nul, buf, buf, 2, buf, buf, buf, nul, nul, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"smk_renderer_backward: null argument" in L.smk_last_error()
    rc = L.smk_renderer_backward(fake, buf, buf, 2, nul, buf, buf, nul, nul, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"null argument" in L.smk_last_error()           # pix_to_face is required
    rc = L.smk_renderer_backward(fake, buf, buf, 2, buf, buf, buf, nul, nul, buf, buf, nul, 0, nul)
    assert rc < 0 and b"workspace too small" in L.smk_last_error()
    rc = L.smk_project_points_backward(buf, buf, 2, 68, nul, buf, buf, nul)
    assert rc < 0 and b"smk_project_points_backward: null argument" in L.smk_last_error()
    rc = L.smk_project_points_backward(buf, buf, -1, 68, buf, buf, buf, nul)
    assert rc < 0 and b"negative size" in L.smk_last_error()
    # an empty batch is a no-op in every backward entry point, whatever the pointers
    assert L.smk_project_points_backward(nul, nul, 0, 68, nul, nul, nul, nul) == 0
    assert L.smk_flame_backward(nul, nul, nul, nul, 0, nul, nul, nul, nul, nul, nul, nul, nul, nul, 0, nul) == 0
    assert L.smk_renderer_backward(nul, nul, nul, 0, nul, nul, nul, nul, nul, nul, nul, nul, 0, nul) == 0
    assert L.smk_flame_backward_workspace_bytes(nul, 4) == 0 and L.smk_renderer_backward_workspace_bytes(nul, 4) == 0


def test_oracle_autograd_reproduces_golden_grad(asset_root, golden):
    """The restatements' autograd (oracle/flame_ref.py, oracle/grad_ref.py) against the reference classes' own
    autograd (tests/golden/grad.npz, oracle/make_golden_grad.py): max-abs error <= 1e-6 x max-abs, per tensor."""
    import numpy as np
    from oracle import flame_ref, grad_ref, make_golden_grad as mg, render_ref
    g = golden("grad")

    def close(a, b):
        a, b = a.detach().double().numpy(), np.asarray(b, np.float64)
        assert a.shape == b.shape and np.abs(a - b).max() <= 1e-6 * np.abs(b).max(), (np.abs(a - b).max(), np.abs(b).max())
    c = flame_ref.FlameConstants(asset_root)
    p, ups = mg.flame_inputs()
    leaves = {k: v.clone().requires_grad_() for k, v in p.items()}
    fo = flame_ref.flame_forward_ref(c, leaves)
    for k, gr in zip(leaves, torch.autograd.grad(sum((fo[k] * ups[k]).sum() for k in ups), list(leaves.values()))):
        close(gr, g["flame/" + k])
    rc = render_ref.RenderConstants(asset_root)
    T = torch.from_numpy
    x, ups = mg.render_inputs(T(g["render/input_vertices"]), {k: T(g["render/input_" + k]) for k in ("landmarks_fan", "landmarks_mp")}, rc)
    leaves = {k: v.clone().requires_grad_() for k, v in x.items()}
    ro = grad_ref.render_forward_grad_ref(rc, leaves["vertices"], leaves["cam"], landmarks_fan=leaves["landmarks_fan"],
                                          landmarks_mp=leaves["landmarks_mp"])
    for k, gr in zip(leaves, torch.autograd.grad(sum((ro[k] * ups[k]).sum() for k in ups), list(leaves.values()))):
        close(gr, g["render/" + k])
