"""GPU parity of the masking kernels (SURVEY.md §8f #1) against the reference-pinned golden fixture.

Tolerances: the face weights go through vertex normals (1e-5 relative, and the `mean z < 0.05` threshold may flip for
faces within 1e-5 of it); the integer pixel coordinates come from a truncated fp32 value (a point may differ by one
pixel only where that value is within 1e-4 of an integer); the composite is exact given the same inputs.
"""
import os

import numpy as np
import pytest
import torch

from smirk_b200 import synth_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "masking.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def faces(asset_root):
    from oracle import flame_ref
    return flame_ref.FlameConstants(asset_root).faces_tensor


def T(a, dt=None):
    t = torch.from_numpy(np.asarray(a))
    return t.to(dt) if dt is not None else t


def test_face_weights(native_lib, g, faces):
    from smirk_b200 import masking
    w = masking.face_weights(T(g["trans_verts"]).to(DEV), faces, T(g["base_prob"])).cpu()
    ref = T(g["face_weights"])
    flipped = (w == 0) != (ref == 0)
    assert int(flipped.sum()) <= 3, "threshold flips: %d" % int(flipped.sum())
    ok = ~flipped
    assert torch.allclose(w[ok], ref[ok], rtol=1e-4, atol=1e-9)


def test_points_from_coords(native_lib, g, faces):
    from smirk_b200 import masking
    coords = {"sampled_faces_indices": T(g["sampled_faces_indices"], torch.long), "barycentric_coords": T(g["barycentric_coords"])}
    pts, _ = masking.mesh_based_mask_uniform_faces(T(g["trans_verts"]).to(DEV), faces, T(g["base_prob"]), mask_ratio=0.05, coords=coords)
    ref = T(g["npoints"], torch.long)[..., :2]                       # (x, y); the reference also truncates a z column nobody reads
    d = (pts.cpu() - ref).abs()
    assert int(d.max()) <= 1 and int((d > 0).sum()) <= 4, "pixel mismatches: %d" % int((d > 0).sum())


def test_compose_matches_reference(native_lib, g, faces):
    from oracle import masking_ref
    from smirk_b200 import masking
    npoints, rbound = T(g["npoints"], torch.long), T(g["rbound"])
    img = synth_inputs.images(npoints.shape[0], int(g["seeds"][2]))
    hull, rmask = T(g["hull"], torch.float32), T(g["rendered_img_nonzero"], torch.float32)
    out = masking.masking_from_points(img.to(DEV), hull, npoints, rbound, wr=10, flame_faces=faces).cpu()
    assert torch.equal(out[:, :, ::2, 1::2], T(g["masked_plain_sub"]))
    gen = torch.Generator().manual_seed(5)
    noise = torch.randn(img.shape, generator=gen) * 0.05 + 1
    centres = torch.bernoulli(torch.ones(img.shape[0], 1, 224, 224) * 0.01, generator=gen)
    out = masking.masking_from_points(img.to(DEV), hull, npoints, rbound, wr=10, rendered_mask=rmask, noise_mult=noise,
                                      random_centres=centres, flame_faces=faces).cpu()
    ref = masking_ref.masking_ref(img, hull, img * masking_ref.point_mask_ref(npoints, rbound, 224), 10, rendered_mask=rmask,
                                  noise_mult=noise, random_centres=centres)
    assert torch.equal(out, ref)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_free_functions_launch_on_the_tensors_device(native_lib, g, faces):
    """face_weights, mesh_based_mask_uniform_faces and masking_from_points run on their tensors' device, not the current
    one: on cuda:1 tensors while cuda:0 is current they return what the same calls return on cuda:0."""
    from smirk_b200 import masking
    tv, bp = T(g["trans_verts"]), T(g["base_prob"])
    coords = {"sampled_faces_indices": T(g["sampled_faces_indices"], torch.long), "barycentric_coords": T(g["barycentric_coords"])}
    npoints, rbound = T(g["npoints"], torch.long), T(g["rbound"])
    img, hull = synth_inputs.images(npoints.shape[0], int(g["seeds"][2])), T(g["hull"], torch.float32)

    def run(dev):
        w = masking.face_weights(tv.to(dev), faces, bp)
        pts, _ = masking.mesh_based_mask_uniform_faces(tv.to(dev), faces, bp, mask_ratio=0.05, coords=coords)
        out = masking.masking_from_points(img.to(dev), hull, npoints, rbound, wr=10, flame_faces=faces)
        return [t.cpu() for t in (w, pts, out)]

    with torch.cuda.device(0):
        on0, on1 = run("cuda:0"), run("cuda:1")
    for a, b in zip(on0, on1):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------ MaskingStage: draws made on the device
def _stage(g, faces, **kw):
    from smirk_b200 import masking
    return masking.MaskingStage(faces, T(g["base_prob"]), n_verts=5023, seed=4242, **kw)


def test_masking_stage_equals_reference_given_its_own_draws(native_lib, g, faces):
    """The device makes the random draws (Philox); exporting them and feeding them to the restated reference functions
    (pinned bit-exactly to src/utils/masking.py by tests/test_masking_oracle.py) must reproduce the masked image."""
    from oracle import masking_ref
    st = _stage(g, faces)
    tv = T(g["trans_verts"])
    B = tv.shape[0]
    img = synth_inputs.images(B, int(g["seeds"][2]))
    hull = T(g["hull"], torch.float32)
    rendered = synth_inputs.images(B, 99) * T(g["rendered_img_nonzero"], torch.float32)      # zero exactly where the mesh is absent
    out, d = st.forward(img.to(DEV), hull.to(DEV), tv.to(DEV), rendered.to(DEV), debug=True)
    d = {k: v.cpu() for k, v in d.items()}
    N = int(0.01 * 5 * 224 * 224)
    assert d["sampled_faces_indices"].shape == (B, N) and int(d["sampled_faces_indices"].min()) >= 0
    w = masking_ref.face_probabilities_ref(tv, faces, T(g["base_prob"]))
    assert bool((w.gather(1, d["sampled_faces_indices"]) > 0).all()), "a zero-weight face was sampled"
    bc = d["barycentric_coords"]
    assert float(bc.min()) >= 0 and torch.allclose(bc.sum(-1), torch.ones(B, N), atol=1e-6)
    assert bool((d["rbound"] >= N // 25).all()) and bool((d["rbound"] <= N).all())
    pts = masking_ref.points_from_coords_ref(tv, faces, d["sampled_faces_indices"], bc)
    dd = (pts[..., :2] - d["npoints"]).abs()
    assert int(dd.max()) <= 1 and int((dd > 0).sum()) <= 6
    rmask = T(g["rendered_img_nonzero"], torch.float32)
    ref = masking_ref.masking_ref(img, hull, img * masking_ref.point_mask_ref(d["npoints"], d["rbound"], 224), 10, rendered_mask=rmask,
                                  noise_mult=d["noise_mult"], random_centres=d["random_centres"])
    assert torch.equal(out.cpu(), ref)
    # moments of the two per-pixel draws (masking.py:84-92): N(1, 0.05^2) and Bernoulli(0.01)
    assert abs(float(d["noise_mult"].mean()) - 1) < 1e-3 and abs(float(d["noise_mult"].std()) - 0.05) < 1e-3
    assert abs(float(d["random_centres"].mean()) - 0.01) < 2e-3


def test_masking_stage_sampling_follows_the_face_weights(native_lib, g, faces):
    """multinomial(weights, N, replacement=True) in distribution: empirical face frequencies over many calls against
    weights / sum(weights); deterministic for a given (seed, counter), fresh on every call."""
    from oracle import masking_ref
    st = _stage(g, faces)
    tv = T(g["trans_verts"])[:1]
    img = synth_inputs.images(1, 5).to(DEV)
    hull, rend = torch.ones(1, 1, 224, 224, device=DEV), torch.zeros(1, 3, 224, 224, device=DEV)
    counts = torch.zeros(faces.shape[0], dtype=torch.float64)
    first = None
    calls = 60
    for c in range(calls):
        out, d = st.forward(img, hull, tv.to(DEV), rend, debug=True)
        idx = d["sampled_faces_indices"].cpu()[0]
        counts += torch.bincount(idx, minlength=faces.shape[0]).double()
        if c == 0:
            first = (out.clone(), idx.clone())
        if c == 1:
            assert not torch.equal(idx, first[1]), "the call counter did not advance"
    n = float(counts.sum())
    # the device's own weights (pinned to the reference's by test_face_weights up to threshold flips of faces whose mean
    # normal z sits within 1e-5 of 0.05)
    from smirk_b200 import masking
    w = masking.face_weights(tv.to(DEV), faces, T(g["base_prob"])).cpu()[0].double()
    p = w / w.sum()
    assert float(counts[p == 0].sum()) == 0
    z = (counts / n - p) / torch.sqrt(p * (1 - p) / n + 1e-30)
    big = p * n >= 20
    assert int(big.sum()) > 500 and float(z[big].abs().max()) < 6.0, "max |z| %.2f" % float(z[big].abs().max())
    st.reseed(4242, 0)
    out2, d2 = st.forward(img, hull, tv.to(DEV), rend, debug=True)
    assert torch.equal(out2, first[0]) and torch.equal(d2["sampled_faces_indices"].cpu()[0], first[1])


# ------------------------------------------------------------------------------ transfer_pixels / masking() with the reference's signatures
def test_transfer_pixels_matches_reference(native_lib, g, faces):
    """masking.py:116-129 incl. duplicate targets (last pair in index order wins) and the rbound variant, against the
    outputs of the reference's own function stored in the golden file."""
    from smirk_b200 import masking
    img = synth_inputs.images(2, int(g["seeds"][2])).to(DEV)
    p1, p2 = T(g["p1"], torch.long), T(g["p2"], torch.long)
    assert torch.equal(masking.transfer_pixels(img, p1, p2).cpu(), T(g["transfer"]))
    assert torch.equal(masking.transfer_pixels(img, p1, p2, rbound=torch.tensor([100, 400])).cpu(), T(g["transfer_rbound"]))


def test_masking_reference_signature(native_lib, g, faces):
    """masking(img, mask, extra_points, wr, rendered_mask, extra_noise, random_mask) (masking.py:71-102): deterministic
    setting against the reference's own output; with the random draws on, structural checks."""
    from oracle import masking_ref
    from smirk_b200 import masking
    npoints, rbound = T(g["npoints"], torch.long), T(g["rbound"])
    img = synth_inputs.images(npoints.shape[0], int(g["seeds"][2]))
    hull = T(g["hull"], torch.float32)
    extra = img * masking_ref.point_mask_ref(npoints, rbound, 224)
    out = masking.masking(img.to(DEV), hull, extra, 10, rendered_mask=None, extra_noise=False, random_mask=0, flame_faces=faces).cpu()
    assert torch.equal(out[:, :, ::2, 1::2], T(g["masked_plain_sub"]))
    torch.manual_seed(3)
    rmask = T(g["rendered_img_nonzero"], torch.float32)
    noisy = masking.masking(img.to(DEV), hull, extra, 10, rendered_mask=rmask, flame_faces=faces).cpu()
    base = masking_ref.masking_ref(img, hull, extra, 10, rendered_mask=rmask)
    sel = extra > 0
    assert torch.equal(noisy[~sel], base[~sel])                         # only retained points see the draws
    knocked = noisy[sel] == base[sel]                                   # a knocked-out point falls back to img * mask
    assert 0.05 < float(knocked.float().mean()) < 0.95                  # 1 % centres x 11x11 patches cover ~70 % of the image; sampled points cluster
    kept = (noisy[sel] > 0) & ~knocked                                  # retained points that carry img * noise
    assert float(kept.float().mean()) > 0.1
    ratio = noisy[sel][kept] / extra[sel][kept]
    assert abs(float(ratio.mean()) - 1) < 0.01 and abs(float(ratio.std()) - 0.05) < 0.01
