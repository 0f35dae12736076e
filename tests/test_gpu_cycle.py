"""GPU suite of the trainer's masking (``TrainMaskingStage``) and the cycle augmentation (``CycleAugmentation``).

Bit-exactness: given the draws the device exports, both stages equal the CPU restatement of tests/cycle_ref.py bit for
bit (signed zeros included).  The only tolerance is on the integer pixel coordinates, which come from a truncated fp32
value (as in tests/test_gpu_masking.py): the masked images are compared with the device's own points fed in, and the
points against the restatement's within one pixel at a handful of points.
"""
import os

import numpy as np
import pytest
import torch

import cycle_ref
from smirk_b200 import synth_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "masking.npz")
KEYS = ("pose_params", "cam", "shape_params", "expression_params", "jaw_params", "eyelid_params")
DIMS = (3, 3, 300, 50, 3, 2)


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def faces(asset_root):
    from oracle import flame_ref
    return flame_ref.FlameConstants(asset_root).faces_tensor


def templates(seed=3):
    """Synthetic stand-in for load_templates(): five keys of different row counts, 100 fp64 columns."""
    rng = np.random.default_rng(seed)
    return {"subj%dtemplate%d" % (i, i): rng.standard_normal((n, 100)) for i, n in enumerate((1, 3, 4, 7, 9))}


def encoder_output(B, seed):
    gen = torch.Generator().manual_seed(seed)
    out = {k: torch.randn(B, d, generator=gen) for k, d in zip(KEYS, DIMS)}
    out["expression_params"][:, :3] *= 3.0                      # some values outside the [-4, 4] clamp
    out["expression_params"][0, 5] = -0.0                       # signed zeros must survive x * 0 as the reference's
    out["jaw_params"][:, 0] = out["jaw_params"][:, 0].abs() * 0.3
    out["eyelid_params"] = torch.rand(B, 2, generator=gen)
    return out


def bits(t):
    return t.contiguous().view(torch.int32)


def _aug(use_eyelids=True, seed=11):
    from smirk_b200.cycle import CycleAugmentation
    return CycleAugmentation(templates(), num_expression=50, use_eyelids=use_eyelids, seed=seed)


# ------------------------------------------------------------------------------------------------ augmentation
@pytest.mark.parametrize("use_eyelids", [True, False])
@pytest.mark.parametrize("Ke", [1, 2])
@pytest.mark.parametrize("B", [1, 2, 5, 32, 256])
def test_augment_bitwise_equals_restatement_given_the_draws(native_lib, B, Ke, use_eyelids):
    aug = _aug(use_eyelids)
    enc = encoder_output(B, 100 + B)
    feats, d = aug({k: v.to(DEV) for k, v in enc.items()}, Ke=Ke, debug=True)
    d = {k: v.cpu() for k, v in d.items()}
    R = Ke * B
    assert sorted(d["gids"].tolist()) == list(range(R))
    n1 = cycle_ref.group_bounds(R)[2] - cycle_ref.group_bounds(R)[1]
    assert sorted(d["perm1"].tolist()) == list(range(n1))
    ref = cycle_ref.augment_ref(enc, Ke, d, templates(), 50, use_eyelids)
    assert list(feats) == list(enc)
    for k in KEYS:
        assert feats[k].shape == (R, enc[k].shape[1])
        assert torch.equal(bits(feats[k].cpu()), bits(ref[k])), k


def test_augment_group_sizes_and_edge_batches(native_lib):
    """Groups split at R/4, 2R/4, 3R/4 (some empty for R < 4), counted on the kernel's own output: without use_eyelids
    the only rows whose jaw is all zero and whose eyelids differ from the input are the zero-expression group's, and
    they are the rows gids[3R/4:].  Pose / cam / shape are the rows r mod B."""
    aug = _aug(use_eyelids=False)
    for B, Ke in ((1, 1), (2, 1), (3, 1), (1, 2), (7, 2), (32, 1), (256, 2)):
        enc = encoder_output(B, 7)
        feats, d = aug({k: v.to(DEV) for k, v in enc.items()}, Ke=Ke, debug=True)
        feats = {k: v.cpu() for k, v in feats.items()}
        R = B * Ke
        c = cycle_ref.group_bounds(R)
        zero_jaw = (feats["jaw_params"] == 0).all(1)
        new_eyelids = (feats["eyelid_params"] != enc["eyelid_params"].repeat(Ke, 1)).any(1)
        assert torch.equal(zero_jaw, new_eyelids)
        assert int(zero_jaw.sum()) == R - c[3], (B, Ke)
        assert sorted(zero_jaw.nonzero().flatten().tolist()) == sorted(d["gids"].cpu()[c[3]:].tolist())
        for k in ("pose_params", "cam", "shape_params"):
            assert torch.equal(feats[k], enc[k].repeat(Ke, 1))


def test_augment_distributions(native_lib):
    """Over many calls: key and in-key row picks are uniform (chi-square), Bernoulli rates are 1/2, normals are N(0,1)
    and uniforms U(0,1) by their first two moments, and every permutation is a permutation."""
    from scipy import stats
    aug = _aug()
    tm = templates()
    enc = {k: v.to(DEV) for k, v in encoder_output(256, 5).items()}
    acc = {}
    for _ in range(40):
        _, d = aug(enc, Ke=2, debug=True)
        for k, v in d.items():
            acc.setdefault(k, []).append(v.cpu())
    cat = {k: torch.cat([x.reshape(-1) for x in v]) for k, v in acc.items()}
    keys = cat["tmpl_key"]
    n = len(keys)
    counts = torch.bincount(keys, minlength=len(tm)).double()
    assert stats.chisquare(counts.numpy()).pvalue > 1e-4
    rows = cat["tmpl_row"]
    for ki, name in enumerate(tm):
        r = rows[keys == ki]
        nr = tm[name].shape[0]
        assert int(r.max()) < nr and int(r.min()) >= 0
        if nr > 1:
            assert stats.chisquare(torch.bincount(r, minlength=nr).double().numpy()).pvalue > 1e-4
    assert n == 40 * 128
    for k in ("param_mask", "jaw_mask"):
        m = cat[k].double()
        assert set(m.unique().tolist()) <= {0.0, 1.0} and abs(float(m.mean()) - 0.5) < 4 * 0.5 / len(m) ** 0.5, k
    for k in ("randn0a", "randn0b", "randn1", "randn2", "randn3", "randn_jaw"):
        x = cat[k].double()
        assert abs(float(x.mean())) < 5 / len(x) ** 0.5 and abs(float(x.var()) - 1) < 10 * (2 / len(x)) ** 0.5, k
    for k in ("rand0a", "rand0b", "rand1a", "rand1b", "rand2a", "rand2b", "rand3", "rand_eyelid", "rand3_eyelid"):
        x = cat[k].double()
        assert float(x.min()) >= 0 and float(x.max()) < 1, k
        assert abs(float(x.mean()) - 0.5) < 5 * (1 / 12 / len(x)) ** 0.5 and abs(float(x.var()) - 1 / 12) < 0.01, k


def test_augment_group_permutation_is_uniform(native_lib):
    """randperm in distribution: over 640 calls at R = 32, the position of a fixed row and the row at a fixed position
    are uniform over the 32 values (chi-square), and the in-group permutation of group 1 likewise."""
    from scipy import stats
    aug = _aug(seed=21)
    enc = {k: v.to(DEV) for k, v in encoder_output(32, 6).items()}
    gids, perm1 = [], []
    for _ in range(640):
        _, d = aug(enc, debug=True)
        gids.append(d["gids"]); perm1.append(d["perm1"])
    gids, perm1 = torch.stack(gids).cpu(), torch.stack(perm1).cpu()
    pos_of_row0 = (gids == 0).nonzero()[:, 1]
    for sample, n in ((pos_of_row0, 32), (gids[:, 0], 32), (gids[:, 17], 32), (perm1[:, 0], 8)):
        assert stats.chisquare(torch.bincount(sample, minlength=n).double().numpy()).pvalue > 1e-4


def test_augment_counter(native_lib):
    """The same (seed, counter) gives the same bits; each call advances the counter; a captured graph replays fresh draws
    that equal eager calls at the same counters."""
    aug = _aug(seed=5)
    enc = {k: v.to(DEV) for k, v in encoder_output(32, 9).items()}
    a = aug(enc)
    b = aug(enc)
    assert not torch.equal(a["expression_params"], b["expression_params"])
    aug.reseed(5, 0)
    a2 = aug(enc)
    for k in KEYS:
        assert torch.equal(bits(a[k]), bits(a2[k]))
    aug.reseed(5, 10)
    eager = [aug(enc) for _ in range(3)]
    aug.reseed(5, 10)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        aug(enc)                                               # warm-up (counter 10)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = aug(enc)
    aug.reseed(5, 10)
    for e in eager:
        gr.replay()
        torch.cuda.synchronize()
        for k in KEYS:
            assert torch.equal(bits(out[k]), bits(e[k])), k


def test_augment_rejects_cpu_tensors(native_lib):
    aug = _aug()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        aug(encoder_output(2, 1))


# ------------------------------------------------------------------------------------------------ trainer masking
def _stage(g, faces, seed=4242):
    from smirk_b200.masking import TrainMaskingStage
    return TrainMaskingStage(faces, torch.from_numpy(g["base_prob"]), mask_ratio=0.01, mask_dilation_radius=10, seed=seed)


def _inputs(g, B, Ke, seed):
    """Meshes, images, hull masks and renders of B faces (Ke*B second-path meshes / renders).  The renders have pixels
    with one zero channel, where the two rendered-mask rules differ."""
    gen = torch.Generator().manual_seed(seed)
    tv0 = torch.from_numpy(g["trans_verts"])
    tv = tv0[torch.arange(B) % tv0.shape[0]] + 0.01 * torch.randn(B, tv0.shape[1], 3, generator=gen)
    tv2 = tv.repeat(Ke, 1, 1) + 0.02 * torch.randn(Ke * B, tv0.shape[1], 3, generator=gen)
    img = synth_inputs.images(B, seed)
    hull = torch.from_numpy(g["hull"]).float()[torch.arange(B) % 2]
    nz = torch.from_numpy(g["rendered_img_nonzero"]).float()
    R = Ke * B
    rend = synth_inputs.images(R, seed + 1) * nz[torch.arange(R) % 2]
    rend[:, 1, 100:110, 100:140] = 0.0                                  # one zero channel inside the face
    return tv, tv2, img, hull, rend


def _check_points(dev_pts, ref_pts):
    dd = (dev_pts - ref_pts).abs()
    assert int(dd.max()) <= 1 and int((dd > 0).sum()) <= max(6, dev_pts.numel() // 20000), int((dd > 0).sum())


@pytest.mark.parametrize("B", [1, 2, 5, 32, 256])
def test_first_path_bitwise_equals_restatement_given_the_draws(native_lib, g, faces, B):
    st = _stage(g, faces)
    tv, _, img, hull, rend = _inputs(g, B, 1, 20 + B)
    out, d = st.first_path(img.to(DEV), hull.to(DEV), tv.to(DEV), rend.to(DEV), debug=True)
    d = {k: v.cpu() for k, v in d.items()}
    N = int(0.01 * 224 * 224)
    assert d["sampled_faces_indices"].shape == (B, N) and "points2" not in d
    bc = d["barycentric_coords"]
    assert float(bc.min()) >= 0 and torch.allclose(bc.sum(-1), torch.ones(B, N), atol=1e-6)
    ref_pts = cycle_ref.masking_ref.points_from_coords_ref(tv, faces, d["sampled_faces_indices"], bc)[..., :2]
    _check_points(d["points1"], ref_pts)
    ref, _ = cycle_ref.first_path_ref(img, hull, tv, rend, faces, None, None, d["noise_mult"], d["random_centres"], points=d["points1"])
    assert torch.equal(bits(out.cpu()), bits(ref))
    assert abs(float(d["random_centres"].mean()) - 0.01) < 3e-3


@pytest.mark.parametrize("Ke", [1, 2])
@pytest.mark.parametrize("B", [1, 2, 5, 32, 256])
def test_second_path_bitwise_equals_restatement_given_the_draws(native_lib, g, faces, B, Ke):
    st = _stage(g, faces)
    tv, tv2, img, hull, rend = _inputs(g, B, Ke, 40 + B)
    out, d = st.second_path(img.to(DEV), hull.to(DEV), tv.to(DEV), tv2.to(DEV), rend.to(DEV), Ke=Ke, debug=True)
    d = {k: v.cpu() for k, v in d.items()}
    R = Ke * B
    assert out.shape == (R, 3, 224, 224) and d["points2"].shape[0] == R
    fidx, bc = d["sampled_faces_indices"], d["barycentric_coords"]
    _check_points(d["points1"], cycle_ref.masking_ref.points_from_coords_ref(tv, faces, fidx, bc)[..., :2])
    _check_points(d["points2"], cycle_ref.masking_ref.points_from_coords_ref(tv2, faces, fidx.repeat(Ke, 1), bc.repeat(Ke, 1, 1))[..., :2])
    ref, _, _ = cycle_ref.second_path_ref(img, hull, tv, tv2, rend, faces, fidx, bc, Ke, d["noise_mult"], d["random_centres"],
                                          points1=d["points1"], points2=d["points2"])
    assert torch.equal(bits(out.cpu()), bits(ref))
    assert abs(float(d["random_centres"].mean()) - 0.005) < 3e-3


def test_second_path_rendered_mask_rule(native_lib, g, faces):
    """A render pixel with one zero channel is foreground for step1 (1 - all(rendered == 0)) and background for step2
    (all(rendered > 0)).  With a full hull the masked image is img * (1 - rendered_mask) wherever no point was retained."""
    st = _stage(g, faces)
    tv, tv2, img, _, _ = _inputs(g, 1, 1, 3)
    hull = torch.ones(1, 1, 224, 224)
    rend = torch.ones(1, 3, 224, 224)
    rend[:, 2, 0:30, 0:30] = 0.0                                        # one zero channel
    rend[:, :, 0:30, 194:224] = 0.0                                     # every channel zero
    rend[:, 0, 194:224, 0:30] = -1.0                                    # a negative channel
    o1, d1 = st.first_path(img.to(DEV), hull.to(DEV), tv.to(DEV), rend.to(DEV), debug=True)
    o2, d2 = st.second_path(img.to(DEV), hull.to(DEV), tv.to(DEV), tv2.to(DEV), rend.to(DEV), debug=True)
    o1, o2 = o1.cpu(), o2.cpu()
    free1 = (cycle_ref.transfer_pixels_ref(img, d1["points1"].cpu(), d1["points1"].cpu()) == 0).all(1, keepdim=True)
    free2 = (cycle_ref.transfer_pixels_ref(img, d2["points1"].cpu(), d2["points2"].cpu()) == 0).all(1, keepdim=True)
    for ys, xs, fg1, fg2 in ((slice(0, 30), slice(0, 30), True, False), (slice(0, 30), slice(194, 224), False, False),
                             (slice(194, 224), slice(0, 30), True, False), (slice(100, 130), slice(100, 130), True, True)):
        for o, free, fg in ((o1, free1, fg1), (o2, free2, fg2)):
            want = torch.zeros_like(img) if fg else img
            sel = free[:, :, ys, xs].expand(-1, 3, -1, -1)
            assert int(sel.sum()) > 0
            assert torch.equal(o[:, :, ys, xs][sel], want[:, :, ys, xs][sel])
    ref2, _, _ = cycle_ref.second_path_ref(img, hull, tv, tv2, rend, faces, None, None, 1, d2["noise_mult"].cpu(), d2["random_centres"].cpu(),
                                           points1=d2["points1"].cpu(), points2=d2["points2"].cpu())
    assert torch.equal(o2, ref2)


def test_train_masking_face_frequencies_follow_the_weights(native_lib, g, faces):
    """multinomial(weights, N, replacement=True) in distribution, as for the demo's MaskingStage."""
    from smirk_b200 import masking
    st = _stage(g, faces)
    tv, _, img, hull, rend = _inputs(g, 1, 1, 8)
    counts = torch.zeros(faces.shape[0], dtype=torch.float64)
    for _ in range(150):
        _, d = st.first_path(img.to(DEV), hull.to(DEV), tv.to(DEV), rend.to(DEV), debug=True)
        counts += torch.bincount(d["sampled_faces_indices"].cpu()[0], minlength=faces.shape[0]).double()
    n = float(counts.sum())
    w = masking.face_weights(tv.to(DEV), faces, torch.from_numpy(g["base_prob"])).cpu()[0].double()
    p = w / w.sum()
    assert float(counts[p == 0].sum()) == 0
    z = (counts / n - p) / torch.sqrt(p * (1 - p) / n + 1e-30)
    big = p * n >= 20
    assert int(big.sum()) > 300 and float(z[big].abs().max()) < 6.0, "max |z| %.2f" % float(z[big].abs().max())


def test_train_masking_counter_and_graph(native_lib, g, faces):
    """Same (seed, counter) -> same bits; each call advances the counter; both paths captured in one CUDA graph replay
    bitwise equal to eager calls at the same counters."""
    st = _stage(g, faces, seed=77)
    B, Ke = 4, 2
    tv, tv2, img, hull, rend = (t.to(DEV) for t in _inputs(g, B, Ke, 12))
    rend1 = rend[:B].contiguous()
    a1 = st.first_path(img, hull, tv, rend1)
    a2 = st.second_path(img, hull, tv, tv2, rend, Ke=Ke)
    b1 = st.first_path(img, hull, tv, rend1)
    assert not torch.equal(a1, b1)
    st.reseed(77, 0)
    assert torch.equal(st.first_path(img, hull, tv, rend1), a1)
    assert torch.equal(st.second_path(img, hull, tv, tv2, rend, Ke=Ke), a2)
    st.reseed(77, 50)
    eager = [(st.first_path(img, hull, tv, rend1), st.second_path(img, hull, tv, tv2, rend, Ke=Ke)) for _ in range(2)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        st.first_path(img, hull, tv, rend1); st.second_path(img, hull, tv, tv2, rend, Ke=Ke)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        o1 = st.first_path(img, hull, tv, rend1)
        o2 = st.second_path(img, hull, tv, tv2, rend, Ke=Ke)
    st.reseed(77, 50)
    for e1, e2 in eager:
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(o1, e1) and torch.equal(o2, e2)


def test_train_masking_rejects_bad_inputs(native_lib, g, faces):
    st = _stage(g, faces)
    tv, tv2, img, hull, rend = _inputs(g, 2, 1, 1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        st.first_path(img, hull, tv, rend)
    with pytest.raises(RuntimeError, match="transformed_vertices_2nd"):
        st.second_path(img.to(DEV), hull.to(DEV), tv.to(DEV), tv2[:1].to(DEV), rend.to(DEV))
