"""CPU suite of the trainer's masking and cycle augmentation: the restatement of tests/cycle_ref.py against the reference
trainer's own step1 / step2 (live where the reference checkout is importable, and against tests/golden/cycle.npz) and the
argument checks of its entry points."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import cycle_ref
import make_golden_cycle as mgc

N_POINTS = int(0.01 * 224 * 224)


def restated_steps(asset_root, B, Ke, seed):
    """The restatement with its draws made from torch's and Python's generators in the reference's order, seeded as
    make_golden_cycle seeds the reference's step1 / step2 -> (masked_1st_path, flame_feats, masked_img_2nd_path)."""
    from oracle import flame_ref
    x = mgc.case_inputs(B, Ke, seed)
    faces = flame_ref.FlameConstants(asset_root).faces_tensor
    torch.manual_seed(seed); random.seed(seed)
    fidx, bary = cycle_ref.sample_draws_ref(x["tv"], faces, x["base_prob"], N_POINTS)
    noise, centres = cycle_ref.noise_draws_ref(B, 224, 0.01)
    m1, _ = cycle_ref.first_path_ref(x["img"], x["hull"], x["tv"], x["rend"], faces, fidx, bary, noise, centres)
    torch.manual_seed(seed + 1); random.seed(seed + 1)
    tm = mgc.synthetic_templates()
    d = cycle_ref.augment_draws_ref(Ke * B, 50, 2, tm)
    feats = cycle_ref.augment_ref(x["enc"], Ke, d, tm)
    fidx, bary = cycle_ref.sample_draws_ref(x["tv"], faces, x["base_prob"], N_POINTS)
    noise, centres = cycle_ref.noise_draws_ref(Ke * B, 224, 0.005)
    m2, p1, p2 = cycle_ref.second_path_ref(x["img"], x["hull"], x["tv"], x["tv2"], x["rend2"], faces, fidx, bary, Ke, noise, centres)
    return m1, feats, m2, cycle_ref.conflicting_targets(p1.repeat(Ke, 1, 1), p2)


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("B,Ke,seed", mgc.CASES)
def test_restatement_reproduces_the_reference_steps_golden(asset_root, golden, B, Ke, seed):
    g = golden("cycle")
    p = "B%d" % B
    assert list(g[p + "/seed"]) == [seed, seed + 1]
    m1, feats, m2, conflicts = restated_steps(asset_root, B, Ke, seed)
    assert int(conflicts.sum()) == int(g[p + "/conflicts"])
    m2 = m2.masked_fill(conflicts, 0.0)                     # the pixels where torch's index_put order decides
    assert list(feats) == list(mgc.KEYS)
    for k, v in feats.items():
        assert torch.equal(bits(v), bits(torch.from_numpy(g[p + "/flame_feats/" + k]))), k
    for name, t in (("masked_1st_path", m1), ("masked_img_2nd_path", m2)):
        assert torch.equal(t[:, :, ::mgc.SUB, ::mgc.SUB], torch.from_numpy(g[p + "/" + name + "/sub"])), name
        assert mgc.digest(t) == str(g[p + "/" + name + "/sha256"]), name


@pytest.mark.parametrize("B,Ke,seed", mgc.CASES)
def test_restatement_reproduces_the_live_reference_steps(asset_root, B, Ke, seed):
    from oracle import ref_harness
    if not ref_harness.available():
        pytest.skip("reference checkout not available; the golden test covers this")
    r1, rfeats, r2, rconf = mgc.run_reference(asset_root, B, Ke, seed)
    m1, feats, m2, conflicts = restated_steps(asset_root, B, Ke, seed)
    assert torch.equal(conflicts, rconf)
    assert torch.equal(bits(m1), bits(r1))
    assert torch.equal(bits(m2.masked_fill(conflicts, 0.0)), bits(r2.masked_fill(conflicts, 0.0)))
    assert list(feats) == list(rfeats)
    for k in feats:
        assert torch.equal(bits(feats[k]), bits(rfeats[k])), k


def test_vectorised_transfer_keeps_the_last_pair():
    """cycle_ref.transfer_pixels_ref (scatter of the last index) against the loop restatement of oracle/masking_ref."""
    from oracle import masking_ref
    gen = torch.Generator().manual_seed(0)
    img = torch.rand(3, 3, 12, 12, generator=gen)
    p1, p2 = torch.randint(0, 12, (3, 40, 2), generator=gen), torch.randint(0, 12, (3, 40, 2), generator=gen)
    assert torch.equal(cycle_ref.transfer_pixels_ref(img, p1, p2), masking_ref.transfer_pixels_ref(img, p1, p2))


def test_rendered_mask_rules_differ_on_one_zero_channel():
    r = torch.ones(1, 3, 2, 2)
    r[0, 1, 0, 0] = 0.0
    r[0, :, 1, 1] = 0.0
    assert cycle_ref.rendered_mask_first(r).flatten().tolist() == [1, 1, 1, 0]
    assert cycle_ref.rendered_mask_second(r).flatten().tolist() == [0, 1, 1, 0]


def test_cycle_entry_points_reject_bad_arguments(native_lib):
    """Checks run before any device work, so fake pointers fail cleanly with a message."""
    from smirk_b200 import _lib
    L = native_lib
    nul, buf = C.c_void_p(0), C.c_void_p(16)
    h = C.c_void_p()
    off = (C.c_int32 * 3)(0, 2, 2)
    rows = (C.c_float * 4)()
    assert L.smk_cycle_create(C.byref(_lib.SmkCycleDesc(2, off, rows, 2)), C.byref(h)) < 0 and b"no rows" in L.smk_last_error()
    assert L.smk_cycle_create(C.byref(_lib.SmkCycleDesc(0, off, rows, 2)), C.byref(h)) < 0 and b"at least one" in L.smk_last_error()
    assert L.smk_cycle_create(None, C.byref(h)) < 0 and b"null" in L.smk_last_error()
    ptrs, dims = (C.c_void_p * 6)(*([16] * 6)), (C.c_int * 6)(3, 3, 300, 50, 3, 2)
    assert L.smk_cycle_augment(nul, ptrs, ptrs, dims, 2, 1, 1, buf, None, nul) < 0 and b"null" in L.smk_last_error()
    args = [buf, 1, buf, buf, buf, None, buf, buf, 2, 1, 224, N_POINTS, 10, C.c_float(0.01), buf, buf] + [None] * 6 + [buf, 1 << 30, nul]
    bad = list(args); bad[1] = 3
    assert L.smk_masking_train_forward(*bad) < 0 and b"step must be 1 or 2" in L.smk_last_error()
    bad = list(args); bad[9] = 2
    assert L.smk_masking_train_forward(*bad) < 0 and b"Ke == 1" in L.smk_last_error()
    bad = list(args); bad[1] = 2
    assert L.smk_masking_train_forward(*bad) < 0 and b"tv_second" in L.smk_last_error()
    bad = list(args); bad[0] = None
    assert L.smk_masking_train_forward(*bad) < 0 and b"null argument" in L.smk_last_error()
    assert L.smk_masking_train_workspace_bytes(None, 2, 1, 224, N_POINTS) == 0


def test_stages_reject_cpu_tensors(native_lib, asset_root):
    from oracle import flame_ref
    from smirk_b200.cycle import CycleAugmentation
    from smirk_b200.masking import TrainMaskingStage
    faces = flame_ref.FlameConstants(asset_root).faces_tensor
    x = mgc.case_inputs(2, 1, 1)
    st = TrainMaskingStage(faces, x["base_prob"])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        st.first_path(x["img"], x["hull"], x["tv"], x["rend"])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        CycleAugmentation(mgc.synthetic_templates())(x["enc"])
    with pytest.raises(RuntimeError, match="must be"):
        CycleAugmentation({"k": np.zeros((3, 10))}, num_expression=50)
