"""Writes tests/golden/cycle.npz: the masked images of the reference trainer's own ``SmirkTrainer.step1`` and the
``flame_feats`` and masked images of its ``step2``, at B = 4 and 5, Ke = 1, on the CPU.

The reference class runs through ``oracle/ref_harness``.  ``__init__`` is bypassed (it loads template and mask assets that
are not shipped); the config is the relevant part of ``configs/config_train.yaml`` with ``device = 'cpu'``; the templates
are synthetic.  Stub encoder, FLAME and Renderer return fixed tensors, and a stub generator records its input and stops
the step, so the step's own masking and augmentation code runs unchanged between them.  Stored per case: the seeds, the
``flame_feats`` tensors, and for each masked image its SHA-256 and every 16th pixel.  Where two point pairs with different
sources hit one target pixel (``cycle_ref.conflicting_targets``, from the points the reference's own ``transfer_pixels``
received), the pixel the reference keeps is an implementation detail of torch's CPU index_put; the second path's digest
is taken with those pixels zeroed, and their count is stored.

    python tests/make_golden_cycle.py <asset root>     (needs the reference checkout)
"""
import hashlib
import os
import random
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cycle_ref  # noqa: E402
OUT = os.path.join(ROOT, "tests", "golden", "cycle.npz")
MASKING = os.path.join(ROOT, "tests", "golden", "masking.npz")
KEYS = ("pose_params", "cam", "shape_params", "expression_params", "eyelid_params", "jaw_params")    # SmirkEncoder's order
DIMS = {"pose_params": 3, "cam": 3, "shape_params": 300, "expression_params": 50, "eyelid_params": 2, "jaw_params": 3}
CASES = ((4, 1, 101), (5, 1, 202))                    # (B, Ke, seed)
SUB = 16


def synthetic_templates():
    """Stand-in for load_templates(): key -> [rows, 100] float64, rows differing per key."""
    rng = np.random.default_rng(17)
    return {"S%02dkey%d" % (i, i): rng.standard_normal((n, 100)) for i, n in enumerate((2, 5, 1, 8, 3, 6))}


def case_inputs(B, Ke, seed):
    """Encoder outputs, the first / second path's meshes and renders, images and hull masks of one case."""
    from smirk_b200 import synth_inputs
    g = np.load(MASKING)
    gen = torch.Generator().manual_seed(seed)
    enc = {k: torch.randn(B, DIMS[k], generator=gen) for k in KEYS}
    enc["eyelid_params"] = torch.rand(B, 2, generator=gen)
    enc["jaw_params"][:, 0] = enc["jaw_params"][:, 0].abs() * 0.3
    tv0 = torch.from_numpy(g["trans_verts"])
    tv = tv0[torch.arange(B) % tv0.shape[0]] + 0.01 * torch.randn(B, tv0.shape[1], 3, generator=gen)
    tv2 = tv.repeat(Ke, 1, 1) + 0.02 * torch.randn(Ke * B, tv0.shape[1], 3, generator=gen)
    nz = torch.from_numpy(g["rendered_img_nonzero"]).float()
    rend = synth_inputs.images(B, seed + 1) * nz[torch.arange(B) % 2]
    rend2 = synth_inputs.images(Ke * B, seed + 2) * nz[torch.arange(Ke * B) % 2]
    rend[:, 1, 100:110, 100:140] = 0.0
    rend2[:, 2, 90:120, 100:110] = 0.0                 # one zero channel: foreground for step1's rule, not step2's
    img = synth_inputs.images(B, seed + 3)
    hull = torch.from_numpy(g["hull"]).float()[torch.arange(B) % 2]
    return dict(enc=enc, tv=tv, tv2=tv2, rend=rend, rend2=rend2, img=img, hull=hull,
                base_prob=torch.from_numpy(g["base_prob"]), lmk_fan=torch.randn(B, 68, 2, generator=gen),
                lmk_mp=torch.randn(B, 105, 2, generator=gen))


class _Stop(Exception):
    pass


def run_reference(asset_root, B, Ke, seed):
    """-> (masked_1st_path, flame_feats, masked_img_2nd_path, conflicting target pixels of step2's transfer) of the
    reference's step1 and step2 with torch and Python seeded with ``seed`` before each step."""
    from oracle import ref_harness
    import torch.nn as nn
    x = case_inputs(B, Ke, seed)
    with ref_harness.reference(asset_root) as ref:
        from src import smirk_trainer
        from oracle import flame_ref
        faces = flame_ref.FlameConstants(asset_root).faces_tensor
        tr = smirk_trainer.SmirkTrainer.__new__(smirk_trainer.SmirkTrainer)
        nn.Module.__init__(tr)

        class Weights(dict):
            __getattr__ = dict.__getitem__
        ns = types.SimpleNamespace
        tr.config = ns(device="cpu",
                       train=ns(mask_ratio=0.01, mask_dilation_radius=10, Ke=Ke, use_base_model_for_regularization=False,
                                freeze_generator_in_second_path=False, visualize_every=50, optimize_shape=False,
                                optimize_expression=True,
                                loss_weights=Weights(landmark_loss=100.0, perceptual_vgg_loss=10.0, reconstruction_loss=10.0,
                                                     emotion_loss=0.0, jaw_regularization=1e-2, expression_regularization=1e-3,
                                                     shape_regularization=100, cycle_loss=1.0, mica_loss=0)),
                       arch=ns(num_expression=50, num_shape=300, use_eyelids=True, enable_fuse_generator=True))
        tr.templates = synthetic_templates()
        tr.face_probabilities = x["base_prob"]
        recorded = {"gen": [], "flame": [], "transfer": []}
        transfer = smirk_trainer.masking_utils.transfer_pixels

        def record_transfer(img, points1, points2, rbound=None):
            recorded["transfer"].append((points1.clone(), points2.clone()))
            return transfer(img, points1, points2, rbound)
        renders = []

        def flame_forward(feats):
            recorded["flame"].append({k: v.clone() for k, v in feats.items()})
            return {"vertices": feats["expression_params"], "landmarks_fan": x["lmk_fan"], "landmarks_mp": x["lmk_mp"]}

        def renderer_forward(vertices, cam, **kw):
            tv, rend = renders.pop(0)
            return {"rendered_img": rend, "transformed_vertices": tv}

        def generator(inp):
            recorded["gen"].append(inp[:, 3:6].clone())
            raise _Stop()
        tr.__dict__["smirk_encoder"] = lambda img: x["enc"]
        tr.__dict__["base_encoder"] = lambda img: x["enc"]
        tr.__dict__["flame"] = ns(forward=flame_forward, faces_tensor=faces)
        tr.__dict__["renderer"] = ns(forward=renderer_forward)
        tr.__dict__["smirk_generator"] = generator
        batch = {"img": x["img"], "mask": x["hull"], "flag_landmarks_fan": torch.ones(B, dtype=torch.bool),
                 "landmarks_fan": x["lmk_fan"], "landmarks_mp": x["lmk_mp"]}
        renders[:] = [(x["tv"], x["rend"])]
        smirk_trainer.masking_utils.transfer_pixels = record_transfer
        try:
            torch.manual_seed(seed); random.seed(seed)
            try:
                tr.step1(batch)
            except _Stop:
                pass
            renders[:] = [(x["tv"], x["rend"]), (x["tv2"], x["rend2"])]
            torch.manual_seed(seed + 1); random.seed(seed + 1)
            try:
                tr.step2(x["enc"], batch, 0)
            except _Stop:
                pass
        finally:
            smirk_trainer.masking_utils.transfer_pixels = transfer
    masked1, masked2 = recorded["gen"]
    p1, p2 = recorded["transfer"][-1]
    return masked1, recorded["flame"][-1], masked2, cycle_ref.conflicting_targets(p1, p2)


def digest(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def main(asset_root):
    out = {}
    for B, Ke, seed in CASES:
        m1, feats, m2, conflicts = run_reference(asset_root, B, Ke, seed)
        m2 = m2.masked_fill(conflicts, 0.0)
        p = "B%d" % B
        out[p + "/seed"] = np.array([seed, seed + 1])
        for k, v in feats.items():
            out[p + "/flame_feats/" + k] = v.numpy()
        for name, t in (("masked_1st_path", m1), ("masked_img_2nd_path", m2)):
            out[p + "/" + name + "/sha256"] = np.array(digest(t))
            out[p + "/" + name + "/sub"] = t[:, :, ::SUB, ::SUB].numpy()
        out[p + "/conflicts"] = np.array(int(conflicts.sum()))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
