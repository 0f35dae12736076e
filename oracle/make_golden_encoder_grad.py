"""ORACLE — TEST INFRASTRUCTURE ONLY.  Writes tests/golden/encoder_grad.npz: torch autograd of sum_k (out[k] * up[k]).sum()
over the six outputs with respect to the image, through the REFERENCE's own ``SmirkEncoder`` (src/smirk_encoder.py; its
timm backbones are the restated ones of oracle/encoder_ref.py through the ``ref_harness`` stub), eval mode, parameters
frozen (as src/smirk_trainer.py:334-337 freezes it for the cycle path), weights ``random_state_dict(seed=7)``.  The
image is the input of encoder.npz; the upstream gradients are seeded (``upstream()``).  The heads, clamps and output
split are the reference's (Tier A); the backbones are the restatement (Tier B, unpinned).  Stored subsampled.
Re-run: ``python -m oracle.make_golden_encoder_grad``.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from smirk_b200 import synth_assets, synth_inputs  # noqa: E402
from oracle import ref_harness  # noqa: E402
from oracle.encoder_replay_ref import OUTPUTS, loss  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
WIDTHS = {"pose_params": 3, "cam": 3, "shape_params": 300, "expression_params": 50, "eyelid_params": 2, "jaw_params": 3}


def encoder_input():
    """The input of encoder.npz."""
    return synth_inputs.images(2, 401)


def upstream(B=2, seed=313):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(B, WIDTHS[k], generator=g) for k in OUTPUTS}


def subsample(g):
    return {"sub": g[:, :, ::4, ::4], "rows": g[:, :, 100:102, :], "sum": g.sum((2, 3))}


def main():
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))
    with ref_harness.reference(root) as R:
        enc = R.SmirkEncoder().eval()
        enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
        enc.requires_grad_(False)
        img = encoder_input().requires_grad_()
        loss(enc(img), upstream()).backward()
        out = {"g_img_" + k: v.numpy() for k, v in subsample(img.grad).items()}
    np.savez_compressed(os.path.join(GOLD, "encoder_grad.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))


if __name__ == "__main__":
    main()
