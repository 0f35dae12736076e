"""ORACLE — TEST INFRASTRUCTURE ONLY.  Writes tests/golden/generator_grad.npz: torch autograd of (y * g_y).sum() with
respect to the input x through the REFERENCE's own ``SmirkGenerator(6, 3, 32, 5)`` (src/smirk_generator.py), eval mode,
parameters frozen (as src/smirk_trainer.py:108-116 runs it for the emotion loss), weights ``random_state_dict(seed=7)``.
x is the input of generator.npz; g_y is seeded (``upstream()``).  Stored subsampled like generator.npz.
Re-run: ``python -m oracle.make_golden_generator_grad``.
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

GOLD = os.path.join(HERE, "..", "tests", "golden")


def generator_input():
    """The input of generator.npz: the reference's rendered image of render.npz + a seeded masked image."""
    r = np.load(os.path.join(GOLD, "render.npz"))
    return torch.cat([torch.from_numpy(r["rendered_img"][:1]), synth_inputs.masked_images(1, 301)], 1)


def upstream(B=1, seed=311):
    return torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(seed))


def subsample(g):
    return {"sub": g[:, :, ::4, ::4], "rows": g[:, :, 100:102, :], "sum": g.sum((2, 3))}


def main():
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))
    with ref_harness.reference(root) as R:
        gen = R.SmirkGenerator(in_channels=6, out_channels=3, init_features=32, res_blocks=5).eval()
        gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
        gen.requires_grad_(False)
        x = generator_input().requires_grad_()
        (gen(x) * upstream()).sum().backward()
        out = {"g_x_" + k: v.numpy() for k, v in subsample(x.grad).items()}
    np.savez_compressed(os.path.join(GOLD, "generator_grad.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))


if __name__ == "__main__":
    main()
