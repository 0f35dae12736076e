"""Writes tests/golden/mica.npz: what the REFERENCE's own MICA (src/models/MICA/mica.py) computes on seeded weights.  It
writes ``mica_ref.mica_state_dict(seed=7)`` as ``assets/mica.tar`` under the synthetic asset root (its ``flameModel`` part
holds the ``regressor.``-prefixed keys among others the loader drops), builds the reference's ``MICA()`` through
oracle.ref_harness (which changes into that root), and stores at B = 3 (``golden_images()``):

  features       the ArcFace embedding before F.normalize [3,512]
  shape_params   [3,300]
  loss_300, grad_300   calculate_mica_shape_loss and its autograd gradient for ``golden_shape_params(300)``
  loss_100, grad_100   the same at D = 100 (the truncation case)

Re-run: ``python tests/make_golden_mica.py``.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from smirk_b200 import synth_assets  # noqa: E402
import mica_ref  # noqa: E402

GOLD = os.path.join(HERE, "golden")
SEED = 7


def golden_images():
    return mica_ref.probe_images(3, 11)


def golden_shape_params(D, B=3):
    g = torch.Generator().manual_seed(100 + D)
    return torch.randn(B, D, generator=g) * 0.05


def asset_root():
    return synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))


def reference_outputs(sd, images):
    """The reference class itself, loaded from a checkpoint of sd: {features, shape_params, loss_D, grad_D}."""
    from oracle import ref_harness
    root = asset_root()
    mica_ref.write_checkpoint(sd, root)
    out = {}
    with ref_harness.reference(root):
        from src.models.MICA.mica import MICA
        ref = MICA().eval()
        with torch.no_grad():
            x = images.sub(0.5).div(0.5)[:, [2, 1, 0], :, :]
            out["features"] = ref.arcface(x)
            out["shape_params"] = ref(images)["shape_params"]
        for D in (300, 100):
            s = golden_shape_params(D, images.shape[0]).requires_grad_()
            loss = ref.calculate_mica_shape_loss(s, images)
            out["loss_%d" % D], = (loss.detach(),)
            out["grad_%d" % D], = torch.autograd.grad(loss, [s])
    return out


def main():
    out = reference_outputs(mica_ref.mica_state_dict(SEED), golden_images())
    out = {k: v.detach().numpy() for k, v in out.items()}
    np.savez_compressed(os.path.join(GOLD, "mica.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))


if __name__ == "__main__":
    main()
