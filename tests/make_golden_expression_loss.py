"""Writes tests/golden/expression_loss.npz: what the REFERENCE's own ExpressionLoss (src/losses/ExpressionLoss.py)
computes on seeded weights.  It writes ``expression_ref.expression_state_dict(seed=7)`` as the reference's checkpoint
under the synthetic asset root (``backbone.*`` with ``backbone.fc.*``, plus ``linear.*``: both are deleted by the loader),
builds the reference's ``ExpressionLoss()`` through oracle.ref_harness (which changes into that root) with
``nn.Module.cuda`` made a no-op, and stores at B = 2 (``golden_inputs()``):

  features_gen, features_tar   the backbone features [2,2048]
  loss_<metric>_mean, loss_<metric>   the loss for each metric, with use_mean True and False
  g_gen                        autograd's gradient to gen of the trainer's call (l2, use_mean=False, then .mean()),
                               subsampled 4x in each spatial direction
  keys                         the module's state_dict keys

Re-run: ``python tests/make_golden_expression_loss.py``.
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
import expression_ref  # noqa: E402

GOLD = os.path.join(HERE, "golden")
SEED = 7
METRICS = ("l2", "l1", "cos")


def golden_inputs():
    gen = expression_ref.probe_images(2, 11)
    return gen, expression_ref.perturbed(gen, 11)


def golden_state_dict():
    return expression_ref.expression_state_dict(SEED)


def subsample(g):
    return g[:, :, ::4, ::4]


def asset_root():
    return synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))


def reference_module(sd):
    """The reference class itself, loaded from a checkpoint of sd (on the CPU)."""
    import torch.nn as nn
    from oracle import ref_harness
    root = asset_root()
    expression_ref.write_checkpoint(sd, root)
    cuda = nn.Module.cuda
    nn.Module.cuda = lambda self, *a, **k: self
    try:
        with ref_harness.reference(root):
            from src.losses.ExpressionLoss import ExpressionLoss
            ref = ExpressionLoss()
    finally:
        nn.Module.cuda = cuda
    return ref.eval()


def reference_outputs(sd, gen, tar):
    ref = reference_module(sd)
    out = {}
    with torch.no_grad():
        out["features_gen"] = ref.backbone(gen).view(gen.shape[0], -1)
        out["features_tar"] = ref.backbone(tar).view(tar.shape[0], -1)
        for metric in METRICS:
            out["loss_%s_mean" % metric] = ref(gen, tar, use_mean=True, metric=metric)
            out["loss_%s" % metric] = ref(gen, tar, use_mean=False, metric=metric)
    gl = gen.clone().requires_grad_()
    out["g_gen"], = torch.autograd.grad(ref(gl, tar, metric="l2", use_mean=False).mean(), [gl])
    out["keys"] = list(ref.state_dict())
    return out


def main():
    gen, tar = golden_inputs()
    out = reference_outputs(golden_state_dict(), gen, tar)
    out["g_gen"] = subsample(out["g_gen"])
    out = {k: (np.array(v) if k == "keys" else v.detach().numpy()) for k, v in out.items()}
    np.savez_compressed(os.path.join(GOLD, "expression_loss.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, v.dtype)


if __name__ == "__main__":
    main()
