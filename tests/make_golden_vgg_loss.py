"""Writes tests/golden/vgg_loss.npz: the loss and torch autograd g_x, g_y of the REFERENCE's own VGGPerceptualLoss
(src/losses/VGGPerceptualLoss.py), imported through oracle.ref_harness with ``torchvision.models.vgg16`` patched first to
return an untrained vgg16 filled with the seeded weights of ``vgg_ref.vgg_state_dict(seed=7)`` (the same for all four of
its calls; there is no network to download the ImageNet weights from).  Inputs: ``golden_inputs()``, B = 2.  The gradients
are stored subsampled 2x in each spatial direction.  Re-run: ``python tests/make_golden_vgg_loss.py``.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from smirk_b200 import synth_assets, synth_inputs  # noqa: E402
import vgg_ref  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def golden_inputs():
    """x, y [2,3,224,224] in [-1, 1) (the generator's output range as the trainer feeds it)."""
    return synth_inputs.images(2, 401) * 2 - 1, synth_inputs.images(2, 402) * 2 - 1


def golden_state_dict():
    import smirk_b200
    return vgg_ref.vgg_state_dict(smirk_b200.VGGPerceptualLoss(weights=None).state_dict(), seed=7)


def subsample(g):
    return g[:, :, ::2, ::2]


def reference_module(sd):
    """The reference class itself, its VGG16 filled with the weights of sd."""
    import torchvision
    from oracle import ref_harness
    feats = {k.split(".", 2)[2]: v for k, v in sd.items() if k.startswith("blocks.")}     # blocks.1.5.weight -> 5.weight
    orig = torchvision.models.vgg16

    def seeded_vgg16(weights=None, **kw):
        m = orig(weights=None)
        m.features[:23].load_state_dict(feats)
        return m
    torchvision.models.vgg16 = seeded_vgg16
    try:
        root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_golden"))
        with ref_harness.reference(root):
            from src.losses.VGGPerceptualLoss import VGGPerceptualLoss
            ref = VGGPerceptualLoss()
    finally:
        torchvision.models.vgg16 = orig
    assert torch.equal(ref.mean, sd["mean"]) and torch.equal(ref.std, sd["std"])
    return ref


def reference_loss_and_grads(sd, x, y):
    """The reference class on (x, y) with the weights of sd: (loss, g_x, g_y)."""
    ref = reference_module(sd)
    xl, yl = x.clone().requires_grad_(), y.clone().requires_grad_()
    loss = ref(xl, yl)
    gx, gy = torch.autograd.grad(loss, [xl, yl])
    return loss.detach(), gx, gy


def main():
    x, y = golden_inputs()
    loss, gx, gy = reference_loss_and_grads(golden_state_dict(), x, y)
    out = {"loss": loss.numpy(), "g_x": subsample(gx).numpy(), "g_y": subsample(gy).numpy()}
    np.savez_compressed(os.path.join(GOLD, "vgg_loss.npz"), **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))


if __name__ == "__main__":
    main()
