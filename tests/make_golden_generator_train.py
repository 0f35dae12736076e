"""Writes tests/golden/generator_train.npz: one train-mode step of the reference's own SmirkGenerator.

The reference class runs through ``oracle/ref_harness`` on the CPU in train mode at (6, 3, 32, 5), B = 2, with
``random_state_dict(seed=7)`` and momentum 0.1.  Stored: the output subsampled every 8th pixel, the running statistics
and ``num_batches_tracked`` after the step, and the gradients of the seeded loss ``(y * gy).sum()`` for every parameter
and the input.  Statistics and gradients are summarised as in ``make_golden_encoder_train``: per tensor its sum and the
values at a seeded index sample.

    python tests/make_golden_generator_train.py <asset root>     (needs the reference checkout)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from make_golden_encoder_train import summarise  # noqa: E402

CFG = (6, 3, 32, 5)
B = 2
SUB = 8


def inputs():
    """-> (state dict, input [B,6,224,224], upstream gradient [B,3,224,224]) of the fixture."""
    import smirk_b200
    from smirk_b200 import synth_inputs
    sd = synth_inputs.random_state_dict(smirk_b200.SmirkGenerator(*CFG).state_dict(), seed=7)
    x = torch.cat([synth_inputs.images(B, 910), synth_inputs.masked_images(B, 911)], 1)[:, :CFG[0]].contiguous()
    gy = torch.randn(B, CFG[1], 224, 224, generator=torch.Generator().manual_seed(912))
    return sd, x, gy


def step(model, x, gy):
    """One train-mode step -> (y, {"input" and every parameter name: gradient})."""
    xl = x.clone().requires_grad_()
    y = model(xl)
    names = [n for n, _ in model.named_parameters()]
    grads = torch.autograd.grad((y * gy.to(y.device)).sum(), [xl] + list(model.parameters()))
    return y, dict(zip(["input"] + names, grads))


def record(y, state, grads):
    rec = {"out": y.detach().cpu()[:, :, ::SUB, ::SUB].numpy()}
    rec.update(summarise("stats_", {k: v for k, v in state.items() if "running_" in k}))
    rec["num_batches_tracked"] = np.array([int(v) for k, v in state.items() if "num_batches" in k])
    rec.update(summarise("grad_", grads))
    return rec


def main(asset_root):
    from oracle import ref_harness
    sd, x, gy = inputs()
    with ref_harness.reference(asset_root) as R:
        ref = R.SmirkGenerator(*CFG)
        ref.load_state_dict(sd)
        ref.train()
        y, grads = step(ref, x, gy)
    path = os.path.join(ROOT, "tests", "golden", "generator_train.npz")
    np.savez_compressed(path, **record(y, ref.state_dict(), grads))
    print("wrote %s (%d KB)" % (path, os.path.getsize(path) // 1024))


if __name__ == "__main__":
    main(sys.argv[1])
