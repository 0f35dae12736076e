"""Writes tests/golden/encoder_train.npz: one train-mode step of the reference's own SmirkEncoder.

The reference class runs through ``oracle/ref_harness`` (its backbones are the restated ``encoder_ref`` ones: Tier B,
unpinned) in train mode at B = 2 with ``random_state_dict(seed=7)``.  Stored: the six outputs, the running statistics and
``num_batches_tracked`` after the step, and the gradients of the seeded loss ``sum_k (out[k] * up[k]).sum()``.  Statistics
and gradients are subsampled: per tensor its sum and the values at a seeded index sample.

    python tests/make_golden_encoder_train.py <asset root>     (needs the reference checkout)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_SAMPLE = 8
B = 2


def inputs():
    """-> (state dict, image [B,3,224,224], upstream gradients) of the fixture."""
    import smirk_b200
    from smirk_b200 import synth_inputs
    sd = synth_inputs.random_state_dict(smirk_b200.SmirkEncoder().state_dict(), seed=7)
    g = torch.Generator().manual_seed(5)
    widths = {"pose_params": 3, "cam": 3, "shape_params": 300, "expression_params": 50, "eyelid_params": 2, "jaw_params": 3}
    up = {k: torch.randn(B, w, generator=g) for k, w in widths.items()}
    return sd, synth_inputs.images(B, 77), up


def sample_index(name, n):
    """The seeded index sample of a flattened tensor of n elements (a function of its name and size)."""
    seed = sum(map(ord, name)) * 131 + n
    return np.random.default_rng(seed).integers(0, n, size=N_SAMPLE)


def summarise(prefix, tensors):
    """{prefix + "names" / "sum" / "sample": the tensor names, their sums [n] (fp64), their sampled values [n, N_SAMPLE]}."""
    names, sums, samples = [], [], []
    for k, v in tensors.items():
        a = v.detach().double().cpu().numpy().ravel()
        names.append(k)
        sums.append(a.sum())
        samples.append(a[sample_index(k, a.size)])
    return {prefix + "names": np.array(names), prefix + "sum": np.array(sums),
            prefix + "sample": np.array(samples, dtype=np.float32)}


def step(model, img, up):
    """One train-mode step of a module with the reference's output dict -> (outputs, {name: gradient})."""
    import encoder_train_ref as tr
    model.train()
    out = model(img)
    names = [n for n, _ in model.named_parameters()]
    grads = torch.autograd.grad(tr.loss(out, up), list(model.parameters()))
    return out, dict(zip(names, grads))


def main(asset_root):
    from oracle import ref_harness
    import encoder_train_ref as tr
    sd, img, up = inputs()
    with ref_harness.reference(asset_root) as R:
        ref = R.SmirkEncoder(n_exp=50, n_shape=300)
        ref.load_state_dict(sd)
        out, grads = step(ref, img, up)
    rec = {"out_" + k: out[k].detach().numpy() for k in tr.OUTPUTS}
    stats = {k: v for k, v in ref.state_dict().items() if "running_" in k}
    rec.update(summarise("stats_", stats))
    rec["num_batches_tracked"] = np.array([int(v) for k, v in ref.state_dict().items() if "num_batches" in k])
    rec.update(summarise("grad_", grads))
    path = os.path.join(ROOT, "tests", "golden", "encoder_train.npz")
    np.savez_compressed(path, **rec)
    print("wrote %s (%d KB)" % (path, os.path.getsize(path) // 1024))


if __name__ == "__main__":
    main(sys.argv[1])
