"""Writes tests/golden/encoder_saved_digests.json: SHA-256 digests of what the grad-mode encoder forward
(``smk_encoder_forward_saved``, seeded weights and images) returns on an H100 — the raw outputs of every backbone the module
holds and every tensor of the saved-activation buffer — for SmirkEncoder and each sub-encoder alone at B = 1, 7 and 32, at
every precision (0 fp32, 1 TF32 with the stem and block 0 unfused, 2 TF32, 3 3xTF32 as benched).  The forward has no
atomics and no data-dependent reduction order, so its bytes are a function of its inputs: a kernel change that keeps the
arithmetic must keep every digest.

Re-run on an H100 at the commit whose bytes are the reference: ``python tests/make_golden_encoder_saved.py [out.json]``.
"""
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from smirk_b200 import synth_inputs  # noqa: E402

GOLD = os.path.join(HERE, "golden", "encoder_saved_digests.json")
MODULES = ("SmirkEncoder", "PoseEncoder", "ShapeEncoder", "ExpressionEncoder")
BATCHES = (1, 7, 32)
PRECISIONS = (0, 1, 2, 3)


def key(precision, name, B):
    """The digests' key; precision 3's carry no prefix."""
    return "%s%s/B%d" % ("" if precision == 3 else "p%d/" % precision, name, B)


def make_module(name, precision=3, dev="cuda"):
    from smirk_b200 import smirk_encoder
    m = getattr(smirk_encoder, name)()
    m.load_state_dict(synth_inputs.random_state_dict(m.state_dict(), seed=7))
    m = m.eval().requires_grad_(False).to(dev)
    m.precision = precision
    return m


def sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def digests(m, B):
    """{"out<i>": digest of raw output i (None for a backbone the module does not hold), "saved": one digest over every
    saved tensor in layout order (the alignment gaps between them are never written, so they are left out)}."""
    from smirk_b200 import _lib
    img = synth_inputs.images(B, 100 + B).cuda()
    h, outs, saved = m._forward_saved(img)
    torch.cuda.synchronize()
    d = {"out%d" % i: (sha(o) if o is not None else None) for i, o in enumerate(outs)}
    views = _lib.saved_views("encoder", h, saved, B)
    d["saved"] = hashlib.sha256("".join(k + sha(v) for k, v in views.items()).encode()).hexdigest()
    return d


def all_digests():
    return {key(p, name, B): digests(make_module(name, p), B) for p in PRECISIONS for name in MODULES for B in BATCHES}


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    res = all_digests()
    res["device"] = torch.cuda.get_device_name(0)
    with open(out, "w") as fh:
        json.dump(res, fh, indent=1, sort_keys=True)
    print("wrote", out)
