"""SHA-256 of the demo's ``MaskingStage`` outputs and exported draws at fixed (seed, counter), for the smirk_b200 package
found under a given tree.  Comparing two trees (two commits, each built with ``python -m smirk_b200.build``) on one GPU
shows whether a change to csrc/masking.cu altered what the demo path computes:

    python tools/masking_digest.py <tree A>;  python tools/masking_digest.py <tree B>

Inputs: the meshes, hull masks and face weights of tests/golden/masking.npz (read from this file's tree), images from
``synth_inputs`` (seeds 5 and 99), seed 4242 at counters 0 and 7; hashed: the masked images and every debug output.
"""
import hashlib
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(tree):
    tree = os.path.abspath(tree)
    sys.path.insert(0, tree)
    import numpy as np
    import torch
    from smirk_b200 import _lib, masking, synth_assets, synth_inputs
    assert os.path.dirname(_lib.__file__).startswith(tree), "imported %s, not the package under %s" % (_lib.__file__, tree)
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_digest_%d" % os.getuid()))
    from oracle import flame_ref
    faces = flame_ref.FlameConstants(root).faces_tensor
    g = np.load(os.path.join(HERE, "tests", "golden", "masking.npz"))
    dev = "cuda:0"
    tv = torch.from_numpy(g["trans_verts"]).to(dev)
    B = tv.shape[0]
    img = synth_inputs.images(B, 5).to(dev)
    hull = torch.from_numpy(g["hull"]).float().to(dev)
    rend = (synth_inputs.images(B, 99) * torch.from_numpy(g["rendered_img_nonzero"]).float()).to(dev)
    st = masking.MaskingStage(faces, torch.from_numpy(g["base_prob"]), n_verts=5023, seed=4242)
    h = hashlib.sha256()
    for counter in (0, 7):
        st.reseed(4242, counter)
        out, d = st.forward(img, hull, tv, rend, debug=True)
        torch.cuda.synchronize()
        for t in [out] + [d[k] for k in sorted(d)]:
            h.update(t.cpu().contiguous().numpy().tobytes())
    print("MaskingStage digest", h.hexdigest())


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
