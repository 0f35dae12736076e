"""Drop-in acceptance (SURVEY.md §8b / §8f #4): the reference's entry script on the smirk_b200 classes.

The flow of the reference's ``demo.py``, restated in tests/demo_flow.py, runs on the real CUDA path under
``python -m smirk_b200.dropin`` and its written grid is compared with tests/golden/demo.npz — the image the unmodified
script wrote with the reference's own classes (oracle/make_golden_demo.py).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


def _run(cmd, cwd=None):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=cwd, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("generator", [False, True])
def test_demo_flow_on_the_gpu_matches_the_reference_run(tmp_path, asset_root, native_lib, generator):
    import cv2
    import torch
    import dropin_support as ds
    img = ds.synthetic_image(str(tmp_path / "face.png"))
    ck = ds.write_checkpoint(str(tmp_path / "ck.pt"), with_generator=generator)
    out, dump = str(tmp_path / "out"), str(tmp_path / "dump.pt")
    _run([sys.executable, "-m", "smirk_b200.dropin", os.path.join(HERE, "demo_flow.py"), "--input_path", img, "--checkpoint", ck,
          "--out_path", out, "--dump", dump] + (["--use_smirk_generator"] if generator else []), cwd=asset_root)
    grid = cv2.imread(os.path.join(out, "face.png")).astype(np.int32)
    g = np.load(os.path.join(HERE, "golden", "demo.npz"))["grid"].astype(np.int32)
    assert grid.shape == (224, 224 * (3 if generator else 2), 3)
    d = np.abs(grid[:, :448] - g)
    assert np.array_equal(grid[:, :224], g[:, :224])                 # the input panel is untouched
    # rendered panel: 8-bit quantisation of values that agree to ~1e-5 may flip the last level; silhouette pixels of a
    # discontinuous rasteriser may differ between any two fp32 evaluation orders (a handful at most)
    assert (d[:, 224:] > 1).mean() < 2e-4, "rendered panel: %.3g of the pixels differ by more than one level" % (d[:, 224:] > 1).mean()
    t = torch.load(dump)
    assert set(t["outputs"]) == {"pose_params", "cam", "shape_params", "expression_params", "eyelid_params", "jaw_params"}
    if generator:
        from oracle import generator_ref
        import smirk_b200
        from smirk_b200 import synth_inputs
        gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
        sd = synth_inputs.random_state_dict(gen.state_dict(), seed=7)
        ref = generator_ref.generator_forward_ref(sd, t["generator_input"])
        err = float((t["reconstructed_img"] - ref).abs().max())
        assert err <= 5e-3, "generator on the demo flow's own input vs oracle: %.3g" % err
        m = t["generator_input"][:, 3:]
        assert float((m > 0).float().mean()) > 0.2                   # a real masked image went in: hull exterior + sampled points
