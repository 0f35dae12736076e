"""CPU suite of the train-mode encoder: the C ABI with the train entry points, their argument checks, the opt-in and mode
checks of the module, the dropin runner's --train flag, and the train-mode restatement (tests/encoder_train_ref.py)
against the reference's own SmirkEncoder (when the reference checkout is present)."""
import copy
import ctypes as C
import os
import re

import pytest
import torch
import torch.nn as nn

import encoder_train_ref as tr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_train_header_prototypes_are_exported_and_bound(native_lib):
    """include/smirk_b200_train.h is included by smirk_b200.h; the library exports each of its 4 prototypes, and each has
    exactly one row in _lib.TRAIN_BINDINGS (header order, no row shared with BINDINGS) with the same return type and
    parameters: count, pointer / value kind, and the trailing stream, which `_lib.call` fills in."""
    from smirk_b200 import _lib
    main = open(os.path.join(ROOT, "include", "smirk_b200.h")).read()
    assert '#include "smirk_b200_train.h"' in main
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "smirk_b200_train.h")).read(), flags=re.S)
    protos = re.findall(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(smk_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M)
    assert [name for _, name, _ in protos] == [name for name, _, _ in _lib.TRAIN_BINDINGS] and len(protos) == 4
    assert not {name for name, _, _ in _lib.TRAIN_BINDINGS} & {name for name, _, _ in _lib.BINDINGS}
    table = {name: (restype, args) for name, restype, args in _lib.TRAIN_BINDINGS}
    returns = {"int": C.c_int, "size_t": C.c_size_t}
    for ret, name, params in protos:
        assert hasattr(native_lib, name), "missing export: " + name
        restype, args = table[name]
        assert restype is returns[ret.strip()], name
        params = [q.strip() for q in params.split(",") if q.strip()]
        assert len(args) == len(params), name
        for q, a in zip(params, args):
            if q.endswith("stream"):
                assert a is _lib.STREAM, (name, q)
            elif "*" in q:
                assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (name, q)
            else:
                assert a is {"int": C.c_int, "size_t": C.c_size_t}[q.rsplit(None, 1)[0]], (name, q)
        assert (name in _lib._TAKES_STREAM) == (args[-1:] == [_lib.STREAM]), name


def test_train_entry_points_reject_bad_arguments(native_lib):
    from smirk_b200 import _lib
    L = native_lib
    vp, nul = C.c_void_p, C.c_void_p(0)
    h = C.c_void_p()
    assert L.smk_encoder_train_create(0, 300, 50, 0, C.byref(h)) < 0 and b"bit set" in L.smk_last_error()
    assert L.smk_encoder_train_create(7, 300, 50, 4, C.byref(h)) < 0 and b"precision" in L.smk_last_error()
    args = _lib.SmkEncoderTrainArgs()
    buf = vp(16)
    rc = L.smk_encoder_forward_train(nul, C.byref(args), buf, 2, buf, buf, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"not a train-mode handle" in L.smk_last_error()
    rc = L.smk_encoder_backward_train(nul, C.byref(args), buf, 2, buf, 1 << 20, buf, buf, buf, buf, None, buf, 1 << 20, nul)
    assert rc < 0 and b"not a train-mode handle" in L.smk_last_error()
    assert L.smk_encoder_train_workspace_bytes(nul, 4) == 0


def _encoder():
    import smirk_b200
    return smirk_b200.SmirkEncoder()


def test_opt_in_and_mode_checks_without_gpu(native_lib):
    """The checks that need no device: the flag (per module, deep-copied; the process-wide default off) and the
    one-momentum rule.  A CPU image fails the device check first, as on the eval path."""
    from smirk_b200 import smirk_encoder
    assert not smirk_encoder.train_mode_default()
    enc = _encoder().train()
    assert enc.allow_train_mode_(True) is enc
    assert all(m._train_allowed() for m in (enc, enc.pose_encoder, enc.shape_encoder, enc.expression_encoder))
    assert copy.deepcopy(enc)._train_allowed() and copy.deepcopy(enc.pose_encoder)._train_allowed()
    enc.allow_train_mode_(False)
    assert not enc._train_allowed()
    assert not _encoder()._train_allowed()
    smirk_encoder.set_train_mode_default(True)
    try:
        assert _encoder()._train_allowed() and not enc._train_allowed()     # the per-module flag wins
    finally:
        smirk_encoder.set_train_mode_default(False)
    bb = _encoder().shape_encoder.encoder
    assert smirk_encoder._bn_settings(bb, "x") == (0.1, 1e-3)
    bb.bn1.momentum = None
    with pytest.raises(RuntimeError, match="one momentum"):
        smirk_encoder._bn_settings(bb, "x")
    for m in bb.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = 1.5
    with pytest.raises(RuntimeError, match="momentum in"):
        smirk_encoder._bn_settings(bb, "x")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        _encoder().train()(torch.zeros(1, 3, 224, 224))


def test_dropin_train_flag_turns_the_default_on_for_the_script(tmp_path):
    """`python -m smirk_b200.dropin --train script` runs the script with the opt-in on; without the flag it stays off.
    In a child process: the runner aliases the reference's modules in sys.modules."""
    import subprocess
    import sys
    script = tmp_path / "probe.py"
    script.write_text("from smirk_b200 import smirk_encoder\nprint('default', smirk_encoder.train_mode_default())\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    for flag, want in ((["--train"], "default True"), ([], "default False")):
        r = subprocess.run([sys.executable, "-s", "-m", "smirk_b200.dropin"] + flag + [str(script)], cwd=str(tmp_path), env=env,
                           capture_output=True, text=True)
        assert r.returncode == 0 and want in r.stdout, r.stderr


def test_restatement_matches_reference_class_in_train_mode(asset_root):
    """Outputs, running statistics and num_batches_tracked after 1 and 3 steps (momentum 0.1 and None), and every
    parameter gradient to 1e-6 of each tensor's scale, against the reference's own SmirkEncoder (restated backbones)."""
    from oracle import ref_harness
    from smirk_b200 import synth_inputs
    if not ref_harness.available():
        pytest.skip("reference checkout not available")
    sd = synth_inputs.random_state_dict(_encoder().state_dict(), seed=7)
    g = torch.Generator().manual_seed(5)
    widths = {"pose_params": 3, "cam": 3, "shape_params": 300, "expression_params": 50, "eyelid_params": 2, "jaw_params": 3}
    up = {k: torch.randn(2, w, generator=g) for k, w in widths.items()}
    with ref_harness.reference(asset_root) as R:
        for momentum in (0.1, None):
            ref = R.SmirkEncoder(n_exp=50, n_shape=300)
            ref.load_state_dict(sd)
            ours = tr.EncoderTrainRef()
            ours.load_state_dict(sd)
            for m in list(ref.modules()) + list(ours.modules()):
                if isinstance(m, nn.BatchNorm2d):
                    m.momentum = momentum
            ref.train(); ours.train()
            for step in range(3):
                img = synth_inputs.images(2, 60 + step)
                o_ref, o = ref(img), ours(img)
                for k in tr.OUTPUTS:
                    assert torch.allclose(o[k], o_ref[k], rtol=0, atol=1e-6 * o_ref[k].abs().max().item() + 1e-12), (momentum, step, k)
                if step == 0:
                    gr = dict(zip([n for n, _ in ref.named_parameters()], torch.autograd.grad(tr.loss(o_ref, up), list(ref.parameters()))))
                    go = dict(zip([n for n, _ in ours.named_parameters()], torch.autograd.grad(tr.loss(o, up), list(ours.parameters()))))
                    assert set(gr) == set(go)
                    for n in gr:
                        err = (go[n].double() - gr[n].double()).abs().max() / tr.grad_scale(n, gr)
                        assert err <= 1e-6, (n, float(err))
                s_ref, s = ref.state_dict(), ours.state_dict()
                for k, v in s_ref.items():
                    if "running_" in k or "num_batches" in k:
                        assert torch.equal(v, s[k]) if "num_batches" in k else torch.allclose(v, s[k], rtol=1e-6, atol=1e-7), (momentum, step, k)


def test_restatement_reproduces_the_golden_train_step(golden):
    """tests/golden/encoder_train.npz (one train-mode step of the reference's SmirkEncoder, tests/make_golden_encoder_train.py):
    outputs, running statistics, num_batches_tracked and the sampled gradients, from the restatement."""
    import make_golden_encoder_train as mg
    gold = golden("encoder_train")
    sd, img, up = mg.inputs()
    ours = tr.EncoderTrainRef()
    ours.load_state_dict(sd)
    out, grads = mg.step(ours, img, up)
    for k in tr.OUTPUTS:
        ref = torch.from_numpy(gold["out_" + k])
        assert (out[k].detach() - ref).abs().max() <= 1e-6 * ref.abs().max(), k
    stats = {k: v for k, v in ours.state_dict().items() if "running_" in k}
    assert [int(v) for k, v in ours.state_dict().items() if "num_batches" in k] == gold["num_batches_tracked"].tolist()
    for prefix, tensors in (("stats_", stats), ("grad_", grads)):
        mine = mg.summarise(prefix, tensors)
        assert mine[prefix + "names"].tolist() == gold[prefix + "names"].tolist()
        for i, name in enumerate(gold[prefix + "names"]):
            if tr.zero_in_exact_arithmetic(str(name)):                # rounding noise on both sides
                continue
            a, b = mine[prefix + "sample"][i], gold[prefix + "sample"][i]
            assert abs(a - b).max() <= 1e-6 * max(abs(b).max(), 1e-30), name
