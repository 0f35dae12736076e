"""CPU suite of the train-mode generator: the argument checks of its entry points, the opt-in and its messages, and the
train-mode oracle (tests/generator_train_ref.py) against the reference's own SmirkGenerator (when the reference checkout
is present)."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn as nn

import generator_train_ref as gtr


def test_entry_points_reject_bad_arguments(native_lib):
    from smirk_b200 import _lib
    L = native_lib
    h, nul, buf = C.c_void_p(), C.c_void_p(0), C.c_void_p(16)
    assert L.smk_generator_train_create(6, 3, 32, 5, 2, C.byref(h)) < 0 and b"precision" in L.smk_last_error()
    assert L.smk_generator_train_create(6, 3, 12, 5, 0, C.byref(h)) < 0 and b"init_features" in L.smk_last_error()
    assert L.smk_generator_train_create(6, 3, 16, 5, 1, C.byref(h)) < 0 and b"tensor-core" in L.smk_last_error()
    args = _lib.SmkGeneratorTrainArgs()
    rc = L.smk_generator_forward_train(nul, C.byref(args), buf, 2, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"not a train-mode handle" in L.smk_last_error()
    rc = L.smk_generator_backward_train(nul, C.byref(args), 2, buf, buf, 1 << 20, buf, buf, None, buf, 1 << 20, nul)
    assert rc < 0 and b"not a train-mode handle" in L.smk_last_error()
    assert L.smk_generator_train_workspace_bytes(nul, 4) == 0
    assert L.smk_debug_train_conv3_wgrad(buf, buf, 4, 1, 8, 8, 8, 8, 0, buf, buf, 1 << 24, nul) < 0 and b"lda" in L.smk_last_error()


def test_opt_in_without_gpu(native_lib):
    """The flag is one flag with the encoder's, per module it overrides the default and deep copies keep it; without it a
    train-mode generator raises before it touches a device tensor.  A CPU input fails the device check first."""
    import smirk_b200
    from smirk_b200 import _lib, smirk_encoder
    g = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    assert not smirk_encoder.train_mode_default() and not g._train_allowed()
    smirk_encoder.set_train_mode_default(True)
    try:
        assert _lib.train_mode_default() and g._train_allowed() and smirk_b200.SmirkEncoder()._train_allowed()
        assert not copy.deepcopy(g).allow_train_mode_(False)._train_allowed()
    finally:
        smirk_encoder.set_train_mode_default(False)
    assert copy.deepcopy(g.allow_train_mode_(True))._train_allowed()
    g.allow_train_mode_(False)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        g.train()(torch.zeros(1, 6, 224, 224))
    with pytest.raises(RuntimeError, match="train-mode.*allow_train_mode_"):
        g._is_train()
    g.eval()
    assert g._is_train() is False
    g.encoder1.enc1norm1.train()
    g.allow_train_mode_(True)
    with pytest.raises(RuntimeError, match="mix train and eval"):
        g._is_train()


def test_dropin_docstring_names_the_generator():
    from smirk_b200 import dropin
    assert "SmirkGenerator" in dropin.__doc__ and "config_train.yaml" in dropin.__doc__


@pytest.mark.parametrize("momentum", [0.1, None])
def test_oracle_matches_reference_class_in_train_mode(asset_root, momentum):
    """Outputs, running statistics and num_batches_tracked over 3 steps, and every parameter and input gradient of the
    first, to 1e-6 of each tensor's scale, against the reference's own SmirkGenerator in train mode (at (6, 3, 16, 2),
    the trainer's layer kinds at a CPU-friendly width)."""
    from oracle import ref_harness
    import smirk_b200
    from smirk_b200 import synth_inputs
    if not ref_harness.available():
        pytest.skip("reference checkout not available")
    cfg = (6, 3, 16, 2)
    sd0 = synth_inputs.random_state_dict(smirk_b200.SmirkGenerator(*cfg).state_dict(), seed=7)
    close = lambda a, b: torch.allclose(a.detach().double(), b.detach().double(), rtol=0, atol=1e-6 * float(b.detach().abs().max()) + 1e-12)
    with ref_harness.reference(asset_root) as R:
        ref = R.SmirkGenerator(*cfg)
        ref.load_state_dict(sd0)
        for m in ref.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.momentum = momentum
        ref.train()
        sd = gtr.cpu_state(ref)
        for step in range(3):
            x = torch.randn(2, 6, 224, 224, generator=torch.Generator().manual_seed(40 + step))
            gy = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(50 + step))
            xr, xo = x.clone().requires_grad_(), x.clone().requires_grad_()
            yr = ref(xr)
            yo = gtr.generator_train_ref(sd, xo, res_blocks=cfg[3], momentum=momentum)
            assert close(yo, yr), step
            for k, v in ref.state_dict().items():
                if "running" in k or "num_batches" in k:
                    assert close(sd[k], v), (step, k)
            if step == 0:
                names = [n for n, _ in ref.named_parameters()]
                gr = torch.autograd.grad((yr * gy).sum(), [xr] + list(ref.parameters()))
                go = torch.autograd.grad((yo * gy).sum(), [xo] + [sd[n] for n in names])
                for n, a, b in zip(["input"] + names, go, gr):
                    assert close(a, b), n


def test_restatement_reproduces_the_golden_file(golden):
    """tests/golden/generator_train.npz (the reference's SmirkGenerator, one train step at B = 2): the train-mode oracle
    gives its subsampled output, running statistics, counters and the sums and samples of every gradient to 1e-6."""
    import make_golden_generator_train as mg
    gold = golden("generator_train")
    sd0, x, gy = mg.inputs()
    import smirk_b200
    m = smirk_b200.SmirkGenerator(*mg.CFG)
    m.load_state_dict(sd0)
    sd = gtr.cpu_state(m)
    xl = x.clone().requires_grad_()
    y = gtr.generator_train_ref(sd, xl, res_blocks=mg.CFG[3])
    names = [n for n, _ in m.named_parameters()]
    grads = torch.autograd.grad((y * gy).sum(), [xl] + [sd[n] for n in names])
    rec = mg.record(y, {k: v.detach() for k, v in sd.items()}, dict(zip(["input"] + names, grads)))
    close = lambda a, b: float(abs(a.astype("float64") - b).max()) <= 1e-6 * float(abs(b).max()) + 1e-12
    assert close(rec["out"], gold["out"])
    assert list(rec["num_batches_tracked"]) == list(gold["num_batches_tracked"]) == [1] * len(gold["num_batches_tracked"])
    for part in ("stats_", "grad_"):
        assert list(rec[part + "names"]) == list(gold[part + "names"])
        for i, n in enumerate(gold[part + "names"]):
            assert close(rec[part + "sample"][i], gold[part + "sample"][i]), n
            scale = float(abs(gold[part + "sample"][i]).max()) * gold[part + "sample"].shape[1] + 1e-12
            assert abs(rec[part + "sum"][i] - gold[part + "sum"][i]) <= 1e-5 * max(scale, abs(gold[part + "sum"][i])), n
