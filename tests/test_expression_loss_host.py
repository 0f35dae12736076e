"""CPU suite for smirk_b200.ExpressionLoss: the torch restatement (tests/expression_ref.py) against the reference class
and its golden fixture, the replay oracle against plain autograd, the module tree and state_dict keys, checkpoint
loading, the arguments the module rejects without a GPU, and the drop-in alias."""
import ctypes as C
import os
import sys
import tempfile

import pytest
import torch

import expression_ref
import make_golden_expression_loss as mg

METRICS = ("l2", "l1", "cos")


def rel_err(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.fixture(scope="module")
def sd():
    return mg.golden_state_dict()


def ref_loss_and_grads(sd, gen, tar, use_mean, metric):
    gl, tl = gen.clone().requires_grad_(), tar.clone().requires_grad_()
    loss = expression_ref.expression_loss_ref(sd, gl, tl, use_mean, metric)
    gg, gt = torch.autograd.grad(loss.sum(), [gl, tl])
    return loss.detach(), gg, gt


def test_restatement_matches_golden(sd, golden):
    gold = golden("expression_loss")
    gen, tar = mg.golden_inputs()
    with torch.no_grad():
        assert rel_err(expression_ref.backbone_ref(sd, gen), gold["features_gen"]) <= 1e-6
        assert rel_err(expression_ref.backbone_ref(sd, tar), gold["features_tar"]) <= 1e-6
        for metric in METRICS:
            for use_mean, key in ((True, "loss_%s_mean"), (False, "loss_%s")):
                got = expression_ref.expression_loss_ref(sd, gen, tar, use_mean, metric)
                assert got.shape == gold[key % metric].shape
                assert rel_err(got, gold[key % metric]) <= 1e-6, (metric, use_mean)
    gl = gen.clone().requires_grad_()
    g, = torch.autograd.grad(expression_ref.expression_loss_ref(sd, gl, tar, False, "l2").mean(), [gl])
    assert rel_err(mg.subsample(g), gold["g_gen"]) <= 1e-6


def test_restatement_matches_reference_class(sd):
    from oracle import ref_harness
    if not ref_harness.available():
        pytest.skip("the reference checkout is not present (the committed fixture pins the same outputs)")
    ref = mg.reference_module(sd)
    gen = expression_ref.probe_images(1, 3)
    tar = expression_ref.perturbed(gen, 3)
    for metric in METRICS:
        for use_mean in (True, False):
            gl, tl = gen.clone().requires_grad_(), tar.clone().requires_grad_()
            rl = ref(gl, tl, use_mean=use_mean, metric=metric)
            rgg, rgt = torch.autograd.grad(rl.sum(), [gl, tl])
            ol, ogg, ogt = ref_loss_and_grads(sd, gen, tar, use_mean, metric)
            assert rl.shape == ol.shape
            assert rel_err(ol, rl.detach()) <= 1e-6 and rel_err(ogg, rgg) <= 1e-6 and rel_err(ogt, rgt) <= 1e-6, (metric, use_mean)
    with pytest.raises(ValueError, match="Unknown metric"):
        ref(gen, tar, metric="l3")


def test_replay_with_the_oracles_own_choices_is_plain_autograd(sd):
    gen = expression_ref.probe_images(1, 5)
    tar = expression_ref.perturbed(gen, 5)
    saved = expression_ref.oracle_saved(sd, gen, tar)
    for metric in METRICS:
        loss, gg, gt = ref_loss_and_grads(sd, gen, tar, False, metric)
        gl, tl = gen.clone().requires_grad_(), tar.clone().requires_grad_()
        rl = expression_ref.expression_loss_replay_ref(sd, gl, tl, saved, False, metric)
        rgg, rgt = torch.autograd.grad(rl.sum(), [gl, tl])
        assert rel_err(rl.detach(), loss) <= 1e-6
        assert rel_err(rgg, gg) <= 1e-6 and rel_err(rgt, gt) <= 1e-6, metric


def test_state_dict_keys_are_the_reference_layout(sd, golden):
    import smirk_b200
    m = smirk_b200.ExpressionLoss(checkpoint=None)
    keys = list(m.state_dict())
    assert keys == list(golden("expression_loss")["keys"]) == list(sd)
    assert len(keys) == 320
    assert len([k for k in keys if not k.endswith("num_batches_tracked") and not k.startswith("backbone.fc.")]) == 265
    assert sum(t.numel() for k, t in m.state_dict().items()
               if not k.endswith("num_batches_tracked") and not k.startswith("backbone.fc.")) == 23561152
    assert not m.backbone.training and not any(p.requires_grad for p in m.parameters())


def test_checkpoint_loads_as_the_reference_does(sd):
    import smirk_b200
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        expression_ref.write_checkpoint(sd, root)
        os.chdir(root)
        try:
            m = smirk_b200.ExpressionLoss()
        finally:
            os.chdir(old)
        fresh = smirk_b200.ExpressionLoss(checkpoint=None).state_dict()
        for k, v in m.state_dict().items():
            if k.startswith("backbone.fc."):                 # deleted from the checkpoint, strict=False: left as built
                assert v.shape == fresh[k].shape, k
            else:
                assert torch.equal(v, sd[k]), k
        os.chdir(root)
        try:
            os.remove(os.path.join(root, expression_ref.CHECKPOINT))
            with pytest.raises(FileNotFoundError):
                smirk_b200.ExpressionLoss()
        finally:
            os.chdir(old)


def test_arguments_rejected_without_a_gpu(native_lib, monkeypatch):
    import smirk_b200
    from smirk_b200 import _lib
    m = smirk_b200.ExpressionLoss(checkpoint=None)
    x = torch.rand(2, 3, 224, 224)
    with pytest.raises(ValueError, match="Unknown metric"):
        m(x, x, metric="l3")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        m(x, x)
    with monkeypatch.context() as mp:                 # the shape checks, reached without a device
        mp.setattr(_lib, "require_cuda", lambda t, name: None)
        with pytest.raises(RuntimeError, match="224x224"):
            m(torch.rand(2, 3, 112, 112), torch.rand(2, 3, 112, 112))
        with pytest.raises(RuntimeError, match="224x224"):
            m(x, torch.rand(2, 224, 224))
        with pytest.raises(RuntimeError, match="same batch size"):
            m(x, torch.rand(3, 3, 224, 224))
    with pytest.raises(RuntimeError, match="train mode"):
        m.train()(x, x)
    m.eval()
    m.backbone.layer2[1].conv2.weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="weight gradients are not implemented"):
        m(x, x)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA tensor"):
        m(x, x)                                       # under no_grad a trainable parameter is fine
    m.backbone.layer2[1].conv2.weight.requires_grad_(False)
    m.precision = 2
    with pytest.raises(RuntimeError, match="precision"):
        m._native_create("cpu")
    keep = [_lib.f32(torch.ones(2048 * 512)) for _ in range(265)]
    arr = (_lib.c_f32p * 265)(*[k[1] for k in keep])
    for precision, n, what in ((2, 265, b"precision"), (0, 264, b"265 tensors")):
        d = _lib.SmkNetDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), n, precision
        h = C.c_void_p()
        assert native_lib.smk_expression_loss_create(C.byref(d), C.byref(h)) < 0
        assert what in native_lib.smk_last_error()


def test_dropin_resolves_expression_loss_to_ours():
    from smirk_b200 import dropin
    import smirk_b200.expression_loss
    saved = {k: v for k, v in sys.modules.items() if k == "src" or k.startswith("src.")}
    with tempfile.TemporaryDirectory() as root:
        try:
            names = dropin.install(root)
            assert "src.losses.ExpressionLoss" in names and len(names) == 7
            from src.losses.ExpressionLoss import ExpressionLoss
            assert ExpressionLoss is smirk_b200.expression_loss.ExpressionLoss
        finally:
            for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
                del sys.modules[k]
            sys.modules.update(saved)
            if root in sys.path:
                sys.path.remove(root)
