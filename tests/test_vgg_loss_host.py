"""CPU suite for smirk_b200.VGGPerceptualLoss: the module tree and state_dict keys of the reference class, the torch
restatement (tests/vgg_ref.py) against the reference class and its golden fixture, the replay oracle against plain
autograd, and the arguments the module rejects."""
import ctypes as C

import pytest
import torch

import make_golden_vgg_loss as mg
import vgg_ref


def rel_err(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def ref_loss_and_grads(sd, x, y):
    xl, yl = x.clone().requires_grad_(), y.clone().requires_grad_()
    loss = vgg_ref.vgg_loss_ref(sd, xl, yl)
    return (loss.detach(),) + torch.autograd.grad(loss, [xl, yl])


def test_state_dict_keys_are_the_reference_layout():
    import torchvision
    import smirk_b200
    m = smirk_b200.VGGPerceptualLoss(weights=None)
    feats = torchvision.models.vgg16(weights=None).features
    want = ["mean", "std"] + ["blocks.%d.%s" % (i, k) for i, (lo, hi) in enumerate(((0, 4), (4, 9), (9, 16), (16, 23)))
                              for k in feats[lo:hi].state_dict()]
    assert list(m.state_dict()) == want and len(want) == 22
    assert [k[:-len(".weight")] for k in want if k.endswith(".weight")] == vgg_ref.CONVS
    assert not any(p.requires_grad for p in m.parameters())
    for a, b in zip(m.blocks.modules(), m.train().blocks.modules()):
        assert type(a) is type(b)
    assert torch.equal(m.mean.flatten(), torch.tensor([0.485, 0.456, 0.406]))


def test_restatement_matches_reference_class_and_golden(golden):
    sd = mg.golden_state_dict()
    x, y = mg.golden_inputs()
    loss, gx, gy = ref_loss_and_grads(sd, x, y)
    gold = golden("vgg_loss")
    assert abs(float(loss) - float(gold["loss"])) <= 1e-6 * abs(float(gold["loss"]))
    assert rel_err(mg.subsample(gx), torch.from_numpy(gold["g_x"])) <= 1e-6
    assert rel_err(mg.subsample(gy), torch.from_numpy(gold["g_y"])) <= 1e-6
    from oracle import ref_harness
    if not ref_harness.available():
        pytest.skip("the reference checkout is not present (the committed fixture pins the same outputs)")
    x1, y1 = x[:1] * 0.5, y[1:] * 0.9
    rl, rgx, rgy = mg.reference_loss_and_grads(sd, x1, y1)
    ol, ogx, ogy = ref_loss_and_grads(sd, x1, y1)
    assert abs(float(ol) - float(rl)) <= 1e-6 * abs(float(rl))
    assert rel_err(ogx, rgx) <= 1e-6 and rel_err(ogy, rgy) <= 1e-6
    keys = list(mg.reference_module(sd).state_dict())
    import smirk_b200
    assert keys == list(smirk_b200.VGGPerceptualLoss(weights=None).state_dict())


def test_replay_with_the_oracles_own_choices_is_plain_autograd():
    sd = mg.golden_state_dict()
    x, y = mg.golden_inputs()
    x, y = x[:1], y[:1]
    saved = vgg_ref.oracle_saved(sd, x, y)
    loss, gx, gy = ref_loss_and_grads(sd, x, y)
    xl, yl = x.clone().requires_grad_(), y.clone().requires_grad_()
    rl = vgg_ref.vgg_loss_replay_ref(sd, xl, yl, saved)
    rgx, rgy = torch.autograd.grad(rl, [xl, yl])
    rl = rl.detach()
    assert abs(float(rl) - float(loss)) <= 1e-6 * float(loss)
    assert rel_err(rgx, gx) <= 1e-6 and rel_err(rgy, gy) <= 1e-6


def test_bad_arguments_raise(native_lib, monkeypatch):
    import smirk_b200
    from smirk_b200 import _lib
    m = smirk_b200.VGGPerceptualLoss(weights=None)
    x = torch.zeros(2, 3, 224, 224)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, x)
    with monkeypatch.context() as mp:                 # the shape checks, reached without a device
        mp.setattr(_lib, "require_cuda", lambda t, name: None)
        with pytest.raises(RuntimeError, match="224x224"):
            m(torch.zeros(2, 3, 256, 256), torch.zeros(2, 3, 256, 256))
        with pytest.raises(RuntimeError, match="224x224"):
            m(x, torch.zeros(2, 3, 112, 112))
        with pytest.raises(RuntimeError, match="same batch size"):
            m(x, torch.zeros(3, 3, 224, 224))
    getattr(m.blocks[1], "5").weight.requires_grad_(True)      # blocks.1.5.weight
    with pytest.raises(RuntimeError, match="weight gradients are not implemented"):
        m(x, x)
    keep = [_lib.f32(torch.ones(512 * 512 * 9)) for _ in range(22)]
    arr = (_lib.c_f32p * 22)(*[k[1] for k in keep])
    for precision, n, what in ((2, 22, b"precision"), (0, 21, b"22 tensors")):
        d = _lib.SmkNetDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), n, precision
        h = C.c_void_p()
        assert native_lib.smk_vgg_loss_create(C.byref(d), C.byref(h)) < 0
        assert what in native_lib.smk_last_error()
