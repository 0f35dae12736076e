"""CPU suite for smirk_b200.MICA: the torch restatement (tests/mica_ref.py) against the reference class and its golden
fixture, the module tree and state_dict keys, checkpoint loading, the ABI of include/smirk_b200_mica.h, the arguments the
module rejects without a GPU, and the drop-in alias."""
import ctypes as C
import os
import re
import sys
import tempfile

import pytest
import torch

import make_golden_mica as mg
import mica_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_err(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.fixture(scope="module")
def sd():
    return mica_ref.mica_state_dict(mg.SEED)


def test_restatement_matches_golden_and_reference_class(sd, golden):
    gold = golden("mica")
    img = mg.golden_images()
    shape, feat = mica_ref.mica_ref(sd, img)
    assert rel_err(feat, gold["features"]) <= 1e-6
    assert rel_err(shape, gold["shape_params"]) <= 1e-6
    for D in (300, 100):
        s = mg.golden_shape_params(D).requires_grad_()
        loss = mica_ref.shape_loss_ref(s, shape)
        g, = torch.autograd.grad(loss, [s])
        assert abs(float(loss) - float(gold["loss_%d" % D])) <= 1e-6 * abs(float(gold["loss_%d" % D]))
        assert rel_err(g, gold["grad_%d" % D]) <= 1e-6
    from oracle import ref_harness
    if not ref_harness.available():
        pytest.skip("the reference checkout is not present (the committed fixture pins the same outputs)")
    img2 = mica_ref.probe_images(1, 3)
    ref = mg.reference_outputs(sd, img2)
    shape2, feat2 = mica_ref.mica_ref(sd, img2)
    assert rel_err(feat2, ref["features"]) <= 1e-6 and rel_err(shape2, ref["shape_params"]) <= 1e-6
    for D in (300, 100):
        s = mg.golden_shape_params(D, 1).requires_grad_()
        loss = mica_ref.shape_loss_ref(s, shape2)
        g, = torch.autograd.grad(loss, [s])
        assert abs(float(loss) - float(ref["loss_%d" % D])) <= 1e-6 * abs(float(ref["loss_%d" % D]))
        assert rel_err(g, ref["grad_%d" % D]) <= 1e-6


def test_state_dict_keys_are_the_reference_layout(sd):
    import smirk_b200
    m = smirk_b200.MICA(checkpoint=None)
    assert list(m.state_dict()) == list(sd)
    assert len([k for k in sd if not k.endswith("num_batches_tracked")]) == 781
    frozen = {n for n, p in m.named_parameters() if not p.requires_grad}
    assert "arcface.layer3.29.conv2.weight" in frozen and "arcface.conv1.weight" in frozen
    assert "arcface.layer4.0.conv1.weight" not in frozen and "regressor.output.weight" not in frozen   # as the reference
    from oracle import ref_harness
    if ref_harness.available():
        with ref_harness.reference(mg.asset_root()):
            from src.models.MICA.arcface import Arcface
            from src.models.MICA.mica import MappingNetwork
            want = ["arcface." + k for k in Arcface().state_dict()] + \
                   ["regressor." + k for k in MappingNetwork(512, 300, 300, hidden=3).state_dict()]
        assert list(m.state_dict()) == want


def test_checkpoint_loads_as_the_reference_does(sd):
    import smirk_b200
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        mica_ref.write_checkpoint(sd, root)
        os.chdir(root)
        try:
            m = smirk_b200.MICA()
        finally:
            os.chdir(old)
        for k, v in m.state_dict().items():
            assert torch.equal(v, sd[k]), k
        os.chdir(root)
        try:
            os.remove(os.path.join(root, "assets", "mica.tar"))
            with pytest.raises(FileNotFoundError):
                smirk_b200.MICA()
        finally:
            os.chdir(old)


def test_mica_header_prototypes_are_exported_and_bound_in_header_order(native_lib):
    """Every prototype of include/smirk_b200_mica.h is exported and has one row in _lib.MICA_BINDINGS, in the header's
    order, with the same return type and parameter kinds, and the trailing stream where the header has one."""
    from smirk_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "smirk_b200_mica.h")).read(), flags=re.S)
    protos = re.findall(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(smk_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M)
    assert len(protos) == 6 and [n for _, n, _ in protos] == [n for n, _, _ in _lib.MICA_BINDINGS]
    assert not {n for n, _, _ in _lib.MICA_BINDINGS} & {n for n, _, _ in _lib.BINDINGS + _lib.LOSS_BINDINGS}
    returns = {"int": C.c_int, "size_t": C.c_size_t, "void": None}
    values = {"int": C.c_int, "size_t": C.c_size_t, "float": C.c_float}
    table = {name: (restype, args) for name, restype, args in _lib.MICA_BINDINGS}
    for ret, name, params in protos:
        assert hasattr(native_lib, name), "missing export: " + name
        restype, args = table[name]
        assert restype is returns[ret.strip()], name
        params = [q.strip() for q in params.split(",") if q.strip() not in ("", "void")]
        assert len(args) == len(params), name
        for q, a in zip(params, args):
            if q.endswith("stream"):
                assert a is _lib.STREAM, (name, q)
            elif "*" in q:
                assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (name, q)
            else:
                assert a is values[q.rsplit(None, 1)[0]], (name, q)


def test_arguments_rejected_without_a_gpu():
    import smirk_b200
    m = smirk_b200.MICA(checkpoint=None).eval()
    for p in m.parameters():
        p.requires_grad = False
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        m(torch.rand(1, 3, 112, 112))
    with pytest.raises(RuntimeError, match="train mode"):
        m.train()(torch.rand(1, 3, 112, 112))
    m.eval()
    m.arcface.fc.weight.requires_grad = True
    with pytest.raises(RuntimeError, match="requires_grad=False"):
        m(torch.rand(1, 3, 112, 112))
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA tensor"):
        m(torch.rand(1, 3, 112, 112))                     # under no_grad the trainable head is fine
    m.precision = 2
    with pytest.raises(RuntimeError, match="precision"):
        m._native_create("cpu")


def test_dropin_resolves_mica_to_ours():
    from smirk_b200 import dropin
    import smirk_b200.mica
    saved = {k: v for k, v in sys.modules.items() if k == "src" or k.startswith("src.")}
    with tempfile.TemporaryDirectory() as root:
        try:
            names = dropin.install(root)
            assert "src.models.MICA.mica" in names
            from src.models.MICA.mica import MICA
            assert MICA is smirk_b200.mica.MICA
        finally:
            for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
                del sys.modules[k]
            sys.modules.update(saved)
            if root in sys.path:
                sys.path.remove(root)
