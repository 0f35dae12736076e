"""CPU suite of the live eval handles: every prototype of include/smirk_b200_live.h is exported and bound in
_lib.LIVE_BINDINGS in the header's order with matching argument kinds, the create / refresh entry points reject bad
arguments without a GPU, and the ``live_weights_`` opt-in is off by default, kept by ``copy.deepcopy`` and set on the
sub-encoders."""
import copy
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_live_header_is_exported_and_bound_in_order(native_lib):
    from smirk_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "smirk_b200_live.h")).read(), flags=re.S)
    protos = re.findall(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(smk_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M)
    assert [name for _, name, _ in protos] == [name for name, _, _ in _lib.LIVE_BINDINGS]
    assert len(protos) == 4
    main = {name for name, _, _ in _lib.BINDINGS}
    returns = {"int": C.c_int}
    values = {"int": C.c_int}
    for (ret, name, params), (bname, restype, args) in zip(protos, _lib.LIVE_BINDINGS):
        assert hasattr(native_lib, name) and name not in main, name
        assert restype is returns[ret.strip()], name
        params = [q.strip() for q in params.split(",") if q.strip()]
        assert len(args) == len(params), name
        for q, a in zip(params, args):
            if q.endswith("stream"):
                assert a is _lib.STREAM, (name, q)
            elif "*" in q:
                assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (name, q)
            else:
                assert a is values[q.rsplit(None, 1)[0]], (name, q)
        assert (name in _lib._TAKES_STREAM) == (args[-1:] == [_lib.STREAM]), name
        assert getattr(native_lib, name).argtypes is not None, name          # lib() set the binding
    assert native_lib.smk_version() == 100


def test_live_entry_points_reject_bad_arguments_without_gpu(native_lib):
    L = native_lib
    h = C.c_void_p()
    assert L.smk_encoder_live_create(0, 300, 50, 0, C.byref(h)) != 0 and b"backbones" in L.smk_last_error()
    assert L.smk_encoder_live_create(7, 300, 50, 4, C.byref(h)) != 0 and b"precision" in L.smk_last_error()
    assert L.smk_generator_live_create(6, 3, 32, 5, 2, C.byref(h)) != 0 and b"precision" in L.smk_last_error()
    assert L.smk_generator_live_create(6, 3, 12, 5, 0, C.byref(h)) != 0 and b"init_features" in L.smk_last_error()
    assert L.smk_encoder_refresh(None, None, None) != 0 and b"not a live handle" in L.smk_last_error()
    assert L.smk_generator_refresh(None, None, None) != 0 and b"not a live handle" in L.smk_last_error()


def test_live_weights_opt_in():
    import smirk_b200
    enc = smirk_b200.SmirkEncoder()
    subs = (enc.pose_encoder, enc.shape_encoder, enc.expression_encoder)
    assert not any(m.__dict__.get("_live") for m in (enc,) + subs)
    assert enc.live_weights_(True) is enc and all(m._live for m in subs)
    cp = copy.deepcopy(enc)
    assert cp._live and all(m._live for m in (cp.pose_encoder, cp.shape_encoder, cp.expression_encoder))
    assert not enc.live_weights_(False).shape_encoder._live
    from smirk_b200.smirk_encoder import ShapeEncoder
    alone = ShapeEncoder().live_weights_()
    assert alone._live and copy.deepcopy(alone)._live
    gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    assert not gen.__dict__.get("_live")
    assert gen.live_weights_(True) is gen and copy.deepcopy(gen)._live
    assert not copy.deepcopy(gen.live_weights_(False))._live
    assert not enc._train_allowed() and not gen._train_allowed()              # independent of the train-mode opt-in
