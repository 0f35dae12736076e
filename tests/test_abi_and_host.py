"""CPU suite: the C-ABI library loads and exports every symbol include/smirk_b200.h declares, the ctypes binding
table matches the header, the reference-compatible modules construct with the reference's state_dict keys, and the
product path fails loudly (no CPU fallback)."""
import copy
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_header_prototype_is_exported_and_bound_in_header_order(native_lib):
    """The library exports every prototype in include/smirk_b200.h (all 117 entry points: the input gradients, the
    video grid, the encoder's and the generator's train modes and their kernel test entry points, the trainer's masking
    and cycle augmentation, and the VGG, MICA and expression losses included), and each has exactly one row in
    _lib.BINDINGS, in the header's order, with the same return type and the same
    parameters: count, pointer / value kind, and the trailing stream where the header has one (which is what makes
    `_lib.call` append the current stream).  The ctypes structure of the augmentation's draws has the header's fields in
    its order, and the kernel test entry points of the expression loss, which the header leaves out, are exported."""
    import ctypes as C
    from smirk_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "smirk_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(smk_[a-z_0-9]+)\s*\(", hdr))
    assert len(declared) >= 19
    for name in sorted(declared):
        assert hasattr(native_lib, name), "missing export: " + name
    assert native_lib.smk_version() == 100
    protos = re.findall(r"^\s*([A-Za-z_][\w ]*?\**)\s*\b(smk_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M)
    table = {name: (restype, args) for name, restype, args in _lib.BINDINGS}
    assert len(protos) == 117 and len(table) == len(_lib.BINDINGS)
    assert [name for _, name, _ in protos] == [name for name, _, _ in _lib.BINDINGS]
    returns = {"int": C.c_int, "size_t": C.c_size_t, "void": None, "const char*": C.c_char_p, "unsigned long long": C.c_ulonglong}
    values = {"int": C.c_int, "size_t": C.c_size_t, "float": C.c_float}
    for ret, name, params in protos:
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
        assert (name in _lib._TAKES_STREAM) == (args[-1:] == [_lib.STREAM]), name
    draws = hdr[hdr.index("int64_t* gids"):hdr.index("} SmkCycleDraws")]
    assert [f for f, _ in _lib.SmkCycleDraws._fields_] == re.findall(r"\*\s*(\w+);", draws)
    for k in ("im2col", "maxpool", "maxpool_bwd", "col2im", "stem_dgrad", "head", "head_bwd"):
        assert hasattr(native_lib, "smk_debug_expression_" + k)


def test_create_rejects_bad_arguments_without_gpu(native_lib):
    import ctypes as C
    from smirk_b200 import _lib
    h = C.c_void_p()
    d = _lib.SmkFlameDesc()
    d.n_joints = 3
    rc = native_lib.smk_flame_create(C.byref(d), C.byref(h))
    assert rc < 0 and b"n_joints" in native_lib.smk_last_error()
    g = _lib.SmkGeneratorDesc()
    assert native_lib.smk_generator_create(C.byref(g), C.byref(h)) < 0


def test_modules_construct_with_reference_keys(asset_root):
    import smirk_b200
    fl, rd = smirk_b200.FLAME(), smirk_b200.Renderer()
    assert fl.faces_tensor.shape == (9976, 3) and fl.faces_tensor.dtype == torch.int64
    assert fl.shapedirs.shape == (5023, 3, 350) and fl.posedirs.shape == (36, 15069)
    assert set(fl.state_dict()) >= {"v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights",
                                    "l_eyelid", "r_eyelid", "eye_pose", "neck_pose", "lmk_faces_idx",
                                    "dynamic_lmk_bary_coords", "full_lmk_faces_idx", "neck_kin_chain", "mp_lmk_bary_coords"}
    assert fl.neck_kin_chain.tolist() == [1, 0]
    assert rd.faces.shape == (1, 3408, 3) and len(rd.final_mask) == 1787 and rd.image_size == 224
    assert set(rd.state_dict()) == {"faces", "face_colors", "raw_uvcoords", "uvcoords", "uvfaces", "face_uvcoords", "constant_factor"}
    assert rd.face_uvcoords.shape == (1, 9976, 3, 3)
    enc = smirk_b200.SmirkEncoder()
    keys = list(enc.state_dict())
    assert keys[0] == "pose_encoder.encoder.conv_stem.weight" and "shape_encoder.encoder.blocks.6.0.conv.weight" in keys
    assert "expression_encoder.encoder.blocks.1.0.conv_pwl.weight" in keys and "pose_encoder.pose_cam_layers.0.bias" in keys
    assert float(enc.pose_encoder.pose_cam_layers[0].bias.detach()[3]) == 7.0          # smirk_encoder.py:30-31
    assert float(enc.shape_encoder.shape_layers[0].weight.detach().abs().max()) == 0.0
    gen = smirk_b200.SmirkGenerator(in_channels=6, out_channels=3, init_features=32, res_blocks=5)
    gk = list(gen.state_dict())
    assert len(gk) == 178 and gk[0] == "encoder1.enc1conv1.weight" and "resnet_blocks.4.conv_block.6.running_var" in gk
    assert gen.upconv4.weight.shape == (512, 256, 2, 2)
    from smirk_b200.masking import MaskingStage
    stage = MaskingStage(fl.faces_tensor, torch.ones(fl.faces_tensor.shape[0]))
    for m in (enc, fl, rd, gen, stage):                                         # base_trainer.py:237 deep-copies the encoder
        m._native.handle = handle = object()                                    # stands in for a packed native handle
        c = copy.deepcopy(m)
        assert "_native_state" not in c.__dict__, type(m).__name__
        assert c._native is not m._native and c._native.handle is None and m._native.handle is handle
        if isinstance(m, torch.nn.Module):
            for a, b in zip(m.state_dict().values(), c.state_dict().values()):
                assert torch.equal(a, b) and (a.numel() == 0 or a.data_ptr() != b.data_ptr())
    assert len(list(enc.pose_encoder.parameters())) > 0


def test_no_cpu_fallback(asset_root):
    import smirk_b200
    fl, rd = smirk_b200.FLAME(), smirk_b200.Renderer()
    with pytest.raises(RuntimeError, match="CUDA"):
        fl.forward({"shape_params": torch.zeros(1, 300), "expression_params": torch.zeros(1, 50),
                    "pose_params": torch.zeros(1, 3), "jaw_params": torch.zeros(1, 3)})
    with pytest.raises(RuntimeError, match="CUDA"):
        rd.forward(torch.zeros(1, 5023, 3), torch.ones(1, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        smirk_b200.SmirkEncoder().eval()(torch.zeros(1, 3, 224, 224))
    with pytest.raises(RuntimeError, match="CUDA"):
        smirk_b200.SmirkGenerator(6, 3, 32, 5).eval()(torch.zeros(1, 6, 224, 224))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "smirk_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "oracle/" not in src.replace("oracle/raster_ref.c)", "").replace("oracle/make_topology_blob.py", "") or f.endswith((".cu", ".py")), f


def test_synthetic_assets_are_deterministic(asset_root, tmp_path):
    import numpy as np
    from smirk_b200 import synth_assets
    b = synth_assets.load_blob()
    m1 = synth_assets.synthetic_flame_model(b["verts"], b["faces"].astype(np.int64), seed=0)
    m2 = synth_assets.synthetic_flame_model(b["verts"], b["faces"].astype(np.int64), seed=0)
    assert np.array_equal(m1["shapedirs"], m2["shapedirs"]) and m1["shapedirs"].shape == (5023, 3, 400)
    assert np.allclose(m1["weights"].sum(1), 1) and np.allclose(m1["J_regressor"].sum(1), 1)


def test_ncu_traffic_tool_parses_an_ncu_csv(tmp_path):
    """tools/ncu_traffic.py (feeds bench.py's roofline.traffic): kernel-name -> tag mapping, unit scaling, --last-pass."""
    import json
    import subprocess
    import sys
    rows = ['"ID","Process ID","Process Name","Host Name","Kernel Name","Context","Stream","Block Size","Grid Size","Device","CC","Section Name","Metric Name","Metric Unit","Metric Value"']
    kernels = ["void smk::<unnamed>::xdw_kernel<1>(CUtensorMap_st)", "void smk::<unnamed>::gemm_tc_kernel<32, 2, 5, 0>(CUtensorMap_st)",
               "void at::native::vectorized_elementwise_kernel<4>()", "void smk::<unnamed>::xdw_kernel<2>(CUtensorMap_st)"]
    for i, k in enumerate(kernels):
        for metric, unit, val in (("dram__bytes_read.sum", "Mbyte", "2.5"), ("dram__bytes_write.sum", "Kbyte", "500"), ("gpu__time_duration.sum", "us", "10")):
            rows.append('"%d","1","python","h","%s","1","7","(320, 1, 1)","(148, 1, 1)","0","10.0","Cmd","%s","%s","%s"' % (i, k, metric, unit, val))
    src, out = tmp_path / "n.csv", tmp_path / "t.json"
    src.write_text("==PROF== Connected\n" + "\n".join(rows) + "\n")
    tool = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "ncu_traffic.py")
    subprocess.check_call([sys.executable, tool, str(src), str(out)], stdout=subprocess.DEVNULL)
    d = json.load(open(out))["kernels"]
    assert set(d) == {"xdw_fused_tc", "pw_gemm_tc"} and d["xdw_fused_tc"]["launches"] == 2
    assert abs(d["xdw_fused_tc"]["traffic_bytes_per_launch"] - 3.0e6) < 1 and abs(d["pw_gemm_tc"]["ncu_us"] - 10.0) < 1e-9
    subprocess.check_call([sys.executable, tool, str(src), str(out), "--last-pass", "1"], stdout=subprocess.DEVNULL)
    assert set(json.load(open(out))["kernels"]) == {"xdw_fused_tc"}
