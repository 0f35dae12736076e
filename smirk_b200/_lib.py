"""ctypes binding of libsmirk_b200.so (the C ABI declared in include/smirk_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the product
path raises.  Build with ``python -m smirk_b200.build`` (or ``__graft_entry__.build()``).
"""
import copy
import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmirk_b200.so")
_lib = None
_TRAIN_MODE_DEFAULT = False


def set_train_mode_default(on):
    """Process-wide default of the train-mode opt-in of the encoder and the generator (off until set; a module's
    ``allow_train_mode_`` overrides it)."""
    global _TRAIN_MODE_DEFAULT
    _TRAIN_MODE_DEFAULT = bool(on)


def train_mode_default():
    return _TRAIN_MODE_DEFAULT


c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)


class SmkFlameDesc(C.Structure):
    _fields_ = [("n_verts", C.c_int), ("n_faces", C.c_int), ("n_betas", C.c_int), ("n_joints", C.c_int),
                ("v_template", c_f32p), ("shapedirs", c_f32p), ("posedirs", c_f32p), ("J_regressor", c_f32p),
                ("lbs_weights", c_f32p), ("l_eyelid", c_f32p), ("r_eyelid", c_f32p), ("faces", c_i32p),
                ("n_static", C.c_int), ("static_faces", c_i32p), ("static_bary", c_f32p),
                ("n_dyn_rows", C.c_int), ("n_dyn", C.c_int), ("dyn_faces", c_i32p), ("dyn_bary", c_f32p),
                ("n_full", C.c_int), ("full_faces", c_i32p), ("full_bary", c_f32p),
                ("n_mp", C.c_int), ("mp_faces", c_i32p), ("mp_bary", c_f32p)]


class SmkRendererDesc(C.Structure):
    _fields_ = [("n_verts", C.c_int), ("n_mask", C.c_int), ("mask_ids", c_i32p), ("n_faces", C.c_int),
                ("faces", c_i32p), ("image_size", C.c_int), ("z_offset", C.c_float)]


class SmkEncoderDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p) * 3), ("n_tensors", C.c_int * 3),
                ("head_w", c_f32p * 3), ("head_b", c_f32p * 3),
                ("n_shape", C.c_int), ("n_exp", C.c_int), ("precision", C.c_int)]


class SmkEncoderTrainArgs(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p) * 3), ("n_tensors", C.c_int * 3),
                ("num_batches_tracked", C.POINTER(C.POINTER(C.c_int64)) * 3),
                ("head_w", c_f32p * 3), ("head_b", c_f32p * 3), ("momentum", C.c_float * 3), ("eps", C.c_float * 3)]


class SmkEncoderTrainGrads(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p) * 3), ("head_w", c_f32p * 3), ("head_b", c_f32p * 3)]


class SmkGeneratorDesc(C.Structure):
    _fields_ = [("in_channels", C.c_int), ("out_channels", C.c_int), ("init_features", C.c_int),
                ("res_blocks", C.c_int), ("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int),
                ("precision", C.c_int)]


class SmkGeneratorTrainArgs(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int), ("num_batches_tracked", C.POINTER(C.POINTER(C.c_int64))),
                ("momentum", C.c_float), ("eps", C.c_float)]


class SmkGeneratorTrainGrads(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p))]


class SmkNetDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int), ("precision", C.c_int)]


# The names of the three frozen networks' descriptors from before they shared SmkNetDesc (the same layout), kept so that
# code written against them still builds the descriptor.
SmkVggLossDesc = SmkMicaDesc = SmkExpressionLossDesc = SmkNetDesc


class SmkMaskingDesc(C.Structure):
    _fields_ = [("n_verts", C.c_int), ("n_faces", C.c_int), ("faces", c_i32p)]


class SmkCycleDesc(C.Structure):
    _fields_ = [("n_keys", C.c_int), ("row_offset", c_i32p), ("rows", c_f32p), ("n_exp", C.c_int)]


class SmkCycleDraws(C.Structure):
    """Device pointers of the augmentation's exported draws (include/smirk_b200.h), in the header's field order."""
    FIELDS = ("gids", "perm1", "param_mask", "jaw_mask", "randn0a", "randn0b", "randn1", "randn2", "randn3", "randn_jaw",
              "rand0a", "rand0b", "rand1a", "rand1b", "rand2a", "rand2b", "rand3", "rand_eyelid", "rand3_eyelid", "tmpl_key", "tmpl_row")
    _fields_ = [(f, C.c_void_p) for f in FIELDS]


# The binding table: one (name, return type, argument types) row per entry point of include/smirk_b200.h, in the
# header's order.  STREAM marks a trailing `void* stream`, which `call` fills in with the current stream.  An `int`
# result is a status code, except for smk_version and smk_profiler_report, which only this file calls.
STREAM = "stream"
_vp, _i, _sz, _f, _vpp = C.c_void_p, C.c_int, C.c_size_t, C.c_float, C.POINTER(C.c_void_p)
BINDINGS = [
    ("smk_version", _i, []),
    ("smk_last_error", C.c_char_p, []),
    ("smk_launch_count", C.c_ulonglong, []),
    ("smk_profiler_enable", None, [_i]),
    ("smk_profiler_reset", None, []),
    ("smk_profiler_report", _i, [C.c_char_p, _sz]),
    ("smk_flame_create", _i, [C.POINTER(SmkFlameDesc), _vpp]),
    ("smk_flame_destroy", None, [_vp]),
    ("smk_flame_workspace_bytes", _sz, [_vp, _i]),
    ("smk_flame_forward", _i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_flame_backward_workspace_bytes", _sz, [_vp, _i]),
    ("smk_flame_backward", _i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_renderer_create", _i, [C.POINTER(SmkRendererDesc), _vpp]),
    ("smk_renderer_destroy", None, [_vp]),
    ("smk_renderer_workspace_bytes", _sz, [_vp, _i]),
    ("smk_renderer_forward", _i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_project_points", _i, [_vp, _vp, _i, _i, _vp, STREAM]),
    ("smk_renderer_backward_workspace_bytes", _sz, [_vp, _i]),
    ("smk_renderer_backward", _i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_project_points_backward", _i, [_vp, _vp, _i, _i, _vp, _vp, _vp, STREAM]),
    ("smk_encoder_create", _i, [C.POINTER(SmkEncoderDesc), _vpp]),
    ("smk_encoder_destroy", None, [_vp]),
    ("smk_encoder_workspace_bytes", _sz, [_vp, _i]),
    ("smk_encoder_forward", _i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_encoder_saved_bytes", _sz, [_vp, _i]),
    ("smk_encoder_forward_saved", _i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_encoder_saved_tensor", _i, [_vp, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_encoder_backward_workspace_bytes", _sz, [_vp, _i]),
    ("smk_encoder_backward", _i, [_vp, _i, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_encoder_train_create", _i, [_i, _i, _i, _i, _vpp]),
    ("smk_encoder_train_workspace_bytes", _sz, [_vp, _i]),
    ("smk_encoder_forward_train", _i, [_vp, C.POINTER(SmkEncoderTrainArgs), _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_encoder_backward_train", _i, [_vp, C.POINTER(SmkEncoderTrainArgs), _vp, _i, _vp, _sz, _vp, _vp, _vp, _vp,
                                        C.POINTER(SmkEncoderTrainGrads), _vp, _sz, STREAM]),
    ("smk_generator_create", _i, [C.POINTER(SmkGeneratorDesc), _vpp]),
    ("smk_generator_destroy", None, [_vp]),
    ("smk_generator_workspace_bytes", _sz, [_vp, _i]),
    ("smk_generator_forward", _i, [_vp, _vp, _i, _vp, _vp, _sz, STREAM]),
    ("smk_generator_saved_bytes", _sz, [_vp, _i]),
    ("smk_generator_forward_saved", _i, [_vp, _vp, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_generator_saved_tensor", _i, [_vp, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_generator_backward_workspace_bytes", _sz, [_vp, _i]),
    ("smk_generator_backward", _i, [_vp, _i, _vp, _vp, _sz, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_generator_train_create", _i, [_i, _i, _i, _i, _i, _vpp]),
    ("smk_generator_train_workspace_bytes", _sz, [_vp, _i]),
    ("smk_generator_forward_train", _i, [_vp, C.POINTER(SmkGeneratorTrainArgs), _vp, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_generator_backward_train", _i, [_vp, C.POINTER(SmkGeneratorTrainArgs), _i, _vp, _vp, _sz, _vp, _vp,
                                          C.POINTER(SmkGeneratorTrainGrads), _vp, _sz, STREAM]),
    ("smk_debug_train_conv3_wgrad", _i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_warp_workspace_bytes", _sz, [_i]),
    ("smk_crop_warp", _i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_warp_u8", _i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_f32chw_to_u8hwc", _i, [_vp, _i, _i, _vp, STREAM]),
    ("smk_hull_mask", _i, [_vp, _i, _i, _i, _vp, STREAM]),
    ("smk_video_workspace_bytes", _sz, [_i, _i]),
    ("smk_video_compose", _i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _sz, STREAM]),
    ("smk_masking_create", _i, [C.POINTER(SmkMaskingDesc), _vpp]),
    ("smk_masking_destroy", None, [_vp]),
    ("smk_masking_workspace_bytes", _sz, [_vp, _i, _i]),
    ("smk_masking_face_weights", _i, [_vp, _vp, _vp, _i, _vp, _vp, _sz, STREAM]),
    ("smk_masking_points", _i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, STREAM]),
    ("smk_masking_compose", _i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_masking_transfer_pixels", _i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_masking_forward_workspace_bytes", _sz, [_vp, _i, _i, _i]),
    ("smk_masking_forward", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp, _vp, _sz, STREAM]),
    ("smk_masking_train_workspace_bytes", _sz, [_vp, _i, _i, _i, _i]),
    ("smk_masking_train_forward", _i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp,
                                       _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_cycle_create", _i, [C.POINTER(SmkCycleDesc), _vpp]),
    ("smk_cycle_destroy", None, [_vp]),
    ("smk_cycle_augment", _i, [_vp, _vpp, _vpp, C.POINTER(C.c_int), _i, _i, _i, _vp, C.POINTER(SmkCycleDraws), STREAM]),
    ("smk_vgg_loss_create", _i, [C.POINTER(SmkNetDesc), _vpp]),
    ("smk_vgg_loss_destroy", None, [_vp]),
    ("smk_vgg_loss_workspace_bytes", _sz, [_vp, _i]),
    ("smk_vgg_loss_forward", _i, [_vp, _vp, _vp, _i, _vp, _vp, _sz, STREAM]),
    ("smk_vgg_loss_saved_bytes", _sz, [_vp, _i, _i]),
    ("smk_vgg_loss_forward_saved", _i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_vgg_loss_saved_tensor", _i, [_vp, _i, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_vgg_loss_backward_workspace_bytes", _sz, [_vp, _i, _i]),
    ("smk_vgg_loss_backward", _i, [_vp, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_mica_create", _i, [C.POINTER(SmkNetDesc), _vpp]),
    ("smk_mica_destroy", None, [_vp]),
    ("smk_mica_workspace_bytes", _sz, [_vp, _i]),
    ("smk_mica_forward", _i, [_vp, _vp, _i, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_mica_shape_loss_forward", _i, [_vp, _vp, _i, _i, _i, _vp, STREAM]),
    ("smk_mica_shape_loss_backward", _i, [_vp, _vp, _i, _i, _i, _vp, _vp, STREAM]),
    ("smk_expression_loss_create", _i, [C.POINTER(SmkNetDesc), _vpp]),
    ("smk_expression_loss_destroy", None, [_vp]),
    ("smk_expression_loss_workspace_bytes", _sz, [_vp, _i]),
    ("smk_expression_loss_forward", _i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_expression_loss_saved_bytes", _sz, [_vp, _i, _i]),
    ("smk_expression_loss_forward_saved", _i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_expression_loss_saved_tensor", _i, [_vp, _i, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_expression_loss_backward_workspace_bytes", _sz, [_vp, _i, _i]),
    ("smk_expression_loss_backward", _i, [_vp, _i, _i, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_peer_alloc", _i, [_sz, _vpp, C.c_char_p]),
    ("smk_peer_free", _i, [_vp]),
    ("smk_peer_open", _i, [C.c_char_p, _vpp]),
    ("smk_peer_close", _i, [_vp]),
    ("smk_peer_push", _i, [_vp, _vp, _sz, STREAM]),
    ("smk_peer_fan_create", _i, [_i, _vpp]),
    ("smk_peer_fan_destroy", None, [_vp]),
    ("smk_peer_fan_push", _i, [_vp, _vpp, _i, _vp, _sz, STREAM]),
    ("smk_debug_conv_f32", _i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, STREAM]),
    ("smk_debug_conv_tc", _i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, STREAM]),
    ("smk_debug_reflect_halo", _i, [_vp, _i, _i, _i, _i, STREAM]),
    ("smk_debug_xdw", _i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp, STREAM]),
    ("smk_debug_conv3_win", _i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _i, STREAM]),
    ("smk_debug_gemm_tc3x", _i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, STREAM]),
    ("smk_debug_xdw3x", _i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, STREAM]),
    ("smk_debug_stem_ds", _i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, STREAM]),
    ("smk_debug_train_bn_forward", _i, [_vp, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_debug_train_bn_backward", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_debug_train_pw_wgrad", _i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_debug_train_dw_forward", _i, [_vp, _vp, _i, _i, _i, _i, _vp, STREAM]),
    ("smk_debug_train_dw_wgrad", _i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_debug_train_dw_dgrad", _i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, STREAM]),
    ("smk_debug_train_stem_forward", _i, [_vp, _vp, _i, _i, _i, _vp, STREAM]),
    ("smk_debug_train_stem_wgrad", _i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, STREAM]),
    ("smk_debug_train_head_backward", _i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, STREAM]),
]
# The live eval handles of include/smirk_b200_live.h, in that header's order.
LIVE_BINDINGS = [
    ("smk_encoder_live_create", _i, [_i, _i, _i, _i, _vpp]),
    ("smk_encoder_refresh", _i, [_vp, C.POINTER(SmkEncoderTrainArgs), STREAM]),
    ("smk_generator_live_create", _i, [_i, _i, _i, _i, _i, _vpp]),
    ("smk_generator_refresh", _i, [_vp, C.POINTER(SmkGeneratorTrainArgs), STREAM]),
]
_TAKES_STREAM = frozenset(name for name, _, args in BINDINGS + LIVE_BINDINGS if args[-1:] == [STREAM])


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("smirk_b200: %s not found — build it with `python -m smirk_b200.build` "
                           "(there is no CPU / PyTorch fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, restype, argtypes in BINDINGS + LIVE_BINDINGS:
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, [_vp if a is STREAM else a for a in argtypes]
    if L.smk_version() != 100:
        raise RuntimeError("smirk_b200: library/header version mismatch (%d)" % L.smk_version())
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        msg = lib().smk_last_error().decode("utf-8", "replace")
        raise RuntimeError("smirk_b200: %s failed (rc=%d): %s" % (what, rc, msg))


def call(name, device, *args):
    """Run entry point ``name`` for tensors on ``device``: under that device (launches go to the tensors' device, not
    the current one) and, for an entry point that takes a stream, on that device's current stream, which is appended
    to ``args``.  Tensors are passed as their data pointers, None as NULL.  An ``int`` result is a status code and
    raises through ``check``; any other result (a workspace size, a launch count) is returned."""
    fn = getattr(lib(), name)
    args = [a.data_ptr() if torch.is_tensor(a) else a for a in args]
    with torch.cuda.device(device):
        if name in _TAKES_STREAM:
            args.append(torch.cuda.current_stream(device).cuda_stream)
        r = fn(*args)
    if fn.restype is not _i:
        return r
    check(r, name)


def f32(a):
    """Host fp32 contiguous numpy array + ctypes pointer (keeps the array alive via the tuple)."""
    if torch.is_tensor(a):
        a = a.detach().cpu().numpy()
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(c_f32p)


def i32(a):
    if torch.is_tensor(a):
        a = a.detach().cpu().numpy()
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(c_i32p)


def require_cuda(t, name):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise RuntimeError("smirk_b200: `%s` must be a CUDA tensor — the hot path has no CPU fallback" % name)


def dev_f32(t, name):
    require_cuda(t, name)
    return t.detach().to(torch.float32).contiguous()


def live_handle(module, kind, dev, key, create_args):
    """The live eval handle ``smk_<kind>_live_create(*create_args)`` of ``module``, kept in its NativeState for ``key``
    (topology and precision: an optimizer step builds nothing).  ``generation`` counts its refreshes."""
    st = module._native
    key = (str(dev),) + tuple(key)
    if st.live_handle is None or st.live_key != key:
        st.live_handle = None
        h = C.c_void_p()
        call("smk_%s_live_create" % kind, dev, *create_args, C.byref(h))
        st.live_handle, st.live_key = NativeHandle(h, "smk_%s_destroy" % kind), key
        st.live_handle.generation = 0
    return st.live_handle


def refresh(kind, h, dev, args):
    """``smk_<kind>_refresh(h, &args)`` on the current stream; bumps the handle's generation."""
    call("smk_%s_refresh" % kind, dev, h, C.byref(args))
    h.generation += 1


class NativeHandle:
    """Owner of one ``Smk*`` handle.  Passed to the C ABI like a ``c_void_p`` (``_as_parameter_``); the native
    object is destroyed when the last Python reference goes away.  Modules drop their reference when their weights
    change; a captured CUDA graph (``SmirkPipeline.capture``) keeps its own, so the packed weights a graph points
    at outlive the module's re-pack."""

    def __init__(self, ptr, destroy_name):
        self._as_parameter_ = ptr
        self._destroy_name = destroy_name

    def __del__(self):
        try:
            if self._as_parameter_ is not None and _lib is not None:
                getattr(_lib, self._destroy_name)(self._as_parameter_)
        except Exception:
            pass
        self._as_parameter_ = None


def create(kind, desc, device):
    """``smk_<kind>_create(&desc, &h)`` on ``device`` -> the handle, destroyed by ``smk_<kind>_destroy``."""
    h = C.c_void_p()
    call("smk_%s_create" % kind, device, C.byref(desc), C.byref(h))
    return NativeHandle(h, "smk_%s_destroy" % kind)


def saved_buffer(kind, handle, B, device):
    """A buffer of ``smk_<kind>_saved_bytes`` for the activations of one grad-mode forward (pass ``numel() * 4`` bytes)."""
    nbytes = call("smk_%s_saved_bytes" % kind, device, handle, B)
    return torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=device)


def saved_views(kind, handle, saved, B, *args, int8=()):
    """{name: view of ``saved``} for every tensor ``smk_<kind>_saved_tensor(handle, B, *args, i, ...)`` lays out in it, in
    layout order: [B,C,H,W] views of the NHWC tensors, [B,C] for 1 x 1 ones (the encoder's head outputs, the expression
    loss's features).  ``args``: the losses' ``need``.  The tensors named in ``int8`` are int8, at byte offset 4 * offset."""
    fn = getattr(lib(), "smk_%s_saved_tensor" % kind)
    name, off, dims = C.c_char_p(), C.c_size_t(), (C.c_int * 4)()
    out, i = {}, 0
    while (rc := fn(handle, B, *args, i, C.byref(name), C.byref(off), dims)) == 0:       # non-zero past the last tensor
        b, h, w, c = dims
        key, n = name.value.decode(), b * h * w * c
        t = saved.view(torch.int8)[4 * off.value:4 * off.value + n] if key in int8 else saved[off.value:off.value + n]
        t = t.view(b, h, w, c)
        out[key] = t.view(b, c) if h == w == 1 else t.permute(0, 3, 1, 2)
        i += 1
    if not out:                                 # not even tensor 0: raise with the library's message
        check(rc, "smk_%s_saved_tensor" % kind)
    return out


class Workspace:
    """Per-module scratch owned by the PyTorch caching allocator, grown on demand.  ``get`` never frees the previous
    buffer itself: it only drops this object's reference, so anything that still holds the old tensor (a captured
    CUDA graph's keep-alive list) keeps the memory."""

    def __init__(self):
        self.buf = None

    def get(self, nbytes, device):
        if self.buf is None or self.buf.device != device or self.buf.numel() < nbytes:
            self.buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        return self.buf


def buffers_signature(module, device, *extra):
    """Cheap change detector for a module's parameters / buffers: versions + storage pointers."""
    s = [str(device)] + list(extra)
    for t in list(module.parameters()) + list(module.buffers()):
        s.append(t._version)
        s.append(t.data_ptr())
    return tuple(s)


class NativeState:
    """Everything native one module owns: the handle and the key it was created for, named workspaces, and tensors
    the module keeps per device."""

    def __init__(self):
        self.handle, self.key, self.workspaces, self.per_device = None, None, {}, {}
        self.train_handle, self.train_key = None, None        # the train-mode handle (topology only) of the encoder or generator
        self.live_handle, self.live_key = None, None          # the live eval handle (weights refreshed on the device per call)


class NativeModule:
    """Base of every module that wraps a native handle.  A subclass implements ``_native_create(device)`` (build the
    descriptor, return ``create(...)``); the handle is created lazily and again whenever ``_native_key(device)``
    changes.  All of it lives in one ``NativeState``, which a deep copy does not share."""

    @property
    def _native(self):
        st = self.__dict__.get("_native_state")
        if st is None:
            st = self.__dict__["_native_state"] = NativeState()
        return st

    def _native_key(self, device):
        return buffers_signature(self, device, *self._native_extras())

    def _native_extras(self):
        """Settings besides the parameters and buffers that the handle is packed for."""
        return ()

    def _native_create(self, device):
        raise NotImplementedError

    def _native_handle(self, device):
        st, key = self._native, self._native_key(device)
        if st.handle is None or st.key != key:
            st.handle = None                   # the native object dies with its last reference (NativeHandle)
            st.handle, st.key = self._native_create(device), key
        return st.handle

    def _native_workspace(self, name, nbytes, device):
        return self._native.workspaces.setdefault(name, Workspace()).get(nbytes, device)

    def graph_keep_alive(self):
        """What a CUDA graph captured over this module must keep alive: the handle (packed weights) and the forward
        workspace it was recorded with."""
        ws = self._native.workspaces.get("forward")
        h = self._native.live_handle if self.__dict__.get("_live") else self._native.handle
        return h, ws.buf if ws is not None else None

    def __deepcopy__(self, memo):
        """Same parameter and buffer values; the copy builds its own native state on first use."""
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k != "_native_state":
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new


class FrozenNet(NativeModule):
    """Base of the trainer's frozen networks (VGGPerceptualLoss, MICA, ExpressionLoss): the handle ``smk_<_kind>_create``
    builds from ``_native_tensors()`` at ``precision`` (0 = fp32 CUDA cores, 1 = TF32 tensor cores, 3 = 3xTF32 tensor
    cores), and the check that the module runs as the trainer runs it.  A subclass sets ``_kind``, ``_name`` (the class in
    messages) and ``_net`` (what the trainer calls the network, in messages)."""

    def _native_extras(self):
        return (self.precision,)

    def _native_tensors(self):
        """The tensors the handle is built from: the state_dict in its order, without num_batches_tracked."""
        return [t for k, t in self.state_dict().items() if not k.endswith("num_batches_tracked")]

    def _native_create(self, device):
        if self.precision not in (0, 1, 3):
            raise RuntimeError("smirk_b200.%s: precision must be 0 (fp32), 1 (TF32) or 3 (3xTF32), got %r" % (self._name, self.precision))
        host = [f32(t) for t in self._native_tensors()]
        arr = (c_f32p * len(host))(*[p for _, p in host])
        d = SmkNetDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(c_f32p)), len(host), self.precision
        return create(self._kind, d, device)

    def _saved_views(self, h, saved, B, need):
        """{name: view of ``saved``} for the buffer of a grad-mode forward with ``need`` (the two losses with an input
        gradient; their int8 tensors are named in ``_int8``)."""
        return saved_views(self._kind, h, saved, B, need, int8=self._int8)

    def _check_frozen(self):
        """BatchNorm runs in eval mode only, and weight gradients are not implemented."""
        if any(m.training for m in self.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)):
            raise RuntimeError("smirk_b200.%s: BatchNorm in train mode is not implemented (the trainer runs %s in eval mode); "
                               "call .eval() on the module" % (self._name, self._net))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("smirk_b200.%s: weight gradients are not implemented (the trainer freezes %s); set "
                               "requires_grad=False on its parameters or run it under torch.no_grad()" % (self._name, self._net))


def check_image_pair(m, a, b):
    """The inputs of a loss of two [B,3,224,224] images on one device (``m._inputs`` names them; ``m._why_224`` says why
    only 224x224 is implemented)."""
    for name, t in zip(m._inputs, (a, b)):
        require_cuda(t, name)
        if t.dim() != 4 or tuple(t.shape[1:]) != (3, 224, 224) or t.shape[0] < 1:
            raise RuntimeError("smirk_b200.%s: expected %s [B,3,224,224], got %s — %s" % (m._name, name, tuple(t.shape), m._why_224))
    if a.shape[0] != b.shape[0] or a.device != b.device:
        raise RuntimeError("smirk_b200.%s: %s and %s must have the same batch size and device, got %s on %s and %s on %s"
                           % ((m._name,) + tuple(m._inputs) + (tuple(a.shape), a.device, tuple(b.shape), b.device)))


def pair_forward_saved(m, a, b, opts, need, loss_shape):
    """-> (handle, loss, saved): the grad-mode forward ``smk_<m._kind>_forward_saved(h, a, b, B, *opts, need, loss, saved,
    ...)`` of a two-image loss for the inputs ``need`` names (1 a, 2 b, 3 both); ``opts``: the loss's int options."""
    dev, kind = a.device, m._kind
    h = m._native_handle(dev)
    a, b = dev_f32(a, m._inputs[0]), dev_f32(b, m._inputs[1])
    B = a.shape[0]
    loss = torch.empty(loss_shape, dtype=torch.float32, device=dev)
    nbytes = call("smk_%s_saved_bytes" % kind, dev, h, B, need)
    saved = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
    ws = m._native_workspace("forward", call("smk_%s_workspace_bytes" % kind, dev, h, B), dev)
    call("smk_%s_forward_saved" % kind, dev, h, a, b, B, *opts, need, loss, saved, saved.numel() * 4, ws, ws.numel())
    return h, loss, saved


class PairLossFunction(torch.autograd.Function):
    """loss = m(a, b) of a frozen two-image loss (VGG's x / y, the expression loss's gen / tar), and its gradient to
    whichever of a and b requires grad, through ``pair_forward_saved`` and ``smk_<m._kind>_backward(h, B, *opts, need,
    saved, ...)``."""

    @staticmethod
    def forward(ctx, a, b, m, opts, loss_shape):
        need = (1 if ctx.needs_input_grad[0] else 0) | (2 if ctx.needs_input_grad[1] else 0)
        h, loss, saved = pair_forward_saved(m, a, b, opts, need, loss_shape)
        ctx.handle, ctx.m, ctx.opts, ctx.need, ctx.B, ctx.dtypes = h, m, opts, need, a.shape[0], (a.dtype, b.dtype)
        ctx.save_for_backward(saved)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        saved, = ctx.saved_tensors
        m, dev, B, need = ctx.m, saved.device, ctx.B, ctx.need
        g = dev_f32(g, "g")
        ga = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 1 else None
        gb = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 2 else None
        ws = m._native_workspace("backward", call("smk_%s_backward_workspace_bytes" % m._kind, dev, ctx.handle, B, need), dev)
        call("smk_%s_backward" % m._kind, dev, ctx.handle, B, *ctx.opts, need, saved, saved.numel() * 4, g, ga, gb, ws, ws.numel())
        return (ga.to(ctx.dtypes[0]) if ga is not None else None, gb.to(ctx.dtypes[1]) if gb is not None else None, None, None, None)


def profiler_report():
    """-> {tag: dict(launches, ms, bytes, flops)} accumulated since the last reset."""
    buf = C.create_string_buffer(1 << 16)
    n = lib().smk_profiler_report(buf, len(buf))
    if n < 0:
        raise RuntimeError("smirk_b200: profiler report buffer too small")
    out = {}
    for ln in buf.value.decode().splitlines():
        tag, launches, ms, by, fl = ln.split()
        out[tag] = dict(launches=int(launches), ms=float(ms), bytes=float(by), flops=float(fl))
    return out
