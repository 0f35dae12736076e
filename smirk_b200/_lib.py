"""ctypes binding of libsmirk_b200.so (the C ABI declared in include/smirk_b200.h, include/smirk_b200_loss.h,
include/smirk_b200_mica.h, include/smirk_b200_expression.h and include/smirk_b200_generator_train.h).

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


class SmkVggLossDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int), ("precision", C.c_int)]


class SmkMicaDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int), ("precision", C.c_int)]


class SmkExpressionLossDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int), ("precision", C.c_int)]


class SmkMaskingDesc(C.Structure):
    _fields_ = [("n_verts", C.c_int), ("n_faces", C.c_int), ("faces", c_i32p)]


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
# The binding table of include/smirk_b200_loss.h (the trainer's losses), in that header's order, by the same rules.
LOSS_BINDINGS = [
    ("smk_vgg_loss_create", _i, [C.POINTER(SmkVggLossDesc), _vpp]),
    ("smk_vgg_loss_destroy", None, [_vp]),
    ("smk_vgg_loss_workspace_bytes", _sz, [_vp, _i]),
    ("smk_vgg_loss_forward", _i, [_vp, _vp, _vp, _i, _vp, _vp, _sz, STREAM]),
    ("smk_vgg_loss_saved_bytes", _sz, [_vp, _i, _i]),
    ("smk_vgg_loss_forward_saved", _i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_vgg_loss_saved_tensor", _i, [_vp, _i, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_vgg_loss_backward_workspace_bytes", _sz, [_vp, _i, _i]),
    ("smk_vgg_loss_backward", _i, [_vp, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _sz, STREAM]),
]
# The binding table of include/smirk_b200_mica.h (MICA and its shape loss), in that header's order, by the same rules.
MICA_BINDINGS = [
    ("smk_mica_create", _i, [C.POINTER(SmkMicaDesc), _vpp]),
    ("smk_mica_destroy", None, [_vp]),
    ("smk_mica_workspace_bytes", _sz, [_vp, _i]),
    ("smk_mica_forward", _i, [_vp, _vp, _i, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_mica_shape_loss_forward", _i, [_vp, _vp, _i, _i, _i, _vp, STREAM]),
    ("smk_mica_shape_loss_backward", _i, [_vp, _vp, _i, _i, _i, _vp, _vp, STREAM]),
]
# The binding table of include/smirk_b200_expression.h (the emotion loss), in that header's order, by the same rules.
EXPRESSION_BINDINGS = [
    ("smk_expression_loss_create", _i, [C.POINTER(SmkExpressionLossDesc), _vpp]),
    ("smk_expression_loss_destroy", None, [_vp]),
    ("smk_expression_loss_workspace_bytes", _sz, [_vp, _i]),
    ("smk_expression_loss_forward", _i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, STREAM]),
    ("smk_expression_loss_saved_bytes", _sz, [_vp, _i, _i]),
    ("smk_expression_loss_forward_saved", _i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_expression_loss_saved_tensor", _i, [_vp, _i, _i, _i, C.POINTER(C.c_char_p), C.POINTER(_sz), C.POINTER(C.c_int)]),
    ("smk_expression_loss_backward_workspace_bytes", _sz, [_vp, _i, _i]),
    ("smk_expression_loss_backward", _i, [_vp, _i, _i, _i, _i, _vp, _sz, _vp, _vp, _vp, _vp, _sz, STREAM]),
]
# The binding table of include/smirk_b200_generator_train.h (the generator's train mode), in that header's order, by the same rules.
GENERATOR_TRAIN_BINDINGS = [
    ("smk_generator_train_create", _i, [_i, _i, _i, _i, _i, _vpp]),
    ("smk_generator_train_workspace_bytes", _sz, [_vp, _i]),
    ("smk_generator_forward_train", _i, [_vp, C.POINTER(SmkGeneratorTrainArgs), _vp, _i, _vp, _vp, _sz, _vp, _sz, STREAM]),
    ("smk_generator_backward_train", _i, [_vp, C.POINTER(SmkGeneratorTrainArgs), _i, _vp, _vp, _sz, _vp, _vp,
                                          C.POINTER(SmkGeneratorTrainGrads), _vp, _sz, STREAM]),
    ("smk_debug_train_conv3_wgrad", _i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _sz, STREAM]),
]
_ALL_BINDINGS = BINDINGS + LOSS_BINDINGS + MICA_BINDINGS + EXPRESSION_BINDINGS + GENERATOR_TRAIN_BINDINGS
_TAKES_STREAM = frozenset(name for name, _, args in _ALL_BINDINGS if args[-1:] == [STREAM])


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("smirk_b200: %s not found — build it with `python -m smirk_b200.build` "
                           "(there is no CPU / PyTorch fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, restype, argtypes in _ALL_BINDINGS:
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


def saved_views(kind, handle, saved, B):
    """{name: view of ``saved``} for every tensor ``smk_<kind>_saved_tensor`` lays out in it, in layout order: [B,C,H,W]
    views of the NHWC tensors, [B,C] for 1 x 1 ones (the encoder's head outputs)."""
    fn = getattr(lib(), "smk_%s_saved_tensor" % kind)
    name, off, dims = C.c_char_p(), C.c_size_t(), (C.c_int * 4)()
    out, i = {}, 0
    while (rc := fn(handle, B, i, C.byref(name), C.byref(off), dims)) == 0:       # non-zero past the last tensor
        b, h, w, c = dims
        t = saved[off.value:off.value + b * h * w * c].view(b, h, w, c)
        out[name.value.decode()] = t.view(b, c) if h == w == 1 else t.permute(0, 3, 1, 2)
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
        return self._native.handle, ws.buf if ws is not None else None

    def __deepcopy__(self, memo):
        """Same parameter and buffer values; the copy builds its own native state on first use."""
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k != "_native_state":
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new


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
