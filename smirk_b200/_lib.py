"""ctypes binding of libsmirk_b200.so (the C ABI declared in include/smirk_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the product
path raises.  Build with ``python -m smirk_b200.build`` (or ``__graft_entry__.build()``).
"""
import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmirk_b200.so")
_lib = None

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
                ("faces", c_i32p), ("image_size", C.c_int)]


class SmkEncoderDesc(C.Structure):
    _fields_ = [("tensors", C.POINTER(c_f32p) * 3), ("n_tensors", C.c_int * 3),
                ("head_w", c_f32p * 3), ("head_b", c_f32p * 3),
                ("n_shape", C.c_int), ("n_exp", C.c_int), ("precision", C.c_int)]


class SmkGeneratorDesc(C.Structure):
    _fields_ = [("in_channels", C.c_int), ("out_channels", C.c_int), ("init_features", C.c_int),
                ("res_blocks", C.c_int), ("tensors", C.POINTER(c_f32p)), ("n_tensors", C.c_int),
                ("precision", C.c_int)]


SYMBOLS = ["smk_version", "smk_last_error", "smk_launch_count", "smk_profiler_enable", "smk_profiler_reset",
           "smk_profiler_report",
           "smk_flame_create", "smk_flame_destroy", "smk_flame_workspace_bytes", "smk_flame_forward",
           "smk_renderer_create", "smk_renderer_destroy", "smk_renderer_workspace_bytes", "smk_renderer_forward",
           "smk_project_points",
           "smk_flame_backward_workspace_bytes", "smk_flame_backward", "smk_renderer_backward_workspace_bytes",
           "smk_renderer_backward", "smk_project_points_backward",
           "smk_encoder_create", "smk_encoder_destroy", "smk_encoder_workspace_bytes", "smk_encoder_forward",
           "smk_generator_create", "smk_generator_destroy", "smk_generator_workspace_bytes", "smk_generator_forward",
           "smk_debug_conv_f32", "smk_debug_conv_tc", "smk_debug_reflect_halo", "smk_debug_xdw", "smk_debug_stem_ds", "smk_debug_gemm_tc3x", "smk_debug_xdw3x", "smk_debug_conv3_win",
           "smk_warp_workspace_bytes", "smk_crop_warp", "smk_warp_u8", "smk_f32chw_to_u8hwc",
           "smk_masking_create", "smk_masking_destroy", "smk_masking_workspace_bytes", "smk_masking_face_weights",
           "smk_masking_points", "smk_masking_compose", "smk_masking_forward_workspace_bytes", "smk_masking_forward", "smk_masking_transfer_pixels",
           "smk_peer_alloc", "smk_peer_free", "smk_peer_open", "smk_peer_close", "smk_peer_push",
           "smk_peer_fan_create", "smk_peer_fan_destroy", "smk_peer_fan_push"]


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("smirk_b200: %s not found — build it with `python -m smirk_b200.build` "
                           "(there is no CPU / PyTorch fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.smk_last_error.restype = C.c_char_p
    for name in SYMBOLS:
        fn = getattr(L, name)
        if name.endswith("_workspace_bytes"):
            fn.restype = C.c_size_t
        elif name.endswith("_destroy"):
            fn.restype = None
    vp, i, sz = C.c_void_p, C.c_int, C.c_size_t
    L.smk_launch_count.restype = C.c_ulonglong
    L.smk_profiler_enable.argtypes = [i]
    L.smk_profiler_enable.restype = None
    L.smk_profiler_reset.restype = None
    L.smk_profiler_report.argtypes = [C.c_char_p, sz]
    L.smk_flame_create.argtypes = [C.POINTER(SmkFlameDesc), C.POINTER(vp)]
    L.smk_flame_destroy.argtypes = [vp]
    L.smk_flame_workspace_bytes.argtypes = [vp, i]
    L.smk_flame_forward.argtypes = [vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.smk_renderer_create.argtypes = [C.POINTER(SmkRendererDesc), C.POINTER(vp)]
    L.smk_renderer_destroy.argtypes = [vp]
    L.smk_renderer_workspace_bytes.argtypes = [vp, i]
    L.smk_renderer_forward.argtypes = [vp, vp, vp, i, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.smk_project_points.argtypes = [vp, vp, i, i, vp, vp]
    L.smk_flame_backward_workspace_bytes.argtypes = [vp, i]
    L.smk_flame_backward.argtypes = [vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.smk_renderer_backward_workspace_bytes.argtypes = [vp, i]
    L.smk_renderer_backward.argtypes = [vp, vp, vp, i, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.smk_project_points_backward.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    L.smk_encoder_create.argtypes = [C.POINTER(SmkEncoderDesc), C.POINTER(vp)]
    L.smk_encoder_destroy.argtypes = [vp]
    L.smk_encoder_workspace_bytes.argtypes = [vp, i]
    L.smk_encoder_forward.argtypes = [vp, vp, i, vp, vp, vp, vp, sz, vp]
    L.smk_generator_create.argtypes = [C.POINTER(SmkGeneratorDesc), C.POINTER(vp)]
    L.smk_generator_destroy.argtypes = [vp]
    L.smk_generator_workspace_bytes.argtypes = [vp, i]
    L.smk_generator_forward.argtypes = [vp, vp, i, vp, vp, sz, vp]
    L.smk_debug_conv_f32.argtypes = [vp, i, i, i, i, i, vp, vp, vp, i, i, i, i, vp, i, vp, i, i, vp]
    L.smk_debug_conv_tc.argtypes = [vp, i, i, i, i, i, vp, vp, vp, i, i, i, i, vp, i, i, vp, i, i, vp]
    L.smk_debug_reflect_halo.argtypes = [vp, i, i, i, i, vp]
    L.smk_debug_xdw.argtypes = [vp, i, i, i, i, vp, vp, vp, i, vp, vp, vp, i, i, vp, vp]
    L.smk_masking_create.argtypes = [vp, vp]
    L.smk_masking_destroy.argtypes = [vp]
    L.smk_masking_workspace_bytes.argtypes = [vp, i, i]
    L.smk_masking_face_weights.argtypes = [vp, vp, vp, i, vp, vp, sz, vp]
    L.smk_masking_points.argtypes = [vp, vp, vp, vp, i, i, i, vp, vp]
    L.smk_masking_forward_workspace_bytes.argtypes = [vp, i, i, i]
    L.smk_masking_forward.argtypes = [vp, vp, vp, vp, vp, vp, i, i, i, i, C.c_float, C.c_float, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.smk_masking_compose.argtypes = [vp, vp, vp, vp, vp, i, vp, vp, vp, vp, i, i, i, vp, vp, sz, vp]
    L.smk_masking_transfer_pixels.argtypes = [vp, vp, vp, vp, i, i, i, vp, vp, sz, vp]
    L.smk_peer_alloc.argtypes = [sz, C.POINTER(vp), C.c_char_p]
    L.smk_peer_free.argtypes = [vp]
    L.smk_peer_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.smk_peer_close.argtypes = [vp]
    L.smk_peer_push.argtypes = [vp, vp, sz, vp]
    L.smk_peer_fan_create.argtypes = [i, C.POINTER(vp)]
    L.smk_peer_fan_destroy.argtypes = [vp]
    L.smk_peer_fan_destroy.restype = None
    L.smk_peer_fan_push.argtypes = [vp, C.POINTER(vp), i, vp, sz, vp]
    L.smk_debug_conv3_win.argtypes = [vp, i, i, i, i, i, vp, vp, vp, i, i, vp, i, vp]
    L.smk_debug_gemm_tc3x.argtypes = [vp, i, i, vp, vp, vp, vp, i, i, i, vp, i, vp, i, vp]
    L.smk_debug_xdw3x.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, i, vp, vp, vp, i, vp, vp]
    L.smk_warp_workspace_bytes.argtypes = [i]
    L.smk_warp_workspace_bytes.restype = C.c_size_t
    L.smk_crop_warp.argtypes = [vp, i, i, i, vp, i, i, vp, vp, C.c_size_t, vp]
    L.smk_warp_u8.argtypes = [vp, i, i, i, vp, i, i, vp, vp, C.c_size_t, vp]
    L.smk_f32chw_to_u8hwc.argtypes = [vp, i, i, vp, vp]
    L.smk_debug_stem_ds.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp]
    if L.smk_version() != 100:
        raise RuntimeError("smirk_b200: library/header version mismatch (%d)" % L.smk_version())
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        msg = lib().smk_last_error().decode("utf-8", "replace")
        raise RuntimeError("smirk_b200: %s failed (rc=%d): %s" % (what, rc, msg))


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


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


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
