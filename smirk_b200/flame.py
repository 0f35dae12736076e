"""``FLAME`` — drop-in for the reference class ``src/FLAME/FLAME.py:44-315``.

Same constructor arguments, buffer names (so ``state_dict`` keys match), ``forward`` signature and
output dict; the arithmetic runs in ``csrc/flame.cu`` through ``smk_flame_forward``.  When grad mode is
on and a parameter requires grad, ``forward`` is differentiable for shape, expression, pose, jaw, neck,
eye pose and eyelid parameters (``smk_flame_backward``); otherwise it is the plain forward.
"""
import pickle
import sys
import types

import numpy as np
import torch
import torch.nn as nn

from . import _lib


def _to_np(a, dtype=np.float32):
    if "scipy.sparse" in str(type(a)):
        a = a.todense()
    if hasattr(a, "r") and not isinstance(a, np.ndarray):      # chumpy array: .r is the value
        a = a.r
    return np.array(a, dtype=dtype)


def _load_flame_pickle(path):
    """The real generic_model.pkl pickles chumpy objects (FLAME.py:54-56); load it without chumpy by
    substituting a minimal stand-in class that only restores the stored value."""
    try:
        with open(path, "rb") as fh:
            return pickle.load(fh, encoding="latin1")
    except ModuleNotFoundError as e:
        if "chumpy" not in str(e):
            raise

    class _Ch:
        def __setstate__(self, st):
            self.__dict__.update(st if isinstance(st, dict) else {})

        @property
        def r(self):
            return np.asarray(self.__dict__.get("x"))

    mods = {}
    for name in ("chumpy", "chumpy.ch", "chumpy.reordering", "chumpy.utils", "chumpy.logic"):
        m = types.ModuleType(name)
        m.Ch = _Ch
        m.__getattr__ = lambda attr, _c=_Ch: _c          # any class name resolves to the stand-in
        mods[name] = m
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        with open(path, "rb") as fh:
            return pickle.load(fh, encoding="latin1")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


class FLAME(_lib.NativeModule, nn.Module):
    def __init__(self, flame_model_path="assets/FLAME2020/generic_model.pkl",
                 flame_lmk_embedding_path="assets/landmark_embedding.npy", n_shape=300, n_exp=50):
        super().__init__()
        m = _load_flame_pickle(flame_model_path)
        self.n_shape, self.n_exp, self.dtype = n_shape, n_exp, torch.float32
        t = lambda a, dt=torch.float32: torch.tensor(a, dtype=dt)
        self.register_buffer("faces_tensor", t(_to_np(m["f"], np.int64), torch.long))
        self.register_buffer("v_template", t(_to_np(m["v_template"])))
        sd = t(_to_np(m["shapedirs"]))
        self.register_buffer("shapedirs", torch.cat([sd[:, :, :n_shape], sd[:, :, 300:300 + n_exp]], 2))
        pd = _to_np(m["posedirs"])
        self.register_buffer("posedirs", t(np.reshape(pd, [-1, pd.shape[-1]]).T.copy()))
        self.register_buffer("J_regressor", t(_to_np(m["J_regressor"])))
        parents = t(_to_np(m["kintree_table"])[0]).long()
        parents[0] = -1
        self.register_buffer("parents", parents)
        self.register_buffer("lbs_weights", t(_to_np(m["weights"])))
        self.register_buffer("l_eyelid", torch.from_numpy(np.load("assets/l_eyelid.npy")).to(self.dtype)[None])
        self.register_buffer("r_eyelid", torch.from_numpy(np.load("assets/r_eyelid.npy")).to(self.dtype)[None])
        self.register_parameter("eye_pose", nn.Parameter(torch.zeros(1, 6), requires_grad=False))
        self.register_parameter("neck_pose", nn.Parameter(torch.zeros(1, 3), requires_grad=False))
        e = np.load(flame_lmk_embedding_path, allow_pickle=True, encoding="latin1")[()]
        tt = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
        self.register_buffer("lmk_faces_idx", tt(e["static_lmk_faces_idx"]).long())
        self.register_buffer("lmk_bary_coords", tt(e["static_lmk_bary_coords"]).to(self.dtype))
        self.register_buffer("dynamic_lmk_faces_idx", tt(e["dynamic_lmk_faces_idx"]).long())
        self.register_buffer("dynamic_lmk_bary_coords", tt(e["dynamic_lmk_bary_coords"]).to(self.dtype))
        self.register_buffer("full_lmk_faces_idx", tt(e["full_lmk_faces_idx"]).long())
        self.register_buffer("full_lmk_bary_coords", tt(e["full_lmk_bary_coords"]).to(self.dtype))
        chain, cur = [], 1
        while cur != -1:
            chain.append(cur)
            cur = int(self.parents[cur])
        self.register_buffer("neck_kin_chain", torch.tensor(chain, dtype=torch.long))
        mp = np.load("assets/mediapipe_landmark_embedding/mediapipe_landmark_embedding.npz")
        self.register_buffer("mp_lmk_faces_idx", torch.from_numpy(mp["lmk_face_idx"].astype("int32")).long())
        self.register_buffer("mp_lmk_bary_coords", torch.from_numpy(mp["lmk_b_coords"]).to(self.dtype))
        if self.parents.tolist() != [-1, 0, 1, 1, 1]:
            raise RuntimeError("smirk_b200.FLAME: unsupported kinematic tree %s" % self.parents.tolist())

    # -- native handle (re-packed when a buffer is replaced / edited in place / moved) ---------------
    def _native_create(self, device):
        keep = []

        def F(x):
            a, p = _lib.f32(x); keep.append(a); return p

        def I(x):
            a, p = _lib.i32(x); keep.append(a); return p

        d = _lib.SmkFlameDesc()
        d.n_verts, d.n_faces = self.v_template.shape[0], self.faces_tensor.shape[0]
        d.n_betas, d.n_joints = self.shapedirs.shape[2], self.J_regressor.shape[0]
        d.v_template, d.shapedirs, d.posedirs = F(self.v_template), F(self.shapedirs), F(self.posedirs)
        d.J_regressor, d.lbs_weights = F(self.J_regressor), F(self.lbs_weights)
        d.l_eyelid, d.r_eyelid, d.faces = F(self.l_eyelid[0]), F(self.r_eyelid[0]), I(self.faces_tensor)
        d.n_static, d.static_faces, d.static_bary = self.lmk_faces_idx.numel(), I(self.lmk_faces_idx), F(self.lmk_bary_coords)
        d.n_dyn_rows, d.n_dyn = self.dynamic_lmk_faces_idx.shape
        d.dyn_faces, d.dyn_bary = I(self.dynamic_lmk_faces_idx), F(self.dynamic_lmk_bary_coords)
        d.n_full, d.full_faces, d.full_bary = self.full_lmk_faces_idx.numel(), I(self.full_lmk_faces_idx), F(self.full_lmk_bary_coords)
        d.n_mp, d.mp_faces, d.mp_bary = self.mp_lmk_faces_idx.numel(), I(self.mp_lmk_faces_idx), F(self.mp_lmk_bary_coords)
        return _lib.create("flame", d, device)

    # -- forward --------------------------------------------------------------------------------------
    @torch.no_grad()
    def run_lbs(self, betas, full_pose, eyelid=None):
        """betas [B,350], full_pose [B,15], eyelid [B,2]|None -> dict incl. joints and LUT row."""
        dev = betas.device
        _lib.require_cuda(betas, "betas")
        h = self._native_handle(dev)
        B = betas.shape[0]
        betas, full_pose = _lib.dev_f32(betas, "betas"), _lib.dev_f32(full_pose, "full_pose")
        eyelid = _lib.dev_f32(eyelid, "eyelid_params") if eyelid is not None else None
        V = self.v_template.shape[0]
        o = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        verts, fan, fan3d, mp = o(B, V, 3), o(B, 68, 3), o(B, self.full_lmk_faces_idx.numel(), 3), o(B, self.mp_lmk_faces_idx.numel(), 3)
        joints = o(B, 5, 3)
        dyn = torch.empty(B, dtype=torch.int32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_flame_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_flame_forward", dev, h, betas, full_pose, eyelid, B, verts, fan, fan3d, mp, joints, dyn, ws, ws.numel())
        return {"vertices": verts, "landmarks_fan": fan, "landmarks_fan_3d": fan3d, "landmarks_mp": mp,
                "joints": joints, "dyn_idx": dyn}

    def forward(self, param_dictionary, zero_expression=False, zero_shape=False, zero_pose=False):
        shape_params = param_dictionary["shape_params"]
        expression_params = param_dictionary["expression_params"]
        pose_params = param_dictionary.get("pose_params", None)
        jaw_params = param_dictionary.get("jaw_params", None)
        eye_pose_params = param_dictionary.get("eye_pose_params", None)
        neck_pose_params = param_dictionary.get("neck_pose_params", None)
        eyelid_params = param_dictionary.get("eyelid_params", None)
        _lib.require_cuda(shape_params, "shape_params")
        B, dev = shape_params.shape[0], shape_params.device
        z = lambda n: torch.zeros(B, n, dtype=torch.float32, device=dev)
        if expression_params.shape[1] < self.n_exp:                                   # FLAME.py:244-248
            expression_params = torch.cat([expression_params, z(self.n_exp - expression_params.shape[1])], 1)
        if shape_params.shape[1] < self.n_shape:
            shape_params = torch.cat([shape_params, z(self.n_shape - shape_params.shape[1])], 1)
        if zero_expression:                                                           # FLAME.py:251-253
            expression_params, jaw_params = torch.zeros_like(expression_params), torch.zeros_like(jaw_params)
        if zero_shape:
            shape_params = torch.zeros_like(shape_params)
        if zero_pose:                                                                 # FLAME.py:259-262
            pose_params = torch.zeros_like(pose_params)
            pose_params[..., 0], pose_params[..., 1] = 0.2, -0.7
        if pose_params is None:
            # the reference dereferences a non-existent self.pose_params here (FLAME.py:265)
            raise AttributeError("'FLAME' object has no attribute 'pose_params'")
        if eye_pose_params is None:
            eye_pose_params = self.eye_pose.expand(B, -1)
        if neck_pose_params is None:
            neck_pose_params = self.neck_pose.expand(B, -1)
        betas = torch.cat([shape_params, expression_params], 1)
        full_pose = torch.cat([pose_params, neck_pose_params.to(dev), jaw_params, eye_pose_params.to(dev)], 1)
        keys = ("vertices", "landmarks_fan", "landmarks_fan_3d", "landmarks_mp")
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (betas, full_pose, eyelid_params)):
            return dict(zip(keys, _FlameFunction.apply(self, betas, full_pose, eyelid_params)))
        r = self.run_lbs(betas, full_pose, eyelid_params)
        return {k: r[k] for k in keys}


class _FlameFunction(torch.autograd.Function):
    """betas, full_pose, eyelid -> (vertices, landmarks_fan, landmarks_fan_3d, landmarks_mp); the backward is
    ``smk_flame_backward``.  Concatenation, zero padding and the ``zero_*`` switches stay in torch autograd."""

    @staticmethod
    def forward(ctx, module, betas, full_pose, eyelid):
        r = module.run_lbs(betas, full_pose, eyelid)
        ctx.module, ctx.has_eyelid = module, eyelid is not None
        ctx.dtypes = (betas.dtype, full_pose.dtype, eyelid.dtype if eyelid is not None else None)
        ctx.save_for_backward(_lib.dev_f32(betas, "betas"), _lib.dev_f32(full_pose, "full_pose"), r["dyn_idx"])
        return r["vertices"], r["landmarks_fan"], r["landmarks_fan_3d"], r["landmarks_mp"]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_verts, g_fan, g_fan3d, g_mp):
        betas, full_pose, dyn = ctx.saved_tensors
        m, dev, B = ctx.module, betas.device, betas.shape[0]
        h = m._native_handle(dev)
        gs = [None if g is None else g.to(torch.float32).contiguous() for g in (g_verts, g_fan, g_fan3d, g_mp)]
        g_betas = torch.empty_like(betas)
        g_pose = torch.empty_like(full_pose)
        g_eyelid = torch.empty(B, 2, dtype=torch.float32, device=dev) if ctx.has_eyelid else None
        ws = m._native_workspace("backward", _lib.call("smk_flame_backward_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_flame_backward", dev, h, betas, full_pose, None, B, dyn, *gs, g_betas, g_pose, g_eyelid, ws, ws.numel())
        return (None, g_betas.to(ctx.dtypes[0]), g_pose.to(ctx.dtypes[1]),
                g_eyelid.to(ctx.dtypes[2]) if g_eyelid is not None else None)
