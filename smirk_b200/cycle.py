"""The cycle path's parameter augmentation of the reference trainer (``src/smirk_trainer.py:189-248``) on the device.

``CycleAugmentation`` takes the encoder's six outputs [B,·] and returns the detached ``flame_feats`` [Ke*B,·] of step2:
pose, cam and shape repeated; expression, jaw and eyelid augmented as the reference does (four random groups: random
expressions, permuted expressions, template injection, zero expression; the jaw and eyelid tweaks).  Every draw is
made on the device by a counter-based generator (Philox4x32-10 keyed by a seed and a call counter in device memory,
``csrc/cycle.cu``), so a call never syncs with the host and replays from a CUDA graph with fresh draws.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

KEYS = ("pose_params", "cam", "shape_params", "expression_params", "jaw_params", "eyelid_params")   # the C ABI's order


class CycleTemplates:
    """Native handle holding the expression templates on one device: fp32 rows plus per-key row offsets."""

    def __init__(self, rows, offsets, n_exp, device):
        r, rp = _lib.f32(rows)
        o, op = _lib.i32(offsets)
        self.handle = _lib.create("cycle", _lib.SmkCycleDesc(len(offsets) - 1, op, rp, int(n_exp)), device)


def group_sizes(R):
    """Sizes of the four groups ``randperm(R)`` is split into (smirk_trainer.py:202); some are empty when R < 4."""
    c = [0, R // 4, 2 * R // 4, 3 * R // 4, R]
    return [c[i + 1] - c[i] for i in range(4)]


class CycleAugmentation(_lib.NativeModule):
    """``templates``: the dict ``src/utils/utils.py:load_templates`` returns (key -> [rows, n] float64 array), in its key
    order.  ``__call__(encoder_output, Ke=1)`` -> the six ``flame_feats`` tensors [Ke*B,·], detached, in
    ``encoder_output``'s key order; ``debug=True`` also returns every draw (``SmkCycleDraws``' fields)."""

    def __init__(self, templates, num_expression=50, use_eyelids=True, seed=0):
        if not templates:
            raise RuntimeError("smirk_b200.CycleAugmentation: no expression templates")
        self.num_expression, self.use_eyelids, self.seed = int(num_expression), bool(use_eyelids), int(seed)
        self.keys = list(templates.keys())
        rows, offsets = [], [0]
        for k in self.keys:
            a = np.asarray(templates[k])
            if a.ndim != 2 or a.shape[0] == 0 or a.shape[1] < self.num_expression:
                raise RuntimeError("smirk_b200.CycleAugmentation: template %r must be [rows, >= %d], got %s" % (k, self.num_expression, a.shape))
            rows.append(a[:, :self.num_expression].astype(np.float32))              # torch.Tensor(ndarray[:n]): fp64 -> fp32
            offsets.append(offsets[-1] + a.shape[0])
        self.rows, self.offsets = np.concatenate(rows, 0), np.asarray(offsets, dtype=np.int32)

    def _native_key(self, device):
        return ()

    def _native_create(self, device):
        return CycleTemplates(self.rows, self.offsets, self.num_expression, device)

    def _rng(self, device):
        per_device = self._native.per_device
        if device not in per_device:
            per_device[device] = torch.tensor([self.seed, 0], dtype=torch.int64, device=device)
        return per_device[device]

    def reseed(self, seed, counter=0):
        self.seed = int(seed)
        for rng in self._native.per_device.values():
            rng.copy_(torch.tensor([self.seed, int(counter)], dtype=torch.int64))

    def graph_keep_alive(self):
        return (self._native.handle,)

    def _draws(self, R, E, De, dev):
        n0, n1, n2, n3 = group_sizes(R)
        i64 = lambda *s: torch.empty(*s, dtype=torch.int64, device=dev)
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        return dict(gids=i64(R), perm1=i64(n1), param_mask=f32(n0, E), jaw_mask=f32(R), randn0a=f32(n0, E), randn0b=f32(n0, E),
                    randn1=f32(n1, E), randn2=f32(n2, E), randn3=f32(n3, E), randn_jaw=f32(R, 3), rand0a=f32(n0, 1), rand0b=f32(n0, 1),
                    rand1a=f32(n1, 1), rand1b=f32(n1, 1), rand2a=f32(n2, 1), rand2b=f32(n2, 1), rand3=f32(n3, 1),
                    rand_eyelid=f32(R, De), rand3_eyelid=f32(n3, De), tmpl_key=i64(n2), tmpl_row=i64(n2))

    @torch.no_grad()
    def forward(self, encoder_output, Ke=1, debug=False):
        missing = [k for k in KEYS if k not in encoder_output]
        if missing:
            raise RuntimeError("smirk_b200.CycleAugmentation: encoder_output lacks %s" % missing)
        ins = [_lib.dev_f32(encoder_output[k], k) for k in KEYS]
        dev, B, Ke = ins[0].device, ins[0].shape[0], int(Ke)
        if Ke < 1 or any(t.dim() != 2 or t.shape[0] != B or t.device != dev for t in ins):
            raise RuntimeError("smirk_b200.CycleAugmentation: expected six [B, n] tensors on one device and Ke >= 1")
        dims = [t.shape[1] for t in ins]
        outs = [torch.empty(Ke * B, d, dtype=torch.float32, device=dev) for d in dims]
        h = self._native_handle(dev)
        draws = self._draws(Ke * B, dims[3], dims[5], dev) if debug else {}
        d = _lib.SmkCycleDraws(*[draws[f].data_ptr() if f in draws and draws[f].numel() else None for f in _lib.SmkCycleDraws.FIELDS])
        _lib.call("smk_cycle_augment", dev, h.handle, (C.c_void_p * 6)(*[t.data_ptr() for t in ins]),
                  (C.c_void_p * 6)(*[t.data_ptr() for t in outs]), (C.c_int * 6)(*dims), B, Ke, int(self.use_eyelids), self._rng(dev),
                  C.byref(d) if debug else None)
        feats = dict(zip(KEYS, outs))
        feats = {k: feats[k] for k in encoder_output if k in feats}
        return (feats, draws) if debug else feats

    __call__ = forward
