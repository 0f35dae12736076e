"""``SmirkEncoder`` — drop-in for the reference ``src/smirk_encoder.py`` (eval BN).

Same class names, constructor arguments, sub-module / parameter names (``state_dict`` keys follow the
timm ``features_only`` MobileNetV3 layout the reference checkpoints use) and output dicts.  The
``nn.Conv2d`` / ``nn.BatchNorm2d`` objects below are parameter containers only — they are never
called; the forward pass runs in ``csrc/encoder.cu`` through ``smk_encoder_forward``.

With grad mode on and an image that requires grad, a frozen (``requires_grad_(False)``) encoder whose BatchNorms are in
eval mode passes the gradient to its input, as the reference trainer's cycle loss (its encoder frozen by
``utils.freeze_module``) and analysis-by-synthesis fitting need: the forward then keeps its activations
(``smk_encoder_forward_saved``) and the backward runs ``smk_encoder_backward``.  Weight gradients are not implemented.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

BN_EPS = 1e-3          # timm tf_* models (BN_EPS_TF_DEFAULT)

# (kind, stride, expansion, out_channels) per block, grouped per stage — timm 0.9.16
# tf_mobilenetv3_{large,small}_minimal_100 with features_only=True (stops after the `cn` stage).
ARCH = {
    "tf_mobilenetv3_large_minimal_100": [
        [("ds", 1, 1.0, 16)],
        [("ir", 2, 4.0, 24), ("ir", 1, 3.0, 24)],
        [("ir", 2, 3.0, 40), ("ir", 1, 3.0, 40), ("ir", 1, 3.0, 40)],
        [("ir", 2, 6.0, 80), ("ir", 1, 2.5, 80), ("ir", 1, 2.3, 80), ("ir", 1, 2.3, 80)],
        [("ir", 1, 6.0, 112), ("ir", 1, 6.0, 112)],
        [("ir", 2, 6.0, 160), ("ir", 1, 6.0, 160), ("ir", 1, 6.0, 160)],
        [("cn", 1, 1.0, 960)],
    ],
    "tf_mobilenetv3_small_minimal_100": [
        [("ds", 2, 1.0, 16)],
        [("ir", 2, 4.5, 24), ("ir", 1, 3.67, 24)],
        [("ir", 2, 4.0, 40), ("ir", 1, 6.0, 40), ("ir", 1, 6.0, 40)],
        [("ir", 1, 3.0, 48), ("ir", 1, 3.0, 48)],
        [("ir", 2, 6.0, 96), ("ir", 1, 6.0, 96), ("ir", 1, 6.0, 96)],
        [("cn", 1, 1.0, 576)],
    ],
}


def _make_divisible(v, divisor=8, round_limit=0.9):
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    if new_v < round_limit * v:
        new_v += divisor
    return new_v


def _conv(cin, cout, k, stride=1, groups=1):
    return nn.Conv2d(cin, cout, k, stride=stride, groups=groups, bias=False)


def _bn(c):
    return nn.BatchNorm2d(c, eps=BN_EPS)


class _Block(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("smirk_b200: backbone blocks are parameter containers; call SmirkEncoder.forward")


class _DS(_Block):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv_dw, self.bn1 = _conv(cin, cin, 3, stride, cin), _bn(cin)
        self.conv_pw, self.bn2 = _conv(cin, cout, 1), _bn(cout)


class _IR(_Block):
    def __init__(self, cin, cout, stride, exp):
        super().__init__()
        mid = _make_divisible(cin * exp)
        self.conv_pw, self.bn1 = _conv(cin, mid, 1), _bn(mid)
        self.conv_dw, self.bn2 = _conv(mid, mid, 3, stride, mid), _bn(mid)
        self.conv_pwl, self.bn3 = _conv(mid, cout, 1), _bn(cout)


class _CN(_Block):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv, self.bn1 = _conv(cin, cout, 1), _bn(cout)


class _Backbone(_Block):
    """Parameter tree of a timm MobileNetV3Features model (conv_stem, bn1, blocks.<stage>.<i>...)."""

    def __init__(self, name):
        super().__init__()
        self.conv_stem, self.bn1 = _conv(3, 16, 3, 2), _bn(16)
        stages, cin = [], 16
        for stage in ARCH[name]:
            blocks = []
            for kind, s, e, c in stage:
                blocks.append(_DS(cin, c, s) if kind == "ds" else _IR(cin, c, s, e) if kind == "ir" else _CN(cin, c))
                cin = c
            stages.append(nn.Sequential(*blocks))
        self.blocks = nn.Sequential(*stages)
        self.feature_dim = cin

    def tensor_list(self):
        """fp32 tensors in state_dict order without num_batches_tracked (the C ABI's contract)."""
        return [v for k, v in self.state_dict().items() if not k.endswith("num_batches_tracked")]


def create_backbone(backbone_name, pretrained=True):
    """Signature of smirk_encoder.py:7-12.  ``pretrained`` is accepted and ignored: there is no network
    access here and the reference always overwrites the weights from its checkpoint (demo.py:55-58)."""
    bb = _Backbone(backbone_name)
    return bb, bb.feature_dim


class _NativeEncoder(_lib.NativeModule, nn.Module):
    """Shared machinery of SmirkEncoder and its three sub-encoders: a native handle over the backbones returned by
    ``_parts()`` (slot 0 = pose / small, 1 = shape / large, 2 = expression / large; None = not part of this module),
    re-packed whenever a parameter / buffer is modified or moved, and the raw forward through the C ABI.

    ``precision``: 0 fp32 CUDA cores | 1 TF32 wgmma 1x1 convs | 2 = 1 + fused expand/depthwise blocks |
    3 = 2 with error-compensated 3xTF32 arithmetic (fp32-equivalent; the parity path)."""

    def _init_native(self, n_exp=50, n_shape=300):
        self.n_exp, self.n_shape = n_exp, n_shape
        self.precision = 0

    def _parts(self):
        raise NotImplementedError

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        keep = []
        d = _lib.SmkEncoderDesc()
        for i, part in enumerate(self._parts()):
            if part is None:
                d.n_tensors[i] = 0
                continue
            enc, head = part
            ts = enc.encoder.tensor_list()
            arr = (_lib.c_f32p * len(ts))()
            for j, t in enumerate(ts):
                a, p = _lib.f32(t)
                keep.append(a)
                arr[j] = p
            keep.append(arr)
            d.tensors[i] = C.cast(arr, C.POINTER(_lib.c_f32p))
            d.n_tensors[i] = len(ts)
            a, p = _lib.f32(head.weight); keep.append(a); d.head_w[i] = p
            a, p = _lib.f32(head.bias); keep.append(a); d.head_b[i] = p
        d.n_shape, d.n_exp, d.precision = self.n_shape, self.n_exp, int(self.precision)
        return _lib.create("encoder", d, device)

    def _check(self, img):
        """Device, shape and mode checks of every call.  The mode is that of the BatchNorms the call runs, as in the
        reference (whose parent module owns none): a parent in train mode over frozen, eval-mode sub-encoders runs."""
        _lib.require_cuda(img, "img")
        for part in self._parts():            # checked on every call: .train() after the first forward must not silently run eval BN
            if part is not None and any(m.training for m in part[0].encoder.modules() if isinstance(m, nn.BatchNorm2d)):
                raise RuntimeError("smirk_b200.%s: train-mode BatchNorm is not implemented (forward/eval only)" % type(self).__name__)
        if img.dim() != 4 or tuple(img.shape[1:]) != (3, 224, 224):
            raise RuntimeError("smirk_b200.%s: expected img [B,3,224,224], got %s" % (type(self).__name__, tuple(img.shape)))

    def _outputs(self, B, dev):
        widths = (6, self.n_shape, self.n_exp + 5)
        return [torch.empty(B, w, dtype=torch.float32, device=dev) if part is not None else None
                for w, part in zip(widths, self._parts())]

    def _run(self, img):
        """img [B,3,224,224] -> (pose_cam [B,6] | None, shape [B,n_shape] | None, expr [B,n_exp+5] | None)."""
        self._check(img)
        if torch.is_grad_enabled() and img.requires_grad:
            parts = [p for p in self._parts() if p is not None]
            if any(t.requires_grad for enc, head in parts for t in list(enc.encoder.parameters()) + list(head.parameters())):
                raise RuntimeError("smirk_b200.%s: weight gradients are not implemented; to pass a gradient to the input, "
                                   "freeze the encoder with .requires_grad_(False)" % type(self).__name__)
            raw = _EncoderFunction.apply(img, self)
            it = iter(raw)
            return [next(it) if p is not None else None for p in self._parts()]
        with torch.no_grad():
            dev = img.device
            h = self._native_handle(dev)
            x = _lib.dev_f32(img, "img")
            B = x.shape[0]
            outs = self._outputs(B, dev)
            ws = self._native_workspace("forward", _lib.call("smk_encoder_workspace_bytes", dev, h, B), dev)
            _lib.call("smk_encoder_forward", dev, h, x, B, *outs, ws, ws.numel())
            return outs

    def _forward_saved(self, img):
        """-> (handle, [raw outputs | None], saved): the grad-mode forward, its activations in a buffer of their own."""
        dev = img.device
        h = self._native_handle(dev)
        x = _lib.dev_f32(img, "img")
        B = x.shape[0]
        outs = self._outputs(B, dev)
        saved = _lib.saved_buffer("encoder", h, B, dev)
        ws = self._native_workspace("forward", _lib.call("smk_encoder_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_encoder_forward_saved", dev, h, x, B, *outs, saved, saved.numel() * 4, ws, ws.numel())
        return h, outs, saved

    @torch.no_grad()
    def saved_activations(self, img):
        """The tensors the backward of ``self(img)`` uses, {name: tensor}, names being the reference's module paths: the
        output of every ReLU as a [B,C,H,W] view of the NHWC buffer (``shape_encoder.encoder.bn1`` for the stem,
        ``….blocks.<stage>.<i>.bn1`` / ``.bn2`` ...) and each head's pre-clamp output [B,n_out]
        (``expression_encoder.expression_layers.0`` ...).  The forward is deterministic and batch-independent, so these
        are the tensors an autograd context of the same input holds."""
        self._check(img)
        h, _, saved = self._forward_saved(img)
        return _lib.saved_views("encoder", h, saved, img.shape[0])


class _EncoderFunction(torch.autograd.Function):
    """Frozen encoder: the raw outputs (pose_cam, shape, expr: those the module holds) of img, and the gradient with
    respect to img only.  An output that receives no gradient arrives as None and its backbone's backward launches
    nothing.  The activations are saved per call, so several forwards may share one backward."""

    @staticmethod
    def forward(ctx, img, module):
        h, outs, saved = module._forward_saved(img)
        ctx.set_materialize_grads(False)
        ctx.handle, ctx.module, ctx.dtype, ctx.B = h, module, img.dtype, img.shape[0]
        ctx.present = [o is not None for o in outs]
        ctx.save_for_backward(saved)
        return tuple(o for o in outs if o is not None)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        saved, = ctx.saved_tensors
        m, dev, B = ctx.module, saved.device, ctx.B
        it = iter(grads)
        g = [next(it) if p else None for p in ctx.present]
        g = [None if t is None else _lib.dev_f32(t, "grad") for t in g]
        g_img = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev)
        ws = m._native_workspace("backward", _lib.call("smk_encoder_backward_workspace_bytes", dev, ctx.handle, B), dev)
        _lib.call("smk_encoder_backward", dev, ctx.handle, B, saved, saved.numel() * 4, *g, g_img, ws, ws.numel())
        return g_img.to(ctx.dtype), None


class PoseEncoder(_NativeEncoder):
    def __init__(self):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_small_minimal_100")
        self.pose_cam_layers = nn.Sequential(nn.Linear(feature_dim, 6))
        self._init_native()
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:26-31
        self.pose_cam_layers[-1].weight.data *= 0.001
        self.pose_cam_layers[-1].bias.data *= 0.001
        self.pose_cam_layers[-1].weight.data[3] = 0
        self.pose_cam_layers[-1].bias.data[3] = 7

    def _parts(self):
        return ((self, self.pose_cam_layers[0]), None, None)

    def forward(self, img):                     # smirk_encoder.py:34-45
        pose_cam = self._run(img)[0]
        return {"pose_params": pose_cam[..., :3], "cam": pose_cam[..., 3:]}


class ShapeEncoder(_NativeEncoder):
    def __init__(self, n_shape=300):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_large_minimal_100")
        self.shape_layers = nn.Sequential(nn.Linear(feature_dim, n_shape))
        self._init_native(n_shape=n_shape)
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:61-63
        self.shape_layers[-1].weight.data *= 0
        self.shape_layers[-1].bias.data *= 0

    def _parts(self):
        return (None, (self, self.shape_layers[0]), None)

    def forward(self, img):                     # smirk_encoder.py:66-73
        return {"shape_params": self._run(img)[1]}


class ExpressionEncoder(_NativeEncoder):
    def __init__(self, n_exp=50):
        super().__init__()
        self.encoder, feature_dim = create_backbone("tf_mobilenetv3_large_minimal_100")
        self.expression_layers = nn.Sequential(nn.Linear(feature_dim, n_exp + 2 + 3))
        self._init_native(n_exp=n_exp)
        self.init_weights()

    def init_weights(self):                     # smirk_encoder.py:90-92
        self.expression_layers[-1].weight.data *= 0.1
        self.expression_layers[-1].bias.data *= 0.1

    def _parts(self):
        return (None, None, (self, self.expression_layers[0]))

    def forward(self, img):                     # smirk_encoder.py:95-110 (clamps applied by the native head kernel)
        expr, ne = self._run(img)[2], self.n_exp
        return {"expression_params": expr[..., :ne], "eyelid_params": expr[..., ne:ne + 2], "jaw_params": expr[..., ne + 2:ne + 5]}


class SmirkEncoder(_NativeEncoder):
    def __init__(self, n_exp=50, n_shape=300):
        super().__init__()
        self.pose_encoder = PoseEncoder()
        self.shape_encoder = ShapeEncoder(n_shape=n_shape)
        self.expression_encoder = ExpressionEncoder(n_exp=n_exp)
        self._init_native(n_exp=n_exp, n_shape=n_shape)

    def _parts(self):
        return ((self.pose_encoder, self.pose_encoder.pose_cam_layers[0]),
                (self.shape_encoder, self.shape_encoder.shape_layers[0]),
                (self.expression_encoder, self.expression_encoder.expression_layers[0]))

    def forward(self, img):                     # smirk_encoder.py:123-133: one native call runs the three backbones concurrently
        pose_cam, shape, expr = self._run(img)
        ne = self.n_exp
        return {
            "pose_params": pose_cam[..., :3], "cam": pose_cam[..., 3:],
            "shape_params": shape,
            "expression_params": expr[..., :ne], "eyelid_params": expr[..., ne:ne + 2],
            "jaw_params": expr[..., ne + 2:ne + 5],
        }
