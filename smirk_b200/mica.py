"""``MICA`` — drop-in for the reference ``src/models/MICA/mica.py``, the frozen face-shape network behind the pretraining
step's ``mica_loss``.

Same module tree and ``state_dict`` keys (``arcface.*``: an ArcFace iResNet-100 with ``IBasicBlock`` layers (3, 13, 30, 3);
``regressor.*``: ``MappingNetwork(512, 300, 300, hidden=3)``), with plain ``nn`` containers whose own ``forward`` is never
called: the network runs in ``csrc/mica.cu`` through ``smk_mica_forward`` (include/smirk_b200_mica.h).

- ``MICA()`` loads ``assets/mica.tar`` relative to the current directory as the reference does: ``checkpoint['arcface']``
  strictly, and from ``checkpoint['flameModel']`` the keys that contain ``network`` or ``output``, ``regressor.`` stripped.
  ``MICA(checkpoint=None)`` gives untrained containers for ``load_state_dict``.
- ``forward(images)`` -> ``{'shape_params': [B,300]}`` for images [B,3,112,112] in [0, 1]; the result never requires grad.
- ``calculate_mica_shape_loss(shape_params, img)``: ``F.mse_loss(shape_params, mica_shape)`` with the reference's warning
  and truncation when D < 300, forward and gradient to ``shape_params`` in CUDA (deterministic, no atomics).

The network is frozen: BatchNorm runs in eval mode only (a module in train mode raises), and in grad mode a parameter
that requires grad raises, since weight gradients are not implemented.  ``precision`` (part of the native handle's key):
0 = fp32 CUDA cores, 1 = TF32 tensor cores, 3 = 3xTF32 tensor cores (fp32-equivalent), as for ``VGGPerceptualLoss``.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

_LAYERS = (3, 13, 30, 3)
_PLANES = (64, 128, 256, 512)


def _bn(c):
    return nn.BatchNorm2d(c, eps=1e-05)


def _conv3(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, kernel_size=3, stride=stride, padding=1, bias=False)


class IBasicBlock(nn.Module):
    """Container with the reference block's parameters: bn1, conv1, bn2, prelu, conv2 (stride), bn3[, downsample]."""

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.bn1, self.conv1, self.bn2 = _bn(inplanes), _conv3(inplanes, planes), _bn(planes)
        self.prelu = nn.PReLU(planes)
        self.conv2, self.bn3 = _conv3(planes, planes, stride), _bn(planes)
        self.downsample = downsample
        self.stride = stride


class Arcface(nn.Module):
    """Container with the reference ``Arcface`` (``IResNet(IBasicBlock, [3, 13, 30, 3])``) parameters, with the layers the
    reference's ``freezer`` freezes at requires_grad=False."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1, self.prelu = _bn(64), nn.PReLU(64)
        inplanes = 64
        for i, (n, planes) in enumerate(zip(_LAYERS, _PLANES)):
            ds = nn.Sequential(nn.Conv2d(inplanes, planes, kernel_size=1, stride=2, bias=False), _bn(planes))
            blocks = [IBasicBlock(inplanes, planes, 2, ds)] + [IBasicBlock(planes, planes) for _ in range(1, n)]
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*blocks))
            inplanes = planes
        self.bn2 = _bn(512)
        self.dropout = nn.Dropout(p=0, inplace=True)
        self.fc = nn.Linear(512 * 49, 512)
        self.features = nn.BatchNorm1d(512, eps=1e-05)
        for m in (self.layer1, self.layer2, self.layer3, self.conv1, self.bn1, self.prelu):
            for p in m.parameters():
                p.requires_grad = False


class MappingNetwork(nn.Module):
    """Container with the reference ``MappingNetwork(512, 300, 300, hidden=3)`` parameters (no skips at hidden <= 5)."""

    def __init__(self, z_dim=512, hidden_dim=300, out_dim=300, hidden=3):
        super().__init__()
        self.network = nn.ModuleList([nn.Linear(z_dim, hidden_dim)] + [nn.Linear(hidden_dim, hidden_dim) for _ in range(hidden)])
        self.output = nn.Linear(hidden_dim, out_dim)


class MICA(_lib.NativeModule, nn.Module):
    def __init__(self, checkpoint="assets/mica.tar"):
        """``checkpoint``: the path the reference loads (relative to the current directory), or None: untrained
        containers for ``load_state_dict``."""
        super().__init__()
        self.arcface = Arcface()
        self.regressor = MappingNetwork(512, 300, 300, hidden=3)
        self.precision = 0
        if checkpoint is not None:
            ck = torch.load(checkpoint)
            self.arcface.load_state_dict(ck["arcface"], strict=True)
            keys = {k.replace("regressor.", ""): v for k, v in ck["flameModel"].items() if "network" in k or "output" in k}
            self.regressor.load_state_dict(keys, strict=True)

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        if self.precision not in (0, 1, 3):
            raise RuntimeError("smirk_b200.MICA: precision must be 0 (fp32), 1 (TF32) or 3 (3xTF32), got %r" % (self.precision,))
        keep = []
        ts = [t for k, t in self.state_dict().items() if not k.endswith("num_batches_tracked")]
        arr = (_lib.c_f32p * len(ts))()
        for j, t in enumerate(ts):
            a, p = _lib.f32(t)
            keep.append(a)
            arr[j] = p
        d = _lib.SmkMicaDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), len(ts), self.precision
        return _lib.create("mica", d, device)

    def _check(self, images):
        if any(m.training for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)):
            raise RuntimeError("smirk_b200.MICA: BatchNorm in train mode is not implemented (the trainer runs MICA in eval "
                               "mode); call .eval() on the module")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("smirk_b200.MICA: weight gradients are not implemented (the trainer freezes MICA); set "
                               "requires_grad=False on its parameters or run it under torch.no_grad()")
        _lib.require_cuda(images, "images")
        if images.dim() != 4 or tuple(images.shape[1:]) != (3, 112, 112) or images.shape[0] < 1:
            raise RuntimeError("smirk_b200.MICA: expected images [B,3,112,112] (the 112x112 ArcFace crops), got %s"
                               % (tuple(images.shape),))

    @torch.no_grad()
    def _run(self, images):
        """-> (shape_params [B,300], arcface features before F.normalize [B,512]); the caller has run ``_check``."""
        dev = images.device
        h = self._native_handle(dev)
        x = _lib.dev_f32(images, "images")
        B = x.shape[0]
        out = torch.empty(B, 300, dtype=torch.float32, device=dev)
        feat = torch.empty(B, 512, dtype=torch.float32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_mica_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_mica_forward", dev, h, x, B, out, feat, ws, ws.numel())
        return out, feat

    def forward(self, images):
        self._check(images)
        return {"shape_params": self._run(images)[0]}

    def arcface_features(self, images):
        """The ArcFace embedding [B,512] the regressor normalises (``self.arcface(images')`` in the reference)."""
        self._check(images)
        return self._run(images)[1]

    def calculate_mica_shape_loss(self, shape_params, img):
        """Runs MICA on the input image and returns the L2 loss between ``shape_params`` and MICA's shape_params."""
        B, D = shape_params.size()
        with torch.no_grad():
            mica_shape = self.forward(img.reshape(-1, 3, 112, 112))["shape_params"]
        if mica_shape.size(-1) > D:
            print(f"Warning: MICA output has more dimensions ({mica_shape.size(-1)}) than the input shape_params ({D}). "
                  f"Truncating the MICA output to {D} dimensions.")
        if mica_shape.shape[0] != B or D > mica_shape.size(-1):
            raise RuntimeError("smirk_b200.MICA: shape_params %s does not match MICA's output %s"
                               % (tuple(shape_params.shape), tuple(mica_shape.shape)))
        return _ShapeLoss.apply(shape_params, mica_shape, D)


class _ShapeLoss(torch.autograd.Function):
    """mse_loss(shape_params, mica_shape[:, :D]) and its gradient to shape_params; mica_shape is a constant."""

    @staticmethod
    def forward(ctx, s, m, D):
        _lib.require_cuda(s, "shape_params")
        dev = s.device
        sf = _lib.dev_f32(s, "shape_params")
        B = sf.shape[0]
        loss = torch.empty((), dtype=torch.float32, device=dev)
        _lib.call("smk_mica_shape_loss_forward", dev, sf, m, B, D, m.shape[1], loss)
        ctx.save_for_backward(sf, m)
        ctx.D, ctx.dtype = D, s.dtype
        return loss.to(s.dtype)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        sf, m = ctx.saved_tensors
        dev, B = sf.device, sf.shape[0]
        g = _lib.dev_f32(g, "g")
        grad = torch.empty(B, ctx.D, dtype=torch.float32, device=dev)
        _lib.call("smk_mica_shape_loss_backward", dev, sf, m, B, ctx.D, m.shape[1], g, grad)
        return grad.to(ctx.dtype), None, None
