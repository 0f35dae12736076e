"""``ExpressionLoss`` — drop-in for the reference ``src/losses/ExpressionLoss.py``, the trainer's emotion loss.

Same module tree and ``state_dict`` keys (``backbone.*``: EMOCA's ResNet-50 with ``Bottleneck`` layers (3, 4, 6, 3), the
stride of each layer's first block on its 3x3 ``conv2``, and the unused ``fc``), with plain ``nn`` containers whose own
``forward`` is never called: the network runs in ``csrc/expression_loss.cu`` through ``smk_expression_loss_forward``
(include/smirk_b200_expression.h), gen and tar as one batch.

- ``ExpressionLoss()`` loads the reference's checkpoint path relative to the current directory as the reference does:
  ``torch.load(path)['state_dict']`` without ``backbone.fc.*`` and ``linear.*``, ``strict=False``.
  ``ExpressionLoss(checkpoint=None)`` gives untrained containers for ``load_state_dict``.
- ``forward(gen, tar, use_mean=True, metric='l2')``: gen, tar [B,3,224,224] as they are (no normalisation); per face
  ``l2`` = mean of the squared feature difference, ``l1`` = mean of its absolute value, ``cos`` = 1 - cosine similarity;
  the mean over the faces (0-dim) with ``use_mean``, else the per-face vector [B].  With grad mode on and gen and/or tar
  requiring grad, the loss passes its gradient to them (``smk_expression_loss_forward_saved`` keeps what the backward
  needs for the inputs that want one; ``smk_expression_loss_backward`` walks the network back).
- ``features(images)`` -> [B,2048], the reference's ``self.backbone(x).view(B, -1)``.

The network is frozen, as the reference freezes it: BatchNorm runs in eval mode only (a module in train mode raises),
and in grad mode a parameter that requires grad raises, since weight gradients are not implemented.  ``precision`` (part
of the native handle's key): 0 = fp32 CUDA cores, 1 = TF32 tensor cores, 3 = 3xTF32 tensor cores (fp32-equivalent), as
for ``VGGPerceptualLoss``.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

CHECKPOINT = "assets/ResNet50/checkpoints/deca-epoch=01-val_loss_total/dataloader_idx_0=1.27607644.ckpt"
_LAYERS = (3, 4, 6, 3)
_METRICS = {"l2": 0, "l1": 1, "cos": 2}


class Bottleneck(nn.Module):
    """Container with the reference block's parameters, registered in its construction order: conv1, conv2, bn1, bn2,
    conv3, bn3, relu[, downsample].  The stride (of a layer's first block) sits on conv2."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride


class ResNet(nn.Module):
    """Container with the parameters of the reference's ``resnet50(num_classes=100, include_top=False,
    emoca_specific=True)``."""

    def __init__(self, num_classes=100):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        inplanes = 64
        for i, n in enumerate(_LAYERS):
            planes, stride = 64 << i, 1 if i == 0 else 2
            ds = nn.Sequential(nn.Conv2d(inplanes, planes * 4, kernel_size=1, stride=stride, bias=False), nn.BatchNorm2d(planes * 4))
            blocks = [Bottleneck(inplanes, planes, stride, ds)] + [Bottleneck(planes * 4, planes) for _ in range(1, n)]
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*blocks))
            inplanes = planes * 4
        self.avgpool = nn.AvgPool2d(7, stride=1)
        self.fc = nn.Linear(2048, num_classes)


class ExpressionLoss(_lib.NativeModule, nn.Module):
    def __init__(self, checkpoint=CHECKPOINT):
        """``checkpoint``: the path the reference loads (relative to the current directory), or None: untrained
        containers for ``load_state_dict``."""
        super().__init__()
        self.backbone = ResNet(num_classes=100).eval()
        self.precision = 0
        if checkpoint is not None:
            sd = torch.load(checkpoint)["state_dict"]
            for k in ("backbone.fc.weight", "backbone.fc.bias", "linear.weight", "linear.bias"):
                del sd[k]
            self.load_state_dict(sd, strict=False)
        for p in self.parameters():
            p.requires_grad = False

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        if self.precision not in (0, 1, 3):
            raise RuntimeError("smirk_b200.ExpressionLoss: precision must be 0 (fp32), 1 (TF32) or 3 (3xTF32), got %r"
                               % (self.precision,))
        keep = []
        ts = [t for k, t in self.state_dict().items()
              if not k.endswith("num_batches_tracked") and not k.startswith("backbone.fc.")]
        arr = (_lib.c_f32p * len(ts))()
        for j, t in enumerate(ts):
            a, p = _lib.f32(t)
            keep.append(a)
            arr[j] = p
        d = _lib.SmkExpressionLossDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), len(ts), self.precision
        return _lib.create("expression_loss", d, device)

    def _check_module(self):
        if any(m.training for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)):
            raise RuntimeError("smirk_b200.ExpressionLoss: BatchNorm in train mode is not implemented (the trainer runs the "
                               "emotion network in eval mode); call .eval() on the module")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("smirk_b200.ExpressionLoss: weight gradients are not implemented (the trainer freezes the "
                               "emotion network); set requires_grad=False on its parameters or run it under torch.no_grad()")
        if self.precision not in (0, 1, 3):
            raise RuntimeError("smirk_b200.ExpressionLoss: precision must be 0 (fp32), 1 (TF32) or 3 (3xTF32), got %r"
                               % (self.precision,))

    @staticmethod
    def _check_images(t, name):
        _lib.require_cuda(t, name)
        if t.dim() != 4 or tuple(t.shape[1:]) != (3, 224, 224) or t.shape[0] < 1:
            raise RuntimeError("smirk_b200.ExpressionLoss: expected %s [B,3,224,224], got %s — the backbone's 7x7 average "
                               "pool gives one 2048-d feature per image only at 224x224, the one size implemented"
                               % (name, tuple(t.shape)))

    def _check_inputs(self, gen, tar):
        self._check_module()
        self._check_images(gen, "gen")
        self._check_images(tar, "tar")
        if gen.shape[0] != tar.shape[0] or gen.device != tar.device:
            raise RuntimeError("smirk_b200.ExpressionLoss: gen and tar must have the same batch size and device, got %s on %s "
                               "and %s on %s" % (tuple(gen.shape), gen.device, tuple(tar.shape), tar.device))

    def forward(self, gen, tar, use_mean=True, metric="l2"):
        if metric not in _METRICS:
            raise ValueError("Unknown metric {}".format(metric))
        self._check_inputs(gen, tar)
        code, use_mean = _METRICS[metric], bool(use_mean)
        if torch.is_grad_enabled() and (gen.requires_grad or tar.requires_grad):
            return _ExpressionLossFunction.apply(gen, tar, self, code, use_mean)
        with torch.no_grad():
            return self._run(gen, tar, code, use_mean)[0]

    def _out(self, B, use_mean, dev):
        return torch.empty(() if use_mean else (B,), dtype=torch.float32, device=dev)

    @torch.no_grad()
    def _run(self, gen, tar, code, use_mean):
        """-> (loss, features [2B,2048]: gen's then tar's); the caller has run ``_check_inputs``."""
        dev = gen.device
        h = self._native_handle(dev)
        gen, tar = _lib.dev_f32(gen, "gen"), _lib.dev_f32(tar, "tar")
        B = gen.shape[0]
        loss = self._out(B, use_mean, dev)
        feat = torch.empty(2 * B, 2048, dtype=torch.float32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_expression_loss_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_expression_loss_forward", dev, h, gen, tar, B, code, int(use_mean), loss, feat, ws, ws.numel())
        return loss, feat

    def features(self, images):
        """[B,2048]: the reference's ``self.backbone(images).view(B, -1)``."""
        self._check_inputs(images, images)
        with torch.no_grad():
            return self._run(images, images, 0, False)[1][:images.shape[0]]

    def _forward_saved(self, gen, tar, code, use_mean, need):
        """-> (handle, loss, saved): the grad-mode forward for the inputs ``need`` names (1 gen, 2 tar, 3 both)."""
        dev = gen.device
        h = self._native_handle(dev)
        gen, tar = _lib.dev_f32(gen, "gen"), _lib.dev_f32(tar, "tar")
        B = gen.shape[0]
        loss = self._out(B, use_mean, dev)
        nbytes = _lib.call("smk_expression_loss_saved_bytes", dev, h, B, need)
        saved = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_expression_loss_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_expression_loss_forward_saved", dev, h, gen, tar, B, code, int(use_mean), need, loss, saved,
                  saved.numel() * 4, ws, ws.numel())
        return h, loss, saved

    @torch.no_grad()
    def saved_activations(self, gen, tar):
        """What the backward of ``self(gen, tar)`` uses when both inputs want a gradient: {"pool": [2B,64,56,56] the
        max-pool output, "pool_argmax": [2B,64,56,56] int8 winning tap ky*3 + kx, "layerL.j.u1" / ".u2" / ".y": [2B,C,H,W]
        post-ReLU outputs of conv1, conv2 and the block (gen's images, then tar's), "features": [2B,2048]}.  The forward
        is deterministic and batch-independent, so these are the tensors an autograd context holds."""
        self._check_inputs(gen, tar)
        h, _, saved = self._forward_saved(gen, tar, 0, False, 3)
        return self._saved_views(h, saved, gen.shape[0], 3)

    @staticmethod
    def _saved_views(h, saved, B, need):
        fn = getattr(_lib.lib(), "smk_expression_loss_saved_tensor")
        name, off, dims = C.c_char_p(), C.c_size_t(), (C.c_int * 4)()
        out, i = {}, 0
        while fn(h, B, need, i, C.byref(name), C.byref(off), dims) == 0:      # non-zero past the last tensor
            b, hh, ww, c = dims
            n, key = b * hh * ww * c, name.value.decode()
            if key == "pool_argmax":
                t = saved.view(torch.int8)[4 * off.value:4 * off.value + n]
            else:
                t = saved[off.value:off.value + n]
            out[key] = t.view(b, c) if key == "features" else t.view(b, hh, ww, c).permute(0, 3, 1, 2)
            i += 1
        return out


class _ExpressionLossFunction(torch.autograd.Function):
    """loss = ExpressionLoss(gen, tar) with frozen weights, and its gradient to whichever of gen and tar requires grad."""

    @staticmethod
    def forward(ctx, gen, tar, module, code, use_mean):
        need = (1 if ctx.needs_input_grad[0] else 0) | (2 if ctx.needs_input_grad[1] else 0)
        h, loss, saved = module._forward_saved(gen, tar, code, use_mean, need)
        ctx.handle, ctx.module, ctx.need, ctx.B, ctx.code, ctx.use_mean = h, module, need, gen.shape[0], code, use_mean
        ctx.dtypes = (gen.dtype, tar.dtype)
        ctx.save_for_backward(saved)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        saved, = ctx.saved_tensors
        m, dev, B, need = ctx.module, saved.device, ctx.B, ctx.need
        g = _lib.dev_f32(g, "g")
        gg = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 1 else None
        gt = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 2 else None
        ws = m._native_workspace("backward", _lib.call("smk_expression_loss_backward_workspace_bytes", dev, ctx.handle, B, need), dev)
        _lib.call("smk_expression_loss_backward", dev, ctx.handle, B, ctx.code, int(ctx.use_mean), need, saved, saved.numel() * 4,
                  g, gg, gt, ws, ws.numel())
        return (gg.to(ctx.dtypes[0]) if gg is not None else None, gt.to(ctx.dtypes[1]) if gt is not None else None,
                None, None, None)
