"""``VGGPerceptualLoss`` — drop-in for the reference ``src/losses/VGGPerceptualLoss.py``, the trainer's perceptual loss.

Same module tree and ``state_dict`` keys (``mean``, ``std``, ``blocks.0.0.weight`` ... ``blocks.3.21.bias``: torchvision
VGG16 ``features[:23]`` cut into four blocks that keep torchvision's indices) and the same ``forward(x, y)``: x and y
[B,3,224,224] in [-1, 1], normalised with the ImageNet mean / std, and the sum over the taps relu1_2, relu2_2, relu3_3 and
relu4_3 of ``l1_loss(phi(x), phi(y))``, a 0-dim fp32 tensor.  The network runs in ``csrc/vgg_loss.cu`` through
``smk_vgg_loss_forward`` (include/smirk_b200_loss.h), x and y as one batch.

The VGG is frozen, as the reference freezes it.  With grad mode on and x and/or y requiring grad, the loss passes its
gradient to them (``smk_vgg_loss_forward_saved`` keeps the activations of the inputs that want one and the L1 sign
maps; ``smk_vgg_loss_backward`` walks the network back).  Weight gradients are not implemented: a parameter that requires
grad raises.  The network has no BatchNorm or dropout, so ``.train()`` and ``.eval()`` change nothing.

``precision`` (part of the native handle's key, so it may change between calls): 0 = fp32 CUDA cores, 1 = TF32 tensor cores,
3 = 3xTF32 tensor cores (fp32-equivalent, the same launches as 1), as for ``SmirkGenerator``.
"""
import ctypes as C
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib

# torchvision's vgg16().features[:23]: conv (in, out) or "M" for a 2x2 max pool, each conv followed by an in-place ReLU
_FEATURES = [(3, 64), (64, 64), "M", (64, 128), (128, 128), "M", (128, 256), (256, 256), (256, 256), "M",
             (256, 512), (512, 512), (512, 512)]
_BLOCKS = ((0, 4), (4, 9), (9, 16), (16, 23))


def _features():
    """Untrained containers with the layout and indices of ``torchvision.models.vgg16().features[:23]``."""
    layers = []
    for item in _FEATURES:
        if item == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(item[0], item[1], kernel_size=3, padding=1), nn.ReLU(inplace=True)]
    return nn.Sequential(OrderedDict((str(i), m) for i, m in enumerate(layers)))


class VGGPerceptualLoss(_lib.NativeModule, nn.Module):
    def __init__(self, weights="DEFAULT"):
        """``weights``: passed to ``torchvision.models.vgg16`` ("DEFAULT": the ImageNet weights the reference loads, which
        torchvision downloads into its hub cache on first use), or None: untrained containers for ``load_state_dict``."""
        super().__init__()
        if weights is None:
            feats = _features()
        else:
            import torchvision
            feats = torchvision.models.vgg16(weights=weights).features
        blocks = [feats[lo:hi].eval() for lo, hi in _BLOCKS]
        for bl in blocks:
            for p in bl.parameters():
                p.requires_grad = False
        self.blocks = nn.ModuleList(blocks)
        self.register_buffer("mean", torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
        self.register_buffer("std", torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))
        self.precision = 0

    def _native_extras(self):
        return (self.precision,)

    def _native_create(self, device):
        keep = []
        ts = list(self.state_dict().values())
        arr = (_lib.c_f32p * len(ts))()
        for j, t in enumerate(ts):
            a, p = _lib.f32(t)
            keep.append(a)
            arr[j] = p
        d = _lib.SmkVggLossDesc()
        d.tensors, d.n_tensors, d.precision = C.cast(arr, C.POINTER(_lib.c_f32p)), len(ts), self.precision
        return _lib.create("vgg_loss", d, device)

    @staticmethod
    def _check_inputs(x, y):
        for name, t in (("x", x), ("y", y)):
            _lib.require_cuda(t, name)
            if t.dim() != 4 or tuple(t.shape[1:]) != (3, 224, 224) or t.shape[0] < 1:
                raise RuntimeError("smirk_b200.VGGPerceptualLoss: expected %s [B,3,224,224], got %s — the reference resizes "
                                   "its inputs to 224x224 bilinearly, which is the identity only at 224x224, the one size "
                                   "implemented" % (name, tuple(t.shape)))
        if x.shape[0] != y.shape[0] or x.device != y.device:
            raise RuntimeError("smirk_b200.VGGPerceptualLoss: x and y must have the same batch size and device, got %s on %s "
                               "and %s on %s" % (tuple(x.shape), x.device, tuple(y.shape), y.device))

    def forward(self, x, y):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("smirk_b200.VGGPerceptualLoss: weight gradients are not implemented (the reference freezes "
                               "the VGG); keep its parameters at requires_grad=False")
        self._check_inputs(x, y)
        if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
            return _VggLossFunction.apply(x, y, self)
        with torch.no_grad():
            dev = x.device
            h = self._native_handle(dev)
            x, y = _lib.dev_f32(x, "x"), _lib.dev_f32(y, "y")
            B = x.shape[0]
            loss = torch.empty((), dtype=torch.float32, device=dev)
            ws = self._native_workspace("forward", _lib.call("smk_vgg_loss_workspace_bytes", dev, h, B), dev)
            _lib.call("smk_vgg_loss_forward", dev, h, x, y, B, loss, ws, ws.numel())
            return loss

    def _forward_saved(self, x, y, need):
        """-> (handle, loss, saved): the grad-mode forward for the inputs ``need`` names (1 x, 2 y, 3 both)."""
        dev = x.device
        h = self._native_handle(dev)
        x, y = _lib.dev_f32(x, "x"), _lib.dev_f32(y, "y")
        B = x.shape[0]
        loss = torch.empty((), dtype=torch.float32, device=dev)
        nbytes = _lib.call("smk_vgg_loss_saved_bytes", dev, h, B, need)
        saved = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_vgg_loss_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_vgg_loss_forward_saved", dev, h, x, y, B, need, loss, saved, saved.numel() * 4, ws, ws.numel())
        return h, loss, saved

    @torch.no_grad()
    def saved_activations(self, x, y):
        """What the backward of ``self(x, y)`` uses when both inputs want a gradient: {"relu1_1" ... "relu4_3": [2B,C,H,W]
        post-ReLU outputs, x's images then y's; "sign1_2" ... "sign4_3": [B,C,H,W] int8 sign(phi(x) - phi(y)) at the taps}.
        The forward is deterministic and batch-independent, so these are the tensors an autograd context holds."""
        self._check_inputs(x, y)
        h, _, saved = self._forward_saved(x, y, 3)
        return self._saved_views(h, saved, x.shape[0], 3)

    @staticmethod
    def _saved_views(h, saved, B, need):
        """{name: [B',C,H,W] view of ``saved``} for the buffer of a grad-mode forward with ``need``, B' = B per saved half."""
        fn = getattr(_lib.lib(), "smk_vgg_loss_saved_tensor")
        name, off, dims = C.c_char_p(), C.c_size_t(), (C.c_int * 4)()
        out, i = {}, 0
        while fn(h, B, need, i, C.byref(name), C.byref(off), dims) == 0:      # non-zero past the last tensor
            b, hh, ww, c = dims
            n, key = b * hh * ww * c, name.value.decode()
            if key.startswith("sign"):
                t = saved.view(torch.int8)[4 * off.value:4 * off.value + n]
            else:
                t = saved[off.value:off.value + n]
            out[key] = t.view(b, hh, ww, c).permute(0, 3, 1, 2)
            i += 1
        return out


class _VggLossFunction(torch.autograd.Function):
    """loss = VGG(x, y) with frozen weights, and its gradient to whichever of x and y requires grad."""

    @staticmethod
    def forward(ctx, x, y, module):
        need = (1 if ctx.needs_input_grad[0] else 0) | (2 if ctx.needs_input_grad[1] else 0)
        h, loss, saved = module._forward_saved(x, y, need)
        ctx.handle, ctx.module, ctx.need, ctx.B, ctx.dtypes = h, module, need, x.shape[0], (x.dtype, y.dtype)
        ctx.save_for_backward(saved)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        saved, = ctx.saved_tensors
        m, dev, B, need = ctx.module, saved.device, ctx.B, ctx.need
        g = _lib.dev_f32(g, "g")
        gx = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 1 else None
        gy = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=dev) if need & 2 else None
        ws = m._native_workspace("backward", _lib.call("smk_vgg_loss_backward_workspace_bytes", dev, ctx.handle, B, need), dev)
        _lib.call("smk_vgg_loss_backward", dev, ctx.handle, B, need, saved, saved.numel() * 4, g, gx, gy, ws, ws.numel())
        return (gx.to(ctx.dtypes[0]) if gx is not None else None, gy.to(ctx.dtypes[1]) if gy is not None else None, None)
