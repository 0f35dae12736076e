"""``VGGPerceptualLoss`` — drop-in for the reference ``src/losses/VGGPerceptualLoss.py``, the trainer's perceptual loss.

Same module tree and ``state_dict`` keys (``mean``, ``std``, ``blocks.0.0.weight`` ... ``blocks.3.21.bias``: torchvision
VGG16 ``features[:23]`` cut into four blocks that keep torchvision's indices) and the same ``forward(x, y)``: x and y
[B,3,224,224] in [-1, 1], normalised with the ImageNet mean / std, and the sum over the taps relu1_2, relu2_2, relu3_3 and
relu4_3 of ``l1_loss(phi(x), phi(y))``, a 0-dim fp32 tensor.  The network runs in ``csrc/vgg_loss.cu`` through
``smk_vgg_loss_forward`` (include/smirk_b200.h), x and y as one batch.

The VGG is frozen, as the reference freezes it.  With grad mode on and x and/or y requiring grad, the loss passes its
gradient to them (``smk_vgg_loss_forward_saved`` keeps the activations of the inputs that want one and the L1 sign
maps; ``smk_vgg_loss_backward`` walks the network back).  Weight gradients are not implemented: a parameter that requires
grad raises.  The network has no BatchNorm or dropout, so ``.train()`` and ``.eval()`` change nothing.

``precision`` (part of the native handle's key, so it may change between calls): 0 = fp32 CUDA cores, 1 = TF32 tensor cores,
3 = 3xTF32 tensor cores (fp32-equivalent, the same launches as 1), as for ``SmirkGenerator``.
"""
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


class VGGPerceptualLoss(_lib.FrozenNet, nn.Module):
    _kind, _name, _net, _inputs = "vgg_loss", "VGGPerceptualLoss", "the VGG", ("x", "y")
    _why_224 = "the reference resizes its inputs to 224x224 bilinearly, which is the identity only at 224x224, the one size implemented"
    _int8 = ("sign1_2", "sign2_2", "sign3_3", "sign4_3")

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

    def forward(self, x, y):
        self._check_frozen()
        _lib.check_image_pair(self, x, y)
        if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
            return _lib.PairLossFunction.apply(x, y, self, (), ())
        with torch.no_grad():
            dev = x.device
            h = self._native_handle(dev)
            x, y = _lib.dev_f32(x, "x"), _lib.dev_f32(y, "y")
            B = x.shape[0]
            loss = torch.empty((), dtype=torch.float32, device=dev)
            ws = self._native_workspace("forward", _lib.call("smk_vgg_loss_workspace_bytes", dev, h, B), dev)
            _lib.call("smk_vgg_loss_forward", dev, h, x, y, B, loss, ws, ws.numel())
            return loss

    @torch.no_grad()
    def saved_activations(self, x, y):
        """What the backward of ``self(x, y)`` uses when both inputs want a gradient: {"relu1_1" ... "relu4_3": [2B,C,H,W]
        post-ReLU outputs, x's images then y's; "sign1_2" ... "sign4_3": [B,C,H,W] int8 sign(phi(x) - phi(y)) at the taps}.
        The forward is deterministic and batch-independent, so these are the tensors an autograd context holds."""
        _lib.check_image_pair(self, x, y)
        h, _, saved = _lib.pair_forward_saved(self, x, y, (), 3, ())
        return self._saved_views(h, saved, x.shape[0], 3)
