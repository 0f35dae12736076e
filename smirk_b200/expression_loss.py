"""``ExpressionLoss`` — drop-in for the reference ``src/losses/ExpressionLoss.py``, the trainer's emotion loss.

Same module tree and ``state_dict`` keys (``backbone.*``: EMOCA's ResNet-50 with ``Bottleneck`` layers (3, 4, 6, 3), the
stride of each layer's first block on its 3x3 ``conv2``, and the unused ``fc``), with plain ``nn`` containers whose own
``forward`` is never called: the network runs in ``csrc/expression_loss.cu`` through ``smk_expression_loss_forward``
(include/smirk_b200.h), gen and tar as one batch.

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


class ExpressionLoss(_lib.FrozenNet, nn.Module):
    _kind, _name, _net, _inputs = "expression_loss", "ExpressionLoss", "the emotion network", ("gen", "tar")
    _why_224 = "the backbone's 7x7 average pool gives one 2048-d feature per image only at 224x224, the one size implemented"
    _int8 = ("pool_argmax",)

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

    def _native_tensors(self):
        """The backbone without the unused fc."""
        return [t for k, t in self.state_dict().items()
                if not k.endswith("num_batches_tracked") and not k.startswith("backbone.fc.")]

    def _check_inputs(self, gen, tar):
        self._check_frozen()
        _lib.check_image_pair(self, gen, tar)

    def forward(self, gen, tar, use_mean=True, metric="l2"):
        if metric not in _METRICS:
            raise ValueError("Unknown metric {}".format(metric))
        self._check_inputs(gen, tar)
        code, use_mean = _METRICS[metric], bool(use_mean)
        if torch.is_grad_enabled() and (gen.requires_grad or tar.requires_grad):
            return _lib.PairLossFunction.apply(gen, tar, self, (code, int(use_mean)), () if use_mean else (gen.shape[0],))
        with torch.no_grad():
            return self._run(gen, tar, code, use_mean)[0]

    @torch.no_grad()
    def _run(self, gen, tar, code, use_mean):
        """-> (loss, features [2B,2048]: gen's then tar's); the caller has run ``_check_inputs``."""
        dev = gen.device
        h = self._native_handle(dev)
        gen, tar = _lib.dev_f32(gen, "gen"), _lib.dev_f32(tar, "tar")
        B = gen.shape[0]
        loss = torch.empty(() if use_mean else (B,), dtype=torch.float32, device=dev)
        feat = torch.empty(2 * B, 2048, dtype=torch.float32, device=dev)
        ws = self._native_workspace("forward", _lib.call("smk_expression_loss_workspace_bytes", dev, h, B), dev)
        _lib.call("smk_expression_loss_forward", dev, h, gen, tar, B, code, int(use_mean), loss, feat, ws, ws.numel())
        return loss, feat

    def features(self, images):
        """[B,2048]: the reference's ``self.backbone(images).view(B, -1)``."""
        self._check_inputs(images, images)
        with torch.no_grad():
            return self._run(images, images, 0, False)[1][:images.shape[0]]

    @torch.no_grad()
    def saved_activations(self, gen, tar):
        """What the backward of ``self(gen, tar)`` uses when both inputs want a gradient: {"pool": [2B,64,56,56] the
        max-pool output, "pool_argmax": [2B,64,56,56] int8 winning tap ky*3 + kx, "layerL.j.u1" / ".u2" / ".y": [2B,C,H,W]
        post-ReLU outputs of conv1, conv2 and the block (gen's images, then tar's), "features": [2B,2048]}.  The forward
        is deterministic and batch-independent, so these are the tensors an autograd context holds."""
        self._check_inputs(gen, tar)
        h, _, saved = _lib.pair_forward_saved(self, gen, tar, (0, 0), 3, (gen.shape[0],))
        return self._saved_views(h, saved, gen.shape[0], 3)
