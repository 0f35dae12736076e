"""A torch restatement of MICA (src/models/MICA/mica.py) for the tests: the ArcFace iResNet-100, the head, F.normalize,
the shape regressor and the shape loss, written from their description, in any float dtype.  Plus ``mica_state_dict(seed)``,
seeded weights for every key of ``smirk_b200.MICA``, and ``write_checkpoint``, an ``assets/mica.tar`` in the reference's
layout.

The weights are meant to look like a trained network's: random BatchNorm statistics and affines, PReLU slopes in
[0, 0.5], He-scaled convolutions, and residual branches damped so the residual stream keeps its scale over 49 blocks.
(The reference's own init, normal(0, 0.1) on every conv, multiplies the stream by a large factor per block and overflows
fp32 long before the last one.)  ``mica_state_dict`` checks that every block output stays within ``BLOCK_SCALE_MAX``.
"""
import os

import torch
import torch.nn.functional as F

LAYERS = (3, 13, 30, 3)
PLANES = (64, 128, 256, 512)
BLOCK_SCALE_MAX = 50.0          # max |y| of any block output on the probe images, relative to 1


def blocks():
    """[(prefix, cin, cout, stride)] of the 49 IBasicBlocks in order."""
    out, cin = [], 64
    for i, (n, planes) in enumerate(zip(LAYERS, PLANES)):
        for j in range(n):
            out.append(("arcface.layer%d.%d." % (i + 1, j), cin, planes, 2 if j == 0 else 1))
            cin = planes
    return out


def _bn(sd, prefix, c, g, weight=(0.5, 1.5)):
    sd[prefix + "weight"] = torch.empty(c).uniform_(*weight, generator=g)
    sd[prefix + "bias"] = torch.randn(c, generator=g) * 0.1
    sd[prefix + "running_mean"] = torch.randn(c, generator=g) * 0.1
    sd[prefix + "running_var"] = torch.empty(c).uniform_(0.5, 1.5, generator=g)
    sd[prefix + "num_batches_tracked"] = torch.tensor(0, dtype=torch.long)


def _he(shape, g, gain=1.0):
    fan_in = 1
    for s in shape[1:]:
        fan_in *= s
    return torch.randn(*shape, generator=g) * (gain * (2.0 / fan_in) ** 0.5)


def mica_state_dict(seed=0, check=True):
    """Seeded weights for every key of ``smirk_b200.MICA`` (state_dict order).  With ``check``, asserts that every block
    output of a probe batch stays within BLOCK_SCALE_MAX."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    sd["arcface.conv1.weight"] = _he((64, 3, 3, 3), g)
    _bn(sd, "arcface.bn1.", 64, g)
    sd["arcface.prelu.weight"] = torch.empty(64).uniform_(0, 0.5, generator=g)
    for prefix, cin, cout, stride in blocks():
        _bn(sd, prefix + "bn1.", cin, g)
        sd[prefix + "conv1.weight"] = _he((cout, cin, 3, 3), g)
        _bn(sd, prefix + "bn2.", cout, g)
        sd[prefix + "prelu.weight"] = torch.empty(cout).uniform_(0, 0.5, generator=g)
        sd[prefix + "conv2.weight"] = _he((cout, cout, 3, 3), g, gain=0.5)
        _bn(sd, prefix + "bn3.", cout, g, weight=(0.1, 0.3))              # the damped residual branch
        if stride == 2:
            sd[prefix + "downsample.0.weight"] = _he((cout, cin, 1, 1), g)
            _bn(sd, prefix + "downsample.1.", cout, g)
    _bn(sd, "arcface.bn2.", 512, g)
    sd["arcface.fc.weight"] = _he((512, 512 * 49), g, gain=0.5)
    sd["arcface.fc.bias"] = torch.randn(512, generator=g) * 0.1
    _bn(sd, "arcface.features.", 512, g)
    k = 512
    for i in range(4):
        sd["regressor.network.%d.weight" % i] = _he((300, k), g, gain=1.0 / 1.04 ** 0.5)
        sd["regressor.network.%d.bias" % i] = torch.randn(300, generator=g) * 0.05
        k = 300
    sd["regressor.output.weight"] = _he((300, 300), g) * 0.25
    sd["regressor.output.bias"] = torch.randn(300, generator=g) * 0.05
    if check:
        scales = []
        arcface_ref(sd, prep(probe_images(1, seed)), scales)
        assert max(scales) <= BLOCK_SCALE_MAX, "block output scale %.3g exceeds %g" % (max(scales), BLOCK_SCALE_MAX)
    return sd


def probe_images(B, seed):
    """Smooth face-crop-like images [B,3,112,112] in [0, 1]."""
    g = torch.Generator().manual_seed(1000 + seed)
    low = torch.rand(B, 3, 8, 8, generator=g)
    img = F.interpolate(low, size=(112, 112), mode="bilinear", align_corners=False)
    return (img * 0.8 + 0.1 * torch.rand(B, 3, 112, 112, generator=g)).clamp(0, 1)


def prep(images):
    """The reference's input transform: (x - 0.5) / 0.5, channels flipped to BGR."""
    return images.sub(0.5).div(0.5)[:, [2, 1, 0], :, :]


def _bn_eval(sd, prefix, x):
    return F.batch_norm(x, sd[prefix + "running_mean"].to(x.dtype), sd[prefix + "running_var"].to(x.dtype),
                        sd[prefix + "weight"].to(x.dtype), sd[prefix + "bias"].to(x.dtype), False, 0.0, 1e-5)


def arcface_ref(sd, x, scales=None):
    """ArcFace embedding [B,512] of the transformed images x; scales (a list) collects max |y| of every block output."""
    dt = x.dtype
    W = lambda k: sd[k].to(dt)                                                        # noqa: E731
    x = F.conv2d(x, W("arcface.conv1.weight"), padding=1)
    x = F.prelu(_bn_eval(sd, "arcface.bn1.", x), W("arcface.prelu.weight"))
    for prefix, cin, cout, stride in blocks():
        identity = x
        out = _bn_eval(sd, prefix + "bn1.", x)
        out = F.conv2d(out, W(prefix + "conv1.weight"), padding=1)
        out = F.prelu(_bn_eval(sd, prefix + "bn2.", out), W(prefix + "prelu.weight"))
        out = F.conv2d(out, W(prefix + "conv2.weight"), stride=stride, padding=1)
        out = _bn_eval(sd, prefix + "bn3.", out)
        if stride == 2:
            identity = _bn_eval(sd, prefix + "downsample.1.", F.conv2d(x, W(prefix + "downsample.0.weight"), stride=2))
        x = out + identity
        if scales is not None:
            scales.append(float(x.abs().max()))
    x = torch.flatten(_bn_eval(sd, "arcface.bn2.", x), 1)
    x = F.linear(x, W("arcface.fc.weight"), W("arcface.fc.bias"))
    return F.batch_norm(x, W("arcface.features.running_mean"), W("arcface.features.running_var"),
                        W("arcface.features.weight"), W("arcface.features.bias"), False, 0.0, 1e-5)


def regressor_ref(sd, z):
    dt = z.dtype
    h = z
    for i in range(4):
        h = F.leaky_relu(F.linear(h, sd["regressor.network.%d.weight" % i].to(dt), sd["regressor.network.%d.bias" % i].to(dt)), 0.2)
    return F.linear(h, sd["regressor.output.weight"].to(dt), sd["regressor.output.bias"].to(dt))


def mica_ref(sd, images, dtype=torch.float32):
    """-> (shape_params [B,300], arcface features [B,512]) for images [B,3,112,112] in [0, 1]."""
    feat = arcface_ref(sd, prep(images.to(dtype)))
    return regressor_ref(sd, F.normalize(feat)), feat


def shape_loss_ref(shape_params, mica_shape):
    """The reference loss on MICA's shape_params: truncated to D columns, then mse_loss."""
    D = shape_params.shape[1]
    return F.mse_loss(shape_params, mica_shape[..., :D])


def write_checkpoint(sd, root):
    """<root>/assets/mica.tar in the reference's layout: {'arcface': ..., 'flameModel': regressor.* keys among others
    that the loader must drop}.  -> its path."""
    os.makedirs(os.path.join(root, "assets"), exist_ok=True)
    flame = {k: v for k, v in sd.items() if k.startswith("regressor.")}
    flame["flame.v_template"] = torch.zeros(4, 3)
    flame["shape_decoder.scale"] = torch.ones(1)
    ck = {"arcface": {k[len("arcface."):]: v for k, v in sd.items() if k.startswith("arcface.")}, "flameModel": flame}
    path = os.path.join(root, "assets", "mica.tar")
    torch.save(ck, path)
    return path
