"""TEST ORACLE — the reference's ExpressionLoss (src/losses/ExpressionLoss.py) restated in torch ops over a ``state_dict``
of smirk_b200.ExpressionLoss, in any float dtype, and a replay variant.  Plus ``expression_state_dict(seed)``, seeded
weights for every key of the module, and ``write_checkpoint``, the reference's checkpoint file layout.

``expression_loss_ref(sd, gen, tar, use_mean, metric)``: the loss; ``backbone_ref(sd, x)``: the [B,2048] features.

``expression_loss_replay_ref(sd, gen, tar, saved, use_mean, metric)`` runs the same arithmetic with the discrete choices
taken from a device run's ``saved_activations``: every ReLU as z * [saved > 0] and the max pool as a gather at the
device's saved argmax taps, the stem's ReLU applied there as [pool > 0].  Its forward equals the loss wherever the device
agrees with it, and autograd through it (in float64) is the exact backward of the device's own choices, the oracle of
the device's input gradient.

The weights are meant to look like a trained network's: random BatchNorm statistics and affines, He-scaled convolutions,
and bn3 gammas damped so the residual stream keeps its scale over 16 blocks; ``expression_state_dict`` checks that every
block output stays within ``BLOCK_SCALE_MAX``.
"""
import os

import torch
import torch.nn.functional as F

LAYERS = (3, 4, 6, 3)
BLOCK_SCALE_MAX = 50.0          # max |y| of any block output on the probe images
CHECKPOINT = "assets/ResNet50/checkpoints/deca-epoch=01-val_loss_total/dataloader_idx_0=1.27607644.ckpt"


def blocks():
    """[(prefix, cin, planes, stride, downsample)] of the 16 Bottlenecks in order."""
    out, cin = [], 64
    for i, n in enumerate(LAYERS):
        planes = 64 << i
        for j in range(n):
            out.append(("backbone.layer%d.%d." % (i + 1, j), cin, planes, 2 if j == 0 and i > 0 else 1, j == 0))
            cin = planes * 4
    return out


def names():
    """The names of the saved tensors of ``saved_activations`` that hold ReLU masks, in forward order."""
    return ["pool"] + [p[len("backbone."):] + k for p, *_ in blocks() for k in ("u1", "u2", "y")]


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


def expression_state_dict(seed=0, check=True):
    """Seeded weights for every key of ``smirk_b200.ExpressionLoss`` (state_dict order: construction order inside a
    block).  With ``check``, asserts that every block output of a probe batch stays within BLOCK_SCALE_MAX."""
    g = torch.Generator().manual_seed(seed)
    sd = {"backbone.conv1.weight": _he((64, 3, 7, 7), g)}
    _bn(sd, "backbone.bn1.", 64, g)
    for prefix, cin, planes, stride, ds in blocks():
        sd[prefix + "conv1.weight"] = _he((planes, cin, 1, 1), g)
        sd[prefix + "conv2.weight"] = _he((planes, planes, 3, 3), g)
        _bn(sd, prefix + "bn1.", planes, g)
        _bn(sd, prefix + "bn2.", planes, g)
        sd[prefix + "conv3.weight"] = _he((planes * 4, planes, 1, 1), g)
        _bn(sd, prefix + "bn3.", planes * 4, g, weight=(0.1, 0.3))           # the damped residual branch
        if ds:
            sd[prefix + "downsample.0.weight"] = _he((planes * 4, cin, 1, 1), g)
            _bn(sd, prefix + "downsample.1.", planes * 4, g)
    sd["backbone.fc.weight"] = torch.randn(100, 2048, generator=g) * 0.01
    sd["backbone.fc.bias"] = torch.zeros(100)
    if check:
        scales = []
        backbone_ref(sd, probe_images(1, seed), scales=scales)
        assert max(scales) <= BLOCK_SCALE_MAX, "block output scale %.3g exceeds %g" % (max(scales), BLOCK_SCALE_MAX)
    return sd


def probe_images(B, seed):
    """Smooth face-like images [B,3,224,224] in [0, 1]."""
    gen = torch.Generator().manual_seed(2000 + seed)
    low = torch.rand(B, 3, 8, 8, generator=gen)
    img = F.interpolate(low, size=(224, 224), mode="bilinear", align_corners=False)
    return (img * 0.8 + 0.1 * torch.rand(B, 3, 224, 224, generator=gen)).clamp(0, 1)


def perturbed(images, seed, amount=0.3):
    """tar for the probe pairs: images + amount * N(0, 1) pixel noise, clamped to [0, 1].  (A smooth perturbation leaves
    the cosine distance of the two features near 1e-4, where fp32's own rounding of 1 - cos is 1e-3 of the loss; this
    one gives about 9e-3.)"""
    g = torch.Generator().manual_seed(500 + seed)
    return (images + amount * torch.randn(images.shape, generator=g)).clamp(0, 1)


def _bn_eval(sd, prefix, x):
    return F.batch_norm(x, sd[prefix + "running_mean"].to(x.dtype), sd[prefix + "running_var"].to(x.dtype),
                        sd[prefix + "weight"].to(x.dtype), sd[prefix + "bias"].to(x.dtype), False, 0.0, 1e-5)


def backbone_ref(sd, x, scales=None, record=None):
    """Features [B,2048] of images x; scales (a list) collects max |y| of every block output; record (a dict) receives
    the tensors of ``saved_activations`` (NCHW) for the oracle's own choices."""
    W = lambda k: sd[k].to(x.dtype)                                                    # noqa: E731
    s = F.relu(_bn_eval(sd, "backbone.bn1.", F.conv2d(x, W("backbone.conv1.weight"), stride=2, padding=3)))
    x, arg = F.max_pool2d(s, 3, 2, 1, return_indices=True)
    if record is not None:
        record["pool"] = x
        # torch's flat index (h * 112 + w) -> the window tap ky*3 + kx
        h, w = arg // 112, arg % 112
        oh = torch.arange(56, device=x.device).view(1, 1, 56, 1)
        ow = torch.arange(56, device=x.device).view(1, 1, 1, 56)
        record["pool_argmax"] = ((h - 2 * oh + 1) * 3 + (w - 2 * ow + 1)).to(torch.int8)
    for prefix, cin, planes, stride, ds in blocks():
        u1 = F.relu(_bn_eval(sd, prefix + "bn1.", F.conv2d(x, W(prefix + "conv1.weight"))))
        u2 = F.relu(_bn_eval(sd, prefix + "bn2.", F.conv2d(u1, W(prefix + "conv2.weight"), stride=stride, padding=1)))
        out = _bn_eval(sd, prefix + "bn3.", F.conv2d(u2, W(prefix + "conv3.weight")))
        identity = _bn_eval(sd, prefix + "downsample.1.", F.conv2d(x, W(prefix + "downsample.0.weight"), stride=stride)) if ds else x
        x = F.relu(out + identity)
        if scales is not None:
            scales.append(float(x.abs().max()))
        if record is not None:
            key = prefix[len("backbone."):]
            record[key + "u1"], record[key + "u2"], record[key + "y"] = u1, u2, x
    return F.avg_pool2d(x, 7, stride=1).view(x.shape[0], -1)


def metric_ref(f_gen, f_tar, use_mean=True, metric="l2"):
    if metric == "l2":
        loss = ((f_gen - f_tar) ** 2).mean(dim=1)
    elif metric == "l1":
        loss = torch.abs(f_gen - f_tar).mean(dim=1)
    elif metric == "cos":
        loss = 1.0 - F.cosine_similarity(f_gen, f_tar, dim=1)
    else:
        raise ValueError("Unknown metric {}".format(metric))
    return loss.mean() if use_mean else loss


def expression_loss_ref(sd, gen, tar, use_mean=True, metric="l2"):
    return metric_ref(backbone_ref(sd, gen), backbone_ref(sd, tar), use_mean, metric)


def backbone_replay_ref(sd, x, saved_half):
    """backbone_ref with the ReLU masks and pool taps of ``saved_half`` ({name: [B,C,H,W]} of one half)."""
    W = lambda k: sd[k].to(x.dtype)                                                    # noqa: E731
    m = lambda t, k: t * (saved_half[k] > 0).to(t.dtype)                              # noqa: E731
    z = _bn_eval(sd, "backbone.bn1.", F.conv2d(x, W("backbone.conv1.weight"), stride=2, padding=3))
    B, C = z.shape[:2]
    win = F.unfold(z, 3, padding=1, stride=2).view(B, C, 9, 56, 56)
    x = torch.gather(win, 2, saved_half["pool_argmax"].long().unsqueeze(2)).squeeze(2)
    x = m(x, "pool")                                                                  # the stem's ReLU at the argmax
    for prefix, cin, planes, stride, ds in blocks():
        key = prefix[len("backbone."):]
        u1 = m(_bn_eval(sd, prefix + "bn1.", F.conv2d(x, W(prefix + "conv1.weight"))), key + "u1")
        u2 = m(_bn_eval(sd, prefix + "bn2.", F.conv2d(u1, W(prefix + "conv2.weight"), stride=stride, padding=1)), key + "u2")
        out = _bn_eval(sd, prefix + "bn3.", F.conv2d(u2, W(prefix + "conv3.weight")))
        identity = _bn_eval(sd, prefix + "downsample.1.", F.conv2d(x, W(prefix + "downsample.0.weight"), stride=stride)) if ds else x
        x = m(out + identity, key + "y")
    return F.avg_pool2d(x, 7, stride=1).view(x.shape[0], -1)


def expression_loss_replay_ref(sd, gen, tar, saved, use_mean=True, metric="l2"):
    """saved: ``ExpressionLoss.saved_activations(gen, tar)`` ([2B, ...]: gen's images, then tar's).  The l1 metric takes
    its signs from the device's saved features, as mean(s * (f_gen - f_tar)), like the ReLU masks."""
    B = gen.shape[0]
    keys = names() + ["pool_argmax"]
    fg = backbone_replay_ref(sd, gen, {k: saved[k][:B] for k in keys})
    ft = backbone_replay_ref(sd, tar, {k: saved[k][B:] for k in keys})
    if metric == "l1":
        s = torch.sign(saved["features"][:B] - saved["features"][B:]).to(fg.dtype)
        loss = (s * (fg - ft)).mean(dim=1)
        return loss.mean() if use_mean else loss
    return metric_ref(fg, ft, use_mean, metric)


def oracle_saved(sd, gen, tar):
    """The oracle's own activations and pool taps, in the layout of saved_activations (for testing the replay)."""
    rg, rt = {}, {}
    with torch.no_grad():
        fg = backbone_ref(sd, gen, record=rg)
        ft = backbone_ref(sd, tar, record=rt)
    out = {k: torch.cat([rg[k], rt[k]]) for k in rg}
    out["features"] = torch.cat([fg, ft])
    return out


def write_checkpoint(sd, root):
    """<root>/CHECKPOINT in the reference's layout: {'state_dict': backbone.* (fc included) and the classifier's
    linear.* that the loader drops}.  -> its path."""
    path = os.path.join(root, CHECKPOINT)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    ck = dict(sd)
    ck["linear.weight"] = torch.randn(8, 2048, generator=torch.Generator().manual_seed(3)) * 0.01
    ck["linear.bias"] = torch.zeros(8)
    torch.save({"state_dict": ck, "epoch": 1}, path)
    return path
