"""ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Mask-replay version of ``oracle/encoder_ref.encoder_forward_ref`` for the encoder's input gradient.  A ReLU or clamp
mask that flips between two correct fp32 evaluations changes the gradient by a whole term, so the device's gradient is
compared with autograd through a forward that makes the DEVICE's discrete choices: every backbone ReLU becomes
``z * [saved > 0]``, and the expression head's ReLU and clamps use masks of the device's saved pre-clamp head output
(torch's rules: ``relu`` passes where p > 0, ``clamp`` on [lo, hi] inclusive), with ``saved`` the tensors of the
device's grad-mode forward (``SmirkEncoder.saved_activations``).  Every other op is linear, so autograd through it is
the exact backward of those choices.

There is one restatement of the network, ``encoder_ref``: this module runs its ``encoder_forward_ref`` (backbones and
head glue) with ``F`` swapped (``relu``) and ``torch`` swapped (``clamp``, and ``no_grad`` made a no-op so that autograd
reaches the image).  Its ``F.relu`` calls come in forward order — per backbone (pose, shape, expression) the stem, then
each block's ReLUs — and then the jaw ReLU of the head glue: the backbone part of that order is ``saved_names`` without
the heads, the order in which ``smk_encoder_saved_tensor`` lists the device's saved tensors.
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import encoder_ref

ENCODERS = (("pose_encoder", "tf_mobilenetv3_small_minimal_100", "pose_cam_layers.0"),
            ("shape_encoder", "tf_mobilenetv3_large_minimal_100", "shape_layers.0"),
            ("expression_encoder", "tf_mobilenetv3_large_minimal_100", "expression_layers.0"))


def saved_names():
    """Names of the saved tensors in the device's order: per backbone the ReLU outputs in forward order (the module path
    of each ReLU's BatchNorm), then its head's pre-clamp output."""
    out = []
    for enc, arch, head in ENCODERS:
        out.append(enc + ".encoder.bn1")
        for s, stage in enumerate(encoder_ref.ARCH[arch]):
            for i, (kind, _, _, _) in enumerate(stage):
                pre = "%s.encoder.blocks.%d.%d." % (enc, s, i)
                out += [pre + "bn1", pre + "bn2"] if kind == "ir" else [pre + "bn1"]
        out.append(enc + "." + head)
    return out


def relu_names():
    return [n for n in saved_names() if ".encoder." in n]


class _Shim:
    """A module with some attributes replaced; the rest come from ``base``."""

    def __init__(self, base, **over):
        self._base = base
        self.__dict__.update(over)

    def __getattr__(self, name):
        return getattr(self._base, name)


@contextlib.contextmanager
def _swapped(relu, clamp):
    f, t = encoder_ref.F, encoder_ref.torch
    encoder_ref.F = _Shim(F, relu=relu)
    encoder_ref.torch = _Shim(torch, clamp=clamp, no_grad=contextlib.nullcontext)
    try:
        yield
    finally:
        encoder_ref.F, encoder_ref.torch = f, t


def _head_masks(raw, n_exp):
    """The expression head's discrete choices from its pre-clamp output, in call order: eyelid clamp, jaw clamp; jaw ReLU."""
    clamps = iter([(raw[..., n_exp:n_exp + 2] >= 0) & (raw[..., n_exp:n_exp + 2] <= 1),
                   (raw[..., n_exp + 3:n_exp + 5] >= -0.2) & (raw[..., n_exp + 3:n_exp + 5] <= 0.2)])
    return clamps, (raw[..., n_exp + 2] > 0).unsqueeze(-1)


def encoder_forward_replay_ref(sd, img, replay, n_exp=50):
    """``encoder_forward_ref`` with the masks of ``replay`` ({saved name: tensor}, as ``saved_activations`` returns)."""
    names = iter(relu_names())
    clamps, jaw = _head_masks(replay["expression_encoder.expression_layers.0"], n_exp)
    jaw_done = []

    def relu(z, inplace=False):
        name = next(names, None)
        if name is None:                                     # the head glue's jaw ReLU (its input is [B, 1])
            jaw_done.append(1)
            return z * jaw.to(z.dtype)
        return z * (replay[name] > 0).to(z.dtype)

    def clamp(z, lo, hi):                                    # the clamp's value, the replayed mask's gradient
        return torch.clamp(z, lo, hi).detach() + (z - z.detach()) * next(clamps).to(z.dtype)

    with _swapped(relu, clamp):
        out = encoder_ref.encoder_forward_ref(sd, img, n_exp=n_exp)
    assert jaw_done == [1] and next(clamps, None) is None, "replay order does not match encoder_ref"
    return out


def encoder_activations_ref(sd, img, n_exp=50):
    """-> (outputs, {saved name: tensor}) of the plain oracle forward with autograd enabled (its own discrete choices):
    the ReLU outputs and the heads' pre-clamp outputs, in the layout of ``saved_activations``."""
    names, act = iter(relu_names()), {}

    def relu(z, inplace=False):
        a = F.relu(z)
        name = next(names, None)
        if name is not None:
            act[name] = a
        return a

    with _swapped(relu, torch.clamp):
        out = encoder_ref.encoder_forward_ref(sd, img, n_exp=n_exp)
    assert next(names, None) is None, "activation order does not match encoder_ref"
    g = lambda k: sd[k].detach().float().cpu()
    for enc, _, head in ENCODERS:
        act[enc + "." + head] = F.linear(out["_features"][enc], g(enc + "." + head + ".weight"), g(enc + "." + head + ".bias"))
    return out, {k: act[k] for k in saved_names()}


OUTPUTS = ("pose_params", "cam", "shape_params", "expression_params", "eyelid_params", "jaw_params")


def loss(out, up):
    """sum_k (out[k] * up[k]).sum() over the six outputs."""
    return sum((out[k] * up[k]).sum() for k in OUTPUTS)
