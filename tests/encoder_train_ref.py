"""Train-mode restatement of ``SmirkEncoder`` (src/smirk_encoder.py:14-133) for the train-mode tests.

``EncoderTrainRef`` holds ``oracle/encoder_ref.BackboneRef`` backbones and the reference's heads under the reference's
module names, so ``load_state_dict`` takes a ``SmirkEncoder`` state dict (``num_batches_tracked`` included).  In train
mode its BatchNorms are torch's own: batch statistics, running-statistics update, and autograd through it gives every
parameter gradient.  With ``replay`` (``SmirkEncoder.saved_activations`` of the device) every backbone ReLU becomes
``z * [saved > 0]`` and the head's clamps and ReLU use the masks of the device's pre-clamp output: autograd through it is
then the exact backward of the device's discrete choices (the mask-replay idea of ``oracle/encoder_replay_ref``).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import encoder_ref, encoder_replay_ref as rr

PARTS = (("pose_encoder", "tf_mobilenetv3_small_minimal_100", "pose_cam_layers", 576),
         ("shape_encoder", "tf_mobilenetv3_large_minimal_100", "shape_layers", 960),
         ("expression_encoder", "tf_mobilenetv3_large_minimal_100", "expression_layers", 960))


class _Sub(nn.Module):
    def __init__(self, arch, head, feat, n_out):
        super().__init__()
        self.encoder = encoder_ref.BackboneRef(arch)
        setattr(self, head, nn.Sequential(nn.Linear(feat, n_out)))


class EncoderTrainRef(nn.Module):
    """``parts``: the sub-encoders this module holds (a SmirkEncoder: all three)."""

    def __init__(self, n_exp=50, n_shape=300, parts=("pose_encoder", "shape_encoder", "expression_encoder")):
        super().__init__()
        self.n_exp, self.parts = n_exp, tuple(parts)
        widths = {"pose_encoder": 6, "shape_encoder": n_shape, "expression_encoder": n_exp + 5}
        for enc, arch, head, feat in PARTS:
            if enc in self.parts:
                setattr(self, enc, _Sub(arch, head, feat, widths[enc]))

    def forward(self, img, replay=None, record=None):
        """record (a dict, optional): receives every backbone ReLU output under its saved-tensor name."""
        names = iter([n for n in rr.relu_names() if n.split(".")[0] in self.parts])

        def relu(z, inplace=False):
            name = next(names)
            a = F.relu(z) if replay is None else z * (replay[name] > 0).to(z.dtype)
            if record is not None:
                record[name] = a
            return a

        raw = {}
        with rr._swapped(relu, torch.clamp):
            for enc, _, head, _ in PARTS:
                if enc in self.parts:
                    sub = getattr(self, enc)
                    f = sub.encoder(img)[-1]
                    pooled = F.adaptive_avg_pool2d(f, (1, 1)).squeeze(-1).squeeze(-1)
                    raw[enc] = getattr(sub, head)(pooled)
        assert next(names, None) is None, "ReLU order does not match encoder_ref"
        out, ne = {}, self.n_exp
        if "pose_encoder" in raw:                               # smirk_encoder.py:34-45
            out["pose_params"], out["cam"] = raw["pose_encoder"][..., :3], raw["pose_encoder"][..., 3:]
        if "shape_encoder" in raw:                              # :66-73
            out["shape_params"] = raw["shape_encoder"]
        if "expression_encoder" in raw:                         # :95-110
            p = raw["expression_encoder"]
            out["expression_params"] = p[..., :ne]
            if replay is None:
                out["eyelid_params"] = torch.clamp(p[..., ne:ne + 2], 0, 1)
                out["jaw_params"] = torch.cat([F.relu(p[..., ne + 2].unsqueeze(-1)), torch.clamp(p[..., ne + 3:ne + 5], -.2, .2)], -1)
            else:
                clamps, jaw = rr._head_masks(replay["expression_encoder.expression_layers.0"].to(p.device), ne)
                clamp = lambda z, lo, hi, m: torch.clamp(z, lo, hi).detach() + (z - z.detach()) * m.to(z.dtype)
                out["eyelid_params"] = clamp(p[..., ne:ne + 2], 0, 1, next(clamps))
                out["jaw_params"] = torch.cat([p[..., ne + 2].unsqueeze(-1) * jaw.to(p.dtype), clamp(p[..., ne + 3:ne + 5], -.2, .2, next(clamps))], -1)
        return out


def from_module(enc, parts=None):
    """An ``EncoderTrainRef`` (CPU, fp32) with the state of the device module ``enc`` (a SmirkEncoder or a sub-encoder),
    in train mode, with each BatchNorm's momentum copied."""
    if parts is None:
        subs = {"PoseEncoder": "pose_encoder", "ShapeEncoder": "shape_encoder", "ExpressionEncoder": "expression_encoder"}
        parts = (subs[type(enc).__name__],) if type(enc).__name__ in subs else tuple(p for p, *_ in PARTS)
    sd = {k: v.detach().cpu().clone() for k, v in enc.state_dict().items()}
    if len(parts) == 1 and not any(k.startswith(parts[0] + ".") for k in sd):
        sd = {parts[0] + "." + k: v for k, v in sd.items()}
    ref = EncoderTrainRef(n_exp=enc.n_exp, n_shape=enc.n_shape, parts=parts)
    ref.load_state_dict(sd)
    momentum = next(m.momentum for m in enc.modules() if isinstance(m, nn.BatchNorm2d))
    for m in ref.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = momentum
    return ref.train()


OUTPUTS = rr.OUTPUTS


def zero_in_exact_arithmetic(name):
    """The bias of a BatchNorm without a ReLU after it (an inverted-residual block's bn3, the depthwise-separable block's
    bn2): its output reaches the loss only through linear maps into train-mode BatchNorms, whose input gradients sum to zero
    over the batch, so its gradient is exactly zero and any computed value is rounding noise."""
    return name.endswith(".bn3.bias") or name.endswith("blocks.0.0.bn2.bias")


def grad_scale(name, grads):
    """The scale a gradient is measured against: its own max-abs, or for a bias whose gradient is zero in exact arithmetic
    the max-abs of its BatchNorm's weight gradient.  grads: {parameter name: gradient} of the oracle."""
    key = name[:-len("bias")] + "weight" if zero_in_exact_arithmetic(name) else name
    return grads[key].detach().double().abs().max().clamp_min(1e-30)


def loss(out, up):
    """sum_k (out[k] * up[k]).sum() over the outputs present."""
    return sum((out[k] * up[k].to(out[k].device)).sum() for k in out)
