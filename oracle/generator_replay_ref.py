"""ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Mask-replay version of ``oracle/generator_ref.generator_forward_ref`` for the generator's input gradient.  A ReLU mask or
max-pool choice that flips between two correct fp32 evaluations changes the gradient by a whole term, so the device's
gradient is compared with autograd through a forward that makes the DEVICE's discrete choices: every ReLU becomes
``z * [saved > 0]`` and every 2x2 max-pool gathers at the indices of the saved pool input (first maximum of the window,
row-major: torch's CPU rule), with ``saved`` the activations of the device's grad-mode forward
(``SmirkGenerator.saved_activations``).  Autograd through it is then the exact backward of those choices.

There is one restatement of the network, ``generator_ref``; this module runs it with its two discrete ops swapped.  Its
``F.relu`` calls come in forward order — per block conv1 and conv2 (``_block``), then each ResNet block's first conv
(``_resblock``) — and its ``F.max_pool2d`` calls are the four encoder pools: that order is ``layer_names``, the same order
in which ``smk_generator_saved_tensor`` lists the device's saved tensors.
"""
import contextlib

import torch.nn.functional as F

from oracle import generator_ref


def layer_names(res_blocks=5):
    """Names of the post-ReLU activations in forward order (the reference's layer names)."""
    enc = ["enc%dconv%d" % (l, j) for l in (1, 2, 3, 4) for j in (1, 2)]
    dec = ["dec%dconv%d" % (l, j) for l in (4, 3, 2, 1) for j in (1, 2)]
    return enc + ["bottleneckconv1", "bottleneckconv2"] + ["res%dconv1" % r for r in range(res_blocks)] + dec


class _Functional:
    """torch.nn.functional with ``relu`` and ``max_pool2d`` replaced."""

    def __init__(self, relu, max_pool2d):
        self.relu, self.max_pool2d = relu, max_pool2d

    def __getattr__(self, name):
        return getattr(F, name)


@contextlib.contextmanager
def _swapped(relu, max_pool2d):
    saved = generator_ref.F
    generator_ref.F = _Functional(relu, max_pool2d)
    try:
        yield
    finally:
        generator_ref.F = saved


def generator_forward_replay_ref(sd, x, replay, res_blocks=5):
    """``generator_forward_ref`` with the ReLU masks and pool indices of ``replay`` ({layer name: [B,C,H,W] activation})."""
    names = iter(layer_names(res_blocks))
    pools = iter(["enc%dconv2" % l for l in (1, 2, 3, 4)])

    def relu(z, inplace=False):
        return z * (replay[next(names)] > 0).to(z.dtype)

    def max_pool2d(t, kernel_size, stride=None, **kw):
        assert kernel_size == 2 and stride == 2 and not kw
        _, idx = F.max_pool2d(replay[next(pools)], 2, 2, return_indices=True)
        return t.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)

    with _swapped(relu, max_pool2d):
        y = generator_ref.generator_forward_ref(sd, x, res_blocks=res_blocks)
    assert next(names, None) is None and next(pools, None) is None, "replay order does not match generator_ref"
    return y


def generator_activations_ref(sd, x, res_blocks=5):
    """-> (y, {layer name: post-ReLU activation}) of the plain oracle forward (its own discrete choices)."""
    names, out = iter(layer_names(res_blocks)), {}

    def relu(z, inplace=False):
        a = F.relu(z)
        out[next(names)] = a
        return a

    with _swapped(relu, F.max_pool2d):
        y = generator_ref.generator_forward_ref(sd, x, res_blocks=res_blocks)
    assert next(names, None) is None, "activation order does not match generator_ref"
    return y, out
