"""Train-mode oracle of ``SmirkGenerator`` for the train-mode tests: ``oracle/generator_ref`` run with its functional ops
swapped, as ``oracle/generator_replay_ref`` does for the eval path, so there is still one restatement of the network.

``generator_train_ref`` swaps ``F.batch_norm`` for torch's train-mode BatchNorm: batch statistics, and the running
statistics of ``sd`` updated in place with factor ``momentum`` (``None``: 1 / num_batches_tracked, as
``nn.BatchNorm2d`` computes it) and ``num_batches_tracked += 1``.  With ``replay`` (the device's
``SmirkGenerator.saved_activations`` in train mode) every ReLU becomes ``z * [saved > 0]`` and every max-pool gathers at
the indices of the device's pool input: autograd through it is then the exact backward of the device's discrete choices.
``generator_ref`` is given a state dict of one-element CPU placeholders, which its own ``detach().float().cpu()`` keeps as
they are; the swapped ops map each placeholder back to the tensor of ``sd`` it stands for.  So autograd reaches the
parameters, and the oracle runs on the device and in the dtype of ``sd`` and ``x``: fp64 for the gradient gates, and
torch + cuDNN on the GPU for the benchmark.
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import generator_ref


def relu_names(res_blocks=5):
    """Names, in the forward's ReLU order, of the device's saved tensors that hold each ReLU output.  ``encNnorm2`` is
    the skip half of ``decNcat``."""
    enc = ["enc%dnorm%d" % (l, j) for l in (1, 2, 3, 4) for j in (1, 2)]
    dec = ["dec%dnorm%d" % (l, j) for l in (4, 3, 2, 1) for j in (1, 2)]
    return enc + ["bottlenecknorm1", "bottlenecknorm2"] + ["res%dnorm1" % r for r in range(res_blocks)] + dec


def relu_outputs(saved):
    """{relu_names entry: [B,C,H,W]} from the device's saved tensors (the skips sliced out of the decoder inputs)."""
    out = dict(saved)
    for l in (1, 2, 3, 4):
        cat = saved["dec%dcat" % l]
        out["enc%dnorm2" % l] = cat[:, cat.shape[1] // 2:]
    return out


class _Functional:
    def __init__(self, **ops):
        self.ops = ops

    def __getattr__(self, name):
        return self.ops[name] if name in self.ops else getattr(F, name)


@contextlib.contextmanager
def _swapped(**ops):
    saved = generator_ref.F
    generator_ref.F = _Functional(**ops)
    try:
        yield
    finally:
        generator_ref.F = saved


def bn_keys(sd):
    return [k[:-len(".running_mean")] for k in sd if k.endswith(".running_mean")]


def generator_train_ref(sd, x, res_blocks=5, momentum=0.1, replay=None, record=None):
    """One train-mode forward of ``generator_ref`` over the tensors of ``sd`` (a state dict with num_batches_tracked,
    updated in place; on the device and in the dtype of ``x``).  record (a dict, optional): receives each up-convolution's
    output under ``upconvN`` (with ``retain_grad``, so a backward leaves its gradient there).  -> y."""
    tok = {k: torch.empty(1) for k in sd}
    real = {t.data_ptr(): sd[k] for k, t in tok.items()}
    L = lambda t: None if t is None else real[t.data_ptr()]
    ups = iter(["upconv%d" % l for l in (4, 3, 2, 1)])
    bns = iter(bn_keys(sd))
    relus = iter(relu_names(res_blocks))
    pools = iter(["enc%dnorm2" % l for l in (1, 2, 3, 4)])

    def batch_norm(z, rm, rv, w, b, training=False, eps=1e-5, **kw):
        p = next(bns)
        assert L(rm) is sd[p + ".running_mean"], "BatchNorm order does not match generator_ref"
        sd[p + ".num_batches_tracked"] += 1
        f = 1.0 / float(sd[p + ".num_batches_tracked"]) if momentum is None else momentum
        return F.batch_norm(z, L(rm), L(rv), L(w), L(b), training=True, momentum=f, eps=eps)

    def relu(z, inplace=False):
        name = next(relus)
        return F.relu(z) if replay is None else z * (replay[name] > 0).to(z.dtype)

    def max_pool2d(t, kernel_size, stride=None, **kw):
        name = next(pools)
        if replay is None:
            return F.max_pool2d(t, kernel_size, stride, **kw)
        _, idx = F.max_pool2d(replay[name], 2, 2, return_indices=True)
        return t.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)

    conv2d = lambda t, w, b=None, **kw: F.conv2d(t, L(w), L(b), **kw)
    def conv_transpose2d(t, w, b=None, **kw):
        u = F.conv_transpose2d(t, L(w), L(b), **kw)
        name = next(ups)
        if record is not None and u.requires_grad:
            u.retain_grad()
            record[name] = u
        return u

    with _swapped(batch_norm=batch_norm, relu=relu, max_pool2d=max_pool2d, conv2d=conv2d, conv_transpose2d=conv_transpose2d):
        y = generator_ref.generator_forward_ref(tok, x, res_blocks=res_blocks)
    assert next(bns, None) is None and next(relus, None) is None, "op order does not match generator_ref"
    return y


def cpu_state(module, device="cpu", dtype=torch.float32):
    """The module's state as tensors on ``device`` (floating ones in ``dtype``; parameters as leaves that require grad),
    num_batches_tracked included."""
    sd = {}
    for k, v in module.state_dict().items():
        t = v.detach().to(device).clone()
        t = t.to(dtype) if t.is_floating_point() else t
        sd[k] = t.requires_grad_() if t.is_floating_point() and "running" not in k else t
    return sd
