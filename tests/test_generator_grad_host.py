"""CPU suite for the generator's input gradient: the oracle's autograd against the reference module's own
(tests/golden/generator_grad.npz, oracle/make_golden_generator_grad.py), the mask-replay oracle against plain autograd,
and argument checking of the input-gradient entry points (before any device work, so no GPU is needed)."""
import ctypes as C

import numpy as np
import torch

def _sd(seed=7):
    import smirk_b200
    from smirk_b200 import synth_inputs
    gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    return synth_inputs.random_state_dict(gen.state_dict(), seed=seed)


def _close(a, b, rtol):
    a, b = a.detach().double().numpy(), np.asarray(b, np.float64)
    assert a.shape == b.shape and np.abs(a - b).max() <= rtol * np.abs(b).max(), (np.abs(a - b).max(), np.abs(b).max())


def test_oracle_autograd_reproduces_golden_generator_grad(golden):
    from oracle import generator_ref, make_golden_generator_grad as mg
    g = golden("generator_grad")
    x = mg.generator_input().requires_grad_()
    (generator_ref.generator_forward_ref(_sd(), x) * mg.upstream()).sum().backward()
    for k, v in mg.subsample(x.grad).items():
        _close(v, g["g_x_" + k], 1e-6)


def test_replay_oracle_with_its_own_masks_equals_autograd():
    """Fed the oracle's own activations, the mask-replay forward (oracle/generator_replay_ref.py) computes the same y as
    generator_ref and has the same input gradient as plain autograd."""
    from oracle import generator_replay_ref as rr, make_golden_generator_grad as mg
    sd = _sd()
    x = mg.generator_input().requires_grad_()
    y, act = rr.generator_activations_ref(sd, x)
    gx, = torch.autograd.grad((y * mg.upstream()).sum(), x)
    assert list(act) == rr.layer_names(5) and len(act) == 23
    x2 = x.detach().clone().requires_grad_()
    y2 = rr.generator_forward_replay_ref(sd, x2, {k: v.detach() for k, v in act.items()})
    assert torch.equal(y2, y)
    gx2, = torch.autograd.grad((y2 * mg.upstream()).sum(), x2)
    _close(gx2, gx, 1e-6)


def test_grad_entry_points_reject_bad_arguments(native_lib):
    L = native_lib
    vp = C.c_void_p
    fake, buf, nul = vp(16), vp(16), vp(0)           # never dereferenced: the checks fail first
    rc = L.smk_generator_forward_saved(nul, buf, 2, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"null handle" in L.smk_last_error()
    rc = L.smk_generator_forward_saved(fake, buf, -1, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_generator_forward_saved(fake, buf, 2, buf, buf, 0, buf, 1 << 20, nul)
    assert rc < 0 and b"saved buffer too small" in L.smk_last_error()
    rc = L.smk_generator_backward(nul, 2, buf, buf, 1 << 20, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"null handle" in L.smk_last_error()
    rc = L.smk_generator_backward(fake, -3, buf, buf, 1 << 20, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_generator_backward(fake, 2, buf, nul, 1 << 20, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"null argument" in L.smk_last_error()
    rc = L.smk_generator_backward(fake, 2, buf, buf, 0, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"saved buffer too small" in L.smk_last_error()
    rc = L.smk_generator_saved_tensor(nul, 2, 0, C.byref(C.c_char_p()), C.byref(C.c_size_t()), (C.c_int * 4)())
    assert rc < 0 and b"null argument" in L.smk_last_error()
    # an empty batch is a no-op, whatever the buffers
    assert L.smk_generator_forward_saved(fake, nul, 0, nul, nul, 0, nul, 0, nul) == 0
    assert L.smk_generator_backward(fake, 0, nul, nul, 0, nul, nul, nul, 0, nul) == 0
    assert L.smk_generator_saved_bytes(nul, 4) == 0 and L.smk_generator_backward_workspace_bytes(nul, 4) == 0

