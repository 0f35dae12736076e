"""CPU suite for the encoder's input gradient: the oracle's autograd against the reference module's own
(tests/golden/encoder_grad.npz, oracle/make_golden_encoder_grad.py), the mask-replay oracle against plain autograd, and
argument checking of the input-gradient entry points (before any device work, so no GPU is needed)."""
import ctypes as C

import numpy as np
import torch

def _sd(seed=7):
    import smirk_b200
    from smirk_b200 import synth_inputs
    return synth_inputs.random_state_dict(smirk_b200.SmirkEncoder().state_dict(), seed=seed)


def _close(a, b, rtol):
    a, b = a.detach().double().numpy(), np.asarray(b, np.float64)
    assert a.shape == b.shape and np.abs(a - b).max() <= rtol * np.abs(b).max(), (np.abs(a - b).max(), np.abs(b).max())


def test_oracle_autograd_reproduces_golden_encoder_grad(golden):
    from oracle import encoder_replay_ref as rr, make_golden_encoder_grad as mg
    g = golden("encoder_grad")
    img = mg.encoder_input().requires_grad_()
    out, _ = rr.encoder_activations_ref(_sd(), img)
    gi, = torch.autograd.grad(rr.loss(out, mg.upstream()), img)
    for k, v in mg.subsample(gi).items():
        _close(v, g["g_img_" + k], 1e-6)


def test_replay_oracle_with_its_own_activations_equals_autograd():
    """Fed the oracle's own activations, the mask-replay forward (oracle/encoder_replay_ref.py) computes the same
    outputs as the plain oracle and has the same input gradient as plain autograd."""
    from oracle import encoder_replay_ref as rr, make_golden_encoder_grad as mg
    sd = _sd()
    img = mg.encoder_input().requires_grad_()
    out, act = rr.encoder_activations_ref(sd, img)
    gi, = torch.autograd.grad(rr.loss(out, mg.upstream()), img)
    assert list(act) == rr.saved_names() and len(act) == 2 * 32 + 24
    img2 = img.detach().clone().requires_grad_()
    out2 = rr.encoder_forward_replay_ref(sd, img2, {k: v.detach() for k, v in act.items()})
    for k in rr.OUTPUTS:
        assert torch.equal(out2[k], out[k]), k
    gi2, = torch.autograd.grad(rr.loss(out2, mg.upstream()), img2)
    _close(gi2, gi, 1e-6)


def test_encoder_grad_entry_points_reject_bad_arguments(native_lib):
    L = native_lib
    vp = C.c_void_p
    fake, buf, nul = vp(16), vp(16), vp(0)           # never dereferenced: the checks fail first
    rc = L.smk_encoder_forward_saved(nul, buf, 2, buf, buf, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"null handle" in L.smk_last_error()
    rc = L.smk_encoder_forward_saved(fake, buf, -1, buf, buf, buf, buf, 1 << 20, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_encoder_forward_saved(fake, buf, 2, buf, buf, buf, buf, 0, buf, 1 << 20, nul)
    assert rc < 0 and b"saved buffer too small" in L.smk_last_error()
    rc = L.smk_encoder_backward(nul, 2, buf, 1 << 20, buf, buf, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"null handle" in L.smk_last_error()
    rc = L.smk_encoder_backward(fake, -3, buf, 1 << 20, buf, buf, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"negative batch" in L.smk_last_error()
    rc = L.smk_encoder_backward(fake, 2, nul, 1 << 20, buf, buf, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"null argument" in L.smk_last_error()
    rc = L.smk_encoder_backward(fake, 2, buf, 0, buf, buf, buf, buf, buf, 1 << 20, nul)
    assert rc < 0 and b"saved buffer too small" in L.smk_last_error()
    rc = L.smk_encoder_saved_tensor(nul, 2, 0, C.byref(C.c_char_p()), C.byref(C.c_size_t()), (C.c_int * 4)())
    assert rc < 0 and b"null argument" in L.smk_last_error()
    # an empty batch is a no-op, whatever the buffers
    assert L.smk_encoder_forward_saved(fake, nul, 0, nul, nul, nul, nul, 0, nul, 0, nul) == 0
    assert L.smk_encoder_backward(fake, 0, nul, 0, nul, nul, nul, nul, nul, 0, nul) == 0
    assert L.smk_encoder_saved_bytes(nul, 4) == 0 and L.smk_encoder_backward_workspace_bytes(nul, 4) == 0
