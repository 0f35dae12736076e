"""GPU suite (-m gpu) for smirk_b200.VGGPerceptualLoss, one layer at a time and bit for bit (the end-to-end loss and
gradient checks are in test_gpu_vgg_loss.py).

1. Every conv of the forward against float64 from the device's own input (the saved activation of the layer before,
   max-pooled in float64 where a pool comes first, which is exact), at precisions 0, 1 and 3 and at B = 1 and 3: 2B = 2
   and 6 images put the 112^2 x 128 layers on both sides of tc_conv's choice between persistent CTAs and one tile per CTA.
   The same run pins the TF32 storage of the precision-1 activations, the sign maps against the saved activations and
   the loss against the float64 L1 means of the device's own tap activations.
2. An integer-valued network (vgg_ref.integer_state_dict; test_vgg_loss_layers_host.py guards its premise) on which
   every operand is exact in TF32 and every sum exact in fp32: activations, sign maps, input gradients and the loss must
   equal float64 bit for bit at every precision, need and B.  The gradient oracle takes its ReLU masks, pool arguments
   and signs from its own float64 forward, not from the device, so a wrong tie-break, a wrong sign-0 case, a wrong mask or
   a wrong saved row fails here.
3. Through the C ABI at need 1, 2 and 3: nothing written past the stated sizes of the saved buffer, the workspaces, the
   loss and the gradients, the gradient `need` does not ask for left untouched, and the need-1 / need-2 saved layouts
   equal the x and y halves of the need-3 one.

----------------------------------------------------------------------------------------------------- error bounds
With a the layer's input, w its weights and K = 9 * Cin (Cin padded to 8 / 32 at the first layer) the GEMM depth, norm =
||a w||_2 is the L2 norm over k of one output's products, computed in float64 next to the reference.
- Precision 3 (3xTF32 wgmma): bound() of test_gpu_generator_x3.py with scale 1.
- Precision 1 (TF32 wgmma): the device's operands are TF32 numbers (activations rounded where they are written, weights
  rounded on the host) and the reference uses the same ones, so every product is exact.  What is left is the single fp32
  accumulator: K / 8 wgmma updates, each truncating up to 2^-23 of a partial sum that grows like a random walk to
  ||a w||_2, in the same direction each time, about 2^-23 (K / 8) ||a w||_2; the bound takes twice that,
  2^-22 (8 + K / 8) ||a w||_2, plus 2^-22 (|acc| + |bias|) for the bias add, and where the output is rounded to TF32
  (every conv but the last) half a TF32 ulp, 2^-11 |ref|.  That last term is reached wherever |ref| lies just above a
  power of two, so the worst err / bound of the rounded layers sits just below 1 (measured on an H100 at 700 W: 0.90 to
  0.99); at the last conv, which is not rounded, it is 0.37.  A reference with the un-rounded weights misses the device
  by 2^-11 |w| per product, which this bound does not allow: against it the worst err / bound is 6 (relu4_2) to 73
  (relu1_1), measured the same way, and the test prints it.
- Precision 0 (fp32 CUDA cores, conv_gemm): one fmaf per k in increasing k, each rounding its partial sum s_k to nearest,
  |delta_k| <= 2^-24 |s_k|, with independent signs.  The partial sums walk to ||a w||_2 around a drift toward acc, so
  the error's standard deviation is at most about 2^-24 sqrt(K / 6) (||a w||_2 + |acc|).  The bound is
  2^-22 sqrt(K) (||a w||_2 + |acc|), about ten standard deviations for up to 19M outputs per layer, plus
  2^-22 (|acc| + |bias|) for the bias fma.
- The loss: the device adds non-negative terms |phi(x) - phi(y)| in fewer than 100 levels of fp32 rounding (the
  difference, 64 sequential adds per thread, the warp and block trees, the partials, the division and the three tap
  adds), so it is within 100 * 2^-24 of the exact loss of its own activations, relatively."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgg_ref
from test_gpu_generator_x3 import EPS, bound
from test_gpu_kernels import tf32_split
from test_gpu_vgg_loss import DEV, inputs, sd_on, vgg

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------- 1. layers vs float64
def layer_bound(precision, K, norm, acc, bias, ref, rounded):
    if precision == 3:
        return bound(K, norm, torch.ones((), dtype=torch.float64, device=norm.device), acc, bias)
    if precision == 0:
        return EPS * (K ** 0.5 * (norm + acc.abs()) + acc.abs() + bias.abs())
    b = EPS * ((8 + K / 8) * norm + acc.abs() + bias.abs())
    return b * (1 + 2.0 ** -11) + 2.0 ** -11 * ref.abs() if rounded else b


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("precision", [0, 1, 3])
def test_layers_vs_fp64(native_lib, precision, B):
    m = vgg(precision)
    x, y = (t.to(DEV) for t in inputs(B, 800 + B))
    with torch.no_grad():
        loss = m(x, y)
        saved = m.saved_activations(x, y)
    sd = sd_on(DEV)
    a0 = vgg_ref.normalise(sd, torch.cat([x, y]))          # the prep kernel's separate fp32 operations
    if precision == 1:
        a0 = tf32_split(a0)[0]
    cin_p = 8 if precision == 0 else 32
    worst, unrounded = [], []
    for l, k in enumerate(vgg_ref.CONVS):
        if l == 0:
            a = a0.double()
        else:
            a = saved[vgg_ref.NAMES[l - 1]].double()
            if l - 1 in vgg_ref.POOL_AFTER:
                a = F.max_pool2d(a, 2, 2)
        w, bias = sd[k + ".weight"], sd[k + ".bias"].double().view(1, -1, 1, 1)
        wr = (tf32_split(w)[0] if precision == 1 else w).double()
        acc = F.conv2d(a, wr, padding=1)
        norm = F.conv2d(a * a, wr * wr, padding=1).sqrt()
        ref = F.relu(acc + bias)
        rounded = precision == 1 and l < len(vgg_ref.CONVS) - 1
        K = 9 * (cin_p if l == 0 else a.shape[1])
        bnd = layer_bound(precision, K, norm, acc, bias, ref, rounded)
        got = saved[vgg_ref.NAMES[l]]
        assert torch.isfinite(got).all(), vgg_ref.NAMES[l]
        err = (got.double() - ref).abs()
        worst.append(float((err / bnd).max()))
        assert bool((err <= bnd).all()), "%s: %d of %d outside the bound, worst err / bound %.3g" % (
            vgg_ref.NAMES[l], int((err > bnd).sum()), err.numel(), worst[-1])
        if rounded:
            assert torch.equal(tf32_split(got)[0], got), "%s: not TF32-representable" % vgg_ref.NAMES[l]
        if precision == 1:
            loose = F.relu(F.conv2d(a, w.double(), padding=1) + bias)
            unrounded.append(float(((got.double() - loose).abs() / bnd).max()))
        del acc, norm, ref, err, bnd
    print("precision %d B %d: worst err / bound per layer %s" % (precision, B, " ".join("%.3f" % r for r in worst)))
    if unrounded:
        print("precision 1 B %d: against un-rounded weights %s" % (B, " ".join("%.1f" % r for r in unrounded)))
    exact = 0.0
    for t, l in enumerate(vgg_ref.TAP_CONVS):
        tap = saved[vgg_ref.NAMES[l]]
        assert torch.equal(saved[vgg_ref.SIGNS[t]], torch.sign(tap[:B] - tap[B:]).to(torch.int8)), vgg_ref.SIGNS[t]
        exact += float((tap[:B].double() - tap[B:].double()).abs().mean())
    rel = abs(float(loss) - exact) / exact
    print("precision %d B %d: loss rel err against its own activations %.2e" % (precision, B, rel))
    assert rel <= 100 * 2.0 ** -24


# ------------------------------------------------------------------------------------- 2. the integer network
_INT_VGGS = {}
INT_SEED = 11


def int_vgg(precision):
    import smirk_b200
    if precision not in _INT_VGGS:
        m = smirk_b200.VGGPerceptualLoss(weights=None)
        m.load_state_dict(vgg_ref.integer_state_dict(INT_SEED))
        m.precision = precision
        _INT_VGGS[precision] = m.to(DEV)
    return _INT_VGGS[precision]


@functools.lru_cache(maxsize=2)
def int_reference(B):
    """-> (x, y, saved, g_x, g_y, loss): the integer network's float64 activations and sign maps, input gradients for
    the upstream gradient vgg_ref.integer_upstream(B), and the loss as the device's fp32 order computes it from the
    exact tap sums."""
    sd = {k: v.double() for k, v in vgg_ref.integer_state_dict(INT_SEED).items()}
    x, y = vgg_ref.integer_inputs(B, 900 + B)
    saved = vgg_ref.oracle_saved(sd, x.double(), y.double())   # on the CPU: the GPU's float64 convolution backward
    xl, yl = x.double().requires_grad_(), y.double().requires_grad_()     # is not exact on these integers
    up = torch.tensor(vgg_ref.integer_upstream(B), dtype=torch.float64)
    gx, gy = torch.autograd.grad(vgg_ref.vgg_loss_replay_ref(sd, xl, yl, saved), [xl, yl], up)
    loss = np.float32(0.0)
    for t, l in enumerate(vgg_ref.TAP_CONVS):
        tap = saved[vgg_ref.NAMES[l]]
        s = float((tap[:B] - tap[B:]).abs().sum())
        assert s < 2 ** 23                                 # a multiple of 0.5: exact in fp32
        term = np.float32(s) / np.float32(tap[:B].numel())
        loss = term if t == 0 else np.float32(loss + term)
    return x.to(DEV), y.to(DEV), {k: v.to(DEV) for k, v in saved.items()}, gx.to(DEV), gy.to(DEV), loss


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("need", [1, 2, 3])
@pytest.mark.parametrize("precision", [0, 1, 3])
def test_integer_network_is_exact(native_lib, precision, need, B):
    x, y, ref, rgx, rgy, rloss = int_reference(B)
    m = int_vgg(precision)
    if need == 3:
        got = m.saved_activations(x, y)
        for k in vgg_ref.NAMES + vgg_ref.SIGNS:
            want = ref[k] if k in vgg_ref.SIGNS else ref[k].float()
            assert torch.equal(got[k], want), "%s: %d of %d differ" % (k, int((got[k] != want).sum()), want.numel())
    xl, yl = x.clone().requires_grad_(bool(need & 1)), y.clone().requires_grad_(bool(need & 2))
    loss = m(xl, yl)
    assert float(loss.detach()) == float(rloss), (float(loss.detach()), float(rloss))
    wrt = [t for t in (xl, yl) if t.requires_grad]
    grads = torch.autograd.grad(loss, wrt, torch.tensor(vgg_ref.integer_upstream(B), device=DEV))
    for got, want, on in ((grads[0], rgx, need & 1), (grads[-1], rgy, need & 2)):
        if on:
            want = want.float()
            assert torch.equal(got, want), "need %d: %d of %d gradient elements differ, max |diff| %g" % (
                need, int((got != want).sum()), want.numel(), float((got - want).abs().max()))


# ------------------------------------------------------------------------------------ 3. buffers and layouts
GUARD = 0x7FC0FACE                 # a quiet NaN whose payload no kernel writes
TAIL = 1 << 16                     # guard words past every buffer


def guarded(nbytes):
    """-> (int32 buffer of nbytes plus TAIL guard words, all holding GUARD, the number of words stated)."""
    assert nbytes % 4 == 0
    n = nbytes // 4
    return torch.full((n + TAIL,), GUARD, dtype=torch.int32, device=DEV), n


def untouched(buf, start=0):
    return bool((buf[start:] == GUARD).all())


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("precision", [0, 1, 3])
def test_buffers_stay_in_bounds_and_saved_layouts(native_lib, precision, B):
    from smirk_b200 import _lib
    m = vgg(precision)
    x, y = (t.to(DEV) for t in inputs(B, 820 + B))
    h = m._native_handle(DEV)
    size = lambda name, *a: _lib.call(name, DEV, h, *a)
    ws, n_ws = guarded(size("smk_vgg_loss_workspace_bytes", B))
    loss0, _ = guarded(4)
    _lib.call("smk_vgg_loss_forward", DEV, h, x, y, B, loss0, ws, 4 * n_ws)
    torch.cuda.synchronize()
    assert untouched(ws, n_ws) and untouched(loss0, 1), "forward"
    views = {}
    img = 3 * 224 * 224 * B
    g = torch.ones((), device=DEV)
    for need in (1, 2, 3):
        saved, n_sv = guarded(size("smk_vgg_loss_saved_bytes", B, need))
        loss, _ = guarded(4)
        _lib.call("smk_vgg_loss_forward_saved", DEV, h, x, y, B, need, loss, saved, 4 * n_sv, ws, 4 * n_ws)
        torch.cuda.synchronize()
        assert untouched(saved, n_sv) and untouched(ws, n_ws) and untouched(loss, 1), "forward_saved, need %d" % need
        assert torch.equal(loss[:1], loss0[:1]), need
        bws, n_bws = guarded(size("smk_vgg_loss_backward_workspace_bytes", B, need))
        (gx, _), (gy, _) = guarded(4 * img), guarded(4 * img)
        before = saved.clone()
        _lib.call("smk_vgg_loss_backward", DEV, h, B, need, saved, 4 * n_sv, g, gx, gy, bws, 4 * n_bws)
        torch.cuda.synchronize()
        assert torch.equal(saved, before) and untouched(bws, n_bws), "backward, need %d" % need
        for buf, on, what in ((gx, need & 1, "g_x"), (gy, need & 2, "g_y")):
            assert untouched(buf, img if on else 0), "backward, need %d: %s" % (need, what)
            if on:
                assert torch.isfinite(buf[:img].view(torch.float32)).all(), "need %d: %s not fully written" % (need, what)
        views[need] = m._saved_views(h, saved[:n_sv].view(torch.float32), B, need)
    for k in vgg_ref.NAMES:
        assert views[1][k].shape[0] == B and views[2][k].shape[0] == B and views[3][k].shape[0] == 2 * B
        assert torch.equal(views[1][k], views[3][k][:B]), k
        assert torch.equal(views[2][k], views[3][k][B:]), k
    for k in vgg_ref.SIGNS:
        assert torch.equal(views[1][k], views[3][k]) and torch.equal(views[2][k], views[3][k]), k
