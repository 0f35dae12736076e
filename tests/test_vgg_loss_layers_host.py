"""CPU guard of the integer-valued VGG network (vgg_ref.integer_state_dict / integer_inputs) that the GPU suite
(tests/test_gpu_vgg_loss_layers.py) runs at every precision and expects to match float64 bit for bit.  That test is only
exact if every operand and partial sum is representable, and only discriminating if the discrete cases the kernels must
get right occur.  Both are checked here in float64 at B = 1, so a change of seed or construction cannot silently make the
exact test wrong or vacuous:

- every activation and every gradient (at the normalised input, at each ReLU output, at the image) is a multiple of 0.5
  below 2^10 in magnitude: at most 11 significant bits, exact in TF32 (zero 3xTF32 tails), and every product and every
  partial sum of the convolutions exact in fp32;
- the L1 sums of the taps stay below 2^21, so at B = 3 the fp32 sums of these multiples of 0.5 are still exact;
- at every layer 30-70 % of the ReLU outputs are active; at every pool, positive windows with tied maxima (the first
  maximum must take the gradient); at every tap, zeros among the signs of phi(x) - phi(y) and both signs otherwise."""
import torch

import vgg_ref


def test_integer_network_is_exact_and_discriminating():
    B = 1                                                      # the GPU test's seeds at B = 1
    sd = {k: v.double() for k, v in vgg_ref.integer_state_dict(seed=11).items()}
    x, y = (t.double() for t in vgg_ref.integer_inputs(B, seed=901))
    saved = vgg_ref.oracle_saved(sd, x, y)
    xl, yl = x.clone().requires_grad_(), y.clone().requires_grad_()
    rec = []
    loss = vgg_ref.vgg_loss_replay_ref(sd, xl, yl, saved, rec)
    grads = torch.autograd.grad(loss, rec + [xl, yl], torch.tensor(vgg_ref.integer_upstream(B), dtype=torch.float64))

    def exact(what, t):
        assert bool(((2 * t).round() == 2 * t).all()), "%s: not a multiple of 0.5" % what
        assert float(t.abs().max()) < 2 ** 10, "%s: max %g" % (what, float(t.abs().max()))
    exact("normalised input", rec[0].detach())
    for k in vgg_ref.NAMES:
        exact(k, saved[k])
    for i, gr in enumerate(grads):
        exact("gradient %d" % i, gr)
    print("max activation %g, max ReLU-output gradient %g, max input gradient %g"
          % (max(float(saved[k].abs().max()) for k in vgg_ref.NAMES), max(float(gr.abs().max()) for gr in grads[1:11] + grads[12:22]),
             max(float(grads[-2].abs().max()), float(grads[-1].abs().max()))))
    assert float(grads[-1].abs().max()) >= 64                  # the gradients are not all trivially small

    for t, l in enumerate(vgg_ref.TAP_CONVS):
        d = saved[vgg_ref.NAMES[l]][:B] - saved[vgg_ref.NAMES[l]][B:]
        assert float(d.abs().sum()) < 2 ** 21, (t, float(d.abs().sum()))
        s = saved[vgg_ref.SIGNS[t]]
        zeros, pos, neg = (float((s == v).double().mean()) for v in (0, 1, -1))
        assert 0.2 <= zeros <= 0.9 and pos >= 0.02 and neg >= 0.02, (t, zeros, pos, neg)
        print("tap %d: L1 sum %.0f, %.2f of the signs 0" % (t, float(d.abs().sum()), zeros))
    for l, k in enumerate(vgg_ref.NAMES):
        v = saved[k]
        active = float((v > 0).double().mean())
        assert 0.3 <= active <= 0.7, (k, active)
        if l in vgg_ref.POOL_AFTER:
            n, C, S, _ = v.shape
            win = v.reshape(n, C, S // 2, 2, S // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(-1, 4)
            mx = win.max(dim=1).values
            tied = (win == mx[:, None]).sum(dim=1) >= 2
            frac = float(tied[mx > 0].double().mean())
            assert frac >= 0.05, (k, frac)
            print("%s: %.2f active, %.3f of the positive pool windows tied" % (k, active, frac))
        else:
            print("%s: %.2f active" % (k, active))
