"""config_train's whole step on the device (tests/train_flow.py) at B = 32, precision 3, with the trainer's real masking
and cycle augmentation: forward + backward of both paths at both freeze parities is bitwise the same twice, a CUDA graph
of the first path replays bitwise equal to eager steps at the same RNG counters, every gradient and running statistic
compared, and 20 Adam steps lower the summed loss."""
import pytest
import torch

import train_flow as tf

pytestmark = pytest.mark.gpu
B = 32


@pytest.fixture(scope="module")
def bases(asset_root, native_lib):
    return tf.make_bases(asset_root)


def _eq(a, b):
    return len(a) == len(b) and all((x is None and y is None) or (x is not None and y is not None and torch.equal(x, y))
                                    for x, y in zip(a, b))


def _run(flow, batch):
    """step1, then step2 at both parities -> [(loss, grads)] and the running statistics."""
    l1, g1, eo = flow.path1(batch)
    out = [(l1, g1)]
    for parity in (0, 1):
        out.append(flow.path2(eo, batch, parity))
    return out, flow.stats()


def test_whole_step_is_bitwise_deterministic(bases):
    batch = tf.make_batch(B, 3000)
    runs = [_run(tf.TrainFlow(bases, 3, seed=5), batch) for _ in range(2)]
    for (la, ga), (lb, gb) in zip(runs[0][0], runs[1][0]):
        assert torch.equal(la, lb) and _eq(ga, gb)
        assert torch.isfinite(la) and all(torch.isfinite(t).all() for t in ga if t is not None)
        assert any(t is not None and float(t.abs().max()) > 0 for t in ga)
    n_enc = len(list(bases["enc"].parameters()))
    g1 = runs[0][0][0][1]                               # step1 trains both networks
    assert any(t is not None and float(t.abs().max()) > 0 for t in g1[:n_enc])
    assert any(t is not None and float(t.abs().max()) > 0 for t in g1[n_enc:])
    assert _eq(runs[0][1], runs[1][1])


def test_first_path_replays_from_a_cuda_graph(bases):
    """step1 (train-mode encoder and generator, FLAME, Renderer, VGG, the trainer's masking) captured once after an eager
    warm-up replays with new batches bitwise equal to an eager flow at the same RNG counters: loss, every gradient, the
    encoder output and, at the end, every running statistic.  The second path is not captured: its frozen network runs
    the eval path, whose handle folds the BatchNorm running statistics into the packed weights on the host, so a graph
    of it would keep the statistics of capture time while the first path keeps updating them."""
    G, E = tf.TrainFlow(bases, 3, seed=9), tf.TrainFlow(bases, 3, seed=9)
    data = [tf.make_batch(B, 3100 + 10 * s) for s in range(3)]
    static = {k: v.clone() for k, v in data[0].items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                          # handles and workspaces exist before capture
        G.path1(static)
    torch.cuda.current_stream().wait_stream(s)
    E.path1(data[0])
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = G.path1(static)
    for step in (1, 2):
        with torch.no_grad():
            for k in static:
                static[k].copy_(data[step][k])
        gr.replay()
        l1, g1, eo = E.path1(data[step])
        assert torch.equal(out[0], l1) and _eq(out[1], g1), step
        assert all(torch.equal(out[2][k], eo[k]) for k in eo), step
    torch.cuda.synchronize()
    assert _eq(G.stats(), E.stats())


def test_adam_lowers_the_summed_loss(bases):
    """20 steps of SmirkTrainer.step: step1's backward and Adam step, then step2's at the batch index's freeze parity, with
    the generator's gradient clipped to 0.1 when it trains (smirk_trainer.py:360-381).  Batch s uses batch s % 3 and the
    RNG counter s % 6, so steps 0 and 18 see the same inputs and draws: the summed loss there falls."""
    flow = tf.TrainFlow(bases, 3, seed=13)
    data = [tf.make_batch(B, 3200 + 10 * s) for s in range(3)]
    opt_e = torch.optim.Adam(flow.enc.parameters(), lr=1e-5)
    opt_g = torch.optim.Adam(flow.gen.parameters(), lr=1e-4, betas=(0.5, 0.999))
    losses = []
    for s in range(20):
        batch, parity = data[s % 3], s % 2
        flow.reseed(s % 6)
        l1, g1, eo = flow.path1(batch)
        for p, g in zip(flow.params1(), g1):
            p.grad = g
        opt_e.step(); opt_g.step()
        l2, g2 = flow.path2(eo, batch, parity)
        opt_e.zero_grad(); opt_g.zero_grad()
        for p, g in zip(flow.params2(parity), g2):
            p.grad = g
        if parity == 0:                                 # the generator trains in the second path
            torch.nn.utils.clip_grad_norm_(flow.gen.parameters(), 0.1)
            opt_g.step()
        else:
            opt_e.step()
        opt_e.zero_grad(); opt_g.zero_grad()
        losses.append(float(l1 + l2))
    print("config_train whole step, Adam: summed loss %.4f -> %.4f" % (losses[0], losses[18]))
    assert all(torch.isfinite(torch.tensor(losses)))
    assert losses[18] < losses[0]
