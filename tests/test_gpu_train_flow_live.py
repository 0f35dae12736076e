"""config_train's whole step (tests/train_flow.py) at B = 32, precision 3, with the frozen network of the second path on
live weights (``live_weights_(True)`` on the encoder and the generator): the second path is bitwise the host-packed one's,
and SmirkTrainer.step — step1's forward, backward and Adam steps, then step2 at the batch's freeze parity with the
generator's gradient clipped to 0.1, and its Adam step — captures as two CUDA graphs, one per freeze parity, whose
alternating replays with new batches are bitwise an eager flow without the opt-in at the same RNG counters: losses,
parameters, Adam state and running statistics."""
import gc

import pytest
import torch

import train_flow as tf

pytestmark = pytest.mark.gpu
B = 32


@pytest.fixture(scope="module")
def bases(asset_root, native_lib):
    return tf.make_bases(asset_root)


def _live(flow):
    flow.enc.live_weights_(True)
    flow.gen.live_weights_(True)
    return flow


def _eq(a, b):
    return len(a) == len(b) and all((x is None and y is None) or (x is not None and y is not None and torch.equal(x, y))
                                    for x, y in zip(a, b))


def test_second_path_on_live_weights_equals_the_host_handle(bases):
    batch = tf.make_batch(B, 3300)
    host, live = tf.TrainFlow(bases, 3, seed=5), _live(tf.TrainFlow(bases, 3, seed=5))
    for parity in (0, 1):
        _, _, eo_h = host.path1(batch)
        _, _, eo_l = live.path1(batch)
        lh, gh = host.path2(eo_h, batch, parity)
        ll, gl = live.path2(eo_l, batch, parity)
        assert torch.equal(lh, ll) and _eq(gh, gl), parity
        assert _eq(host.stats(), live.stats()), parity
    assert live.enc._native.live_handle is not None and live.gen._native.live_handle is not None


class Trainer:
    """SmirkTrainer.step over a flow: capturable Adam (smirk_trainer.py's optimizers), the gradients written into
    preallocated ``.grad`` tensors (a parameter a path does not reach has ``.grad = None`` for that step, so Adam skips it
    as it does eagerly)."""

    def __init__(self, flow):
        self.flow = flow
        self.opt_e = torch.optim.Adam(flow.enc.parameters(), lr=1e-5, capturable=True)
        self.opt_g = torch.optim.Adam(flow.gen.parameters(), lr=1e-4, betas=(0.5, 0.999), capturable=True)
        self.buf = {p: torch.zeros_like(p) for p in flow.params1()}

    def _set_grads(self, params, grads):
        for p in self.flow.params1():
            p.grad = None
        for p, g in zip(params, grads):
            if g is not None:
                self.buf[p].copy_(g)
                p.grad = self.buf[p]

    def step(self, batch, parity):
        f = self.flow
        l1, g1, eo = f.path1(batch)
        self._set_grads(f.params1(), g1)
        self.opt_e.step(); self.opt_g.step()
        l2, g2 = f.path2(eo, batch, parity)
        self._set_grads(f.params2(parity), g2)
        if parity == 0:                                 # the generator trains in the second path
            torch.nn.utils.clip_grad_norm_(f.gen.parameters(), 0.1)
            self.opt_g.step()
        else:
            self.opt_e.step()
        self._set_grads([], [])
        return l1, l2

    def state(self):
        out = [p.detach() for p in self.flow.params1()] + self.flow.stats()
        for opt in (self.opt_e, self.opt_g):
            for p in opt.param_groups[0]["params"]:
                out += [v for k, v in sorted(opt.state[p].items())]
        return out


def _free_device_memory():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_whole_step_replays_from_two_cuda_graphs(bases):
    """The eager flow runs first and keeps only its losses and final state, so its workspaces are gone before the graphed
    flow allocates its own and the two graphs' memory; the graphs share one pool (captured and replayed in the same order)."""
    data = [tf.make_batch(B, 3400 + 10 * s) for s in range(3)]
    schedule = [(parity, data[0]) for parity in (0, 1)] + [(step % 2, data[(step + 1) % 3]) for step in range(4)]
    _free_device_memory()
    held = torch.cuda.memory_allocated()
    E = Trainer(tf.TrainFlow(bases, 3, seed=17))
    eager = [tuple(t.clone() for t in E.step(batch, parity)) for parity, batch in schedule]
    eager_state = [t.clone() for t in E.state()]
    del E
    _free_device_memory()
    torch.cuda.reset_peak_memory_stats()
    G = Trainer(_live(tf.TrainFlow(bases, 3, seed=17)))
    static = {k: v.clone() for k, v in data[0].items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                          # handles, workspaces and Adam state exist before capture
        for parity, batch in schedule[:2]:
            G.step(static, parity)
    torch.cuda.current_stream().wait_stream(s)
    graphs, outs = [], []
    for parity in (0, 1):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=graphs[0].pool() if graphs else None):
            outs.append(G.step(static, parity))
        graphs.append(g)
    for step, (parity, batch) in enumerate(schedule[2:]):
        with torch.no_grad():
            for k in static:
                static[k].copy_(batch[k])
        graphs[parity].replay()
        l1, l2 = eager[2 + step]
        assert torch.equal(outs[parity][0], l1) and torch.equal(outs[parity][1], l2), step
    torch.cuda.synchronize()
    print("whole step from two CUDA graphs: %.1f GiB held before the test, peak %.1f GiB"
          % (held / 2 ** 30, torch.cuda.max_memory_allocated() / 2 ** 30))
    assert _eq(G.state(), eager_state)
