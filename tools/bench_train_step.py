"""Time config_train's whole step (tests/train_flow.py: encoder and generator in train mode at precision 3, FLAME,
Renderer, VGG loss, the trainer's masking and cycle augmentation; forward + backward of each path, no optimizer) at
B = 32, Ke = 1, on one GPU, in three arms:

  torch   the masking and augmentation as torch code: the augmentation of tests/cycle_ref.py with its draws made by
          torch's and Python's generators on the host and moved to the device (as the reference makes them) and its
          arithmetic on the device; the masking through ``smirk_b200.masking``'s functions with the reference's
          signatures (``torch.multinomial`` / ``rand`` / ``randn`` / ``bernoulli`` and boolean indexing on the device, which
          sync with the host; their deterministic parts are this project's kernels, as in the other arms);
  device  ``TrainMaskingStage`` and ``CycleAugmentation``, eager;
  graph   the device arm with path1 captured once in a CUDA graph (the second path's frozen network runs the eval path,
          whose handle folds BatchNorm statistics on the host, so it is not captured; its rows repeat the device arm).

Then SmirkTrainer.step as the trainer runs it (tests/test_gpu_train_flow_live.py's Trainer: step1's forward, backward and
Adam steps, then step2 at the batch's freeze parity with its Adam step, the generator's gradient clipped at parity 0),
parities alternating, in three more arms:

  step_host   eager, the second path's frozen network on the host-packed eval handle, rebuilt on every step because the
              first path changed its weights and running statistics;
  step_live   eager, the frozen network on live weights (``live_weights_(True)``: folded and repacked on the device);
  step_graph  step_live captured as two CUDA graphs, one per freeze parity, replayed alternately.

The arms alternate in each of --rounds rounds after --warmup steps; each time is the median over rounds of CUDA-event
times over --iters calls, with [min, max] (the trainer-step arms: per step, over --iters pairs of steps).
--trainer-step-only skips the path arms.  Then per arm and path the CUDA activities of one call (torch.profiler), and
for the device arm the library's event-profiler tags of one whole step (the stages' own times, the largest tags).  The
GPU's name and power limit are read in the same call.  Prints one JSON line.

    python tools/bench_train_step.py [--iters 5] [--warmup 2] [--rounds 5] [--batch 32] [--trainer-step-only]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def timed(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class TorchMasking:
    """The trainer's masking lines (smirk_trainer.py:76-92, :262-293) with the reference-signature functions."""

    def __init__(self, faces, base_prob):
        self.faces, self.base_prob = faces, base_prob

    def first_path(self, img, hull, tv, rendered):
        import cycle_ref
        from smirk_b200 import masking
        pts, _ = masking.mesh_based_mask_uniform_faces(tv.detach(), self.faces, self.base_prob, mask_ratio=0.01)
        extra = masking.transfer_pixels(img, pts, pts)
        return masking.masking(img, hull, extra, 10, rendered_mask=cycle_ref.rendered_mask_first(rendered), flame_faces=self.faces)

    def second_path(self, img, hull, tv, tv2, rendered2, Ke=1):
        import cycle_ref
        from smirk_b200 import masking
        p1, coords = masking.mesh_based_mask_uniform_faces(tv, self.faces, self.base_prob, mask_ratio=0.01)
        coords = {k: v.repeat(Ke, *([1] * (v.dim() - 1))) for k, v in coords.items()}
        p2, _ = masking.mesh_based_mask_uniform_faces(tv2, self.faces, self.base_prob, mask_ratio=0.01, coords=coords)
        extra = masking.transfer_pixels(img.repeat(Ke, 1, 1, 1), p1.repeat(Ke, 1, 1), p2)
        return masking.masking(img.repeat(Ke, 1, 1, 1), hull.repeat(Ke, 1, 1, 1), extra, 10,
                               rendered_mask=cycle_ref.rendered_mask_second(rendered2), extra_noise=True, random_mask=0.005,
                               flame_faces=self.faces)


class TorchAugment:
    """smirk_trainer.py:189-248: host draws in the reference's order, moved to the device, the arithmetic there."""

    def __init__(self, templates):
        self.templates = templates

    def __call__(self, encoder_output, Ke=1):
        import cycle_ref
        B = encoder_output["expression_params"].shape[0]
        dev = encoder_output["expression_params"].device
        d = cycle_ref.augment_draws_ref(Ke * B, encoder_output["expression_params"].shape[1], 2, self.templates)
        return cycle_ref.augment_ref(encoder_output, Ke, {k: v.to(dev) for k, v in d.items()}, self.templates)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--trainer-step-only", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_step needs a GPU"
    import tempfile
    import make_golden_cycle as mgc
    import train_flow as tf
    from smirk_b200 import _lib, synth_assets
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_bench_train_step"))
    old = os.getcwd()
    os.chdir(root)
    try:
        bases = tf.make_bases(root)
    finally:
        os.chdir(old)
    B = args.batch
    gpu = {"gpu": torch.cuda.get_device_properties(0).name, "power_limit_w": power_limit_w(), "B": B, "Ke": 1, "precision": 3}
    step_ms = trainer_steps(tf, bases, B, args)
    if args.trainer_step_only:
        print(json.dumps(dict(gpu, trainer_step_ms_median_min_max=step_ms)))
        return
    batch = tf.make_batch(B, 7)
    flows = {"torch": tf.TrainFlow(bases, 3, seed=1), "device": tf.TrainFlow(bases, 3, seed=1), "graph": tf.TrainFlow(bases, 3, seed=1)}
    flows["torch"].masking = TorchMasking(bases["faces"], bases["base_prob"])
    flows["torch"].augment = TorchAugment(mgc.synthetic_templates())

    def calls(flow, eo):
        return (lambda: flow.path1(batch), lambda: flow.path2(eo, batch, 0), lambda: flow.path2(eo, batch, 1))

    eo = flows["device"].path1(batch)[2]
    arms = {}
    for name in ("torch", "device"):
        arms[name] = calls(flows[name], eo)
        for fn in arms[name]:
            for _ in range(args.warmup):
                fn()
    G = flows["graph"]
    static = {k: v.clone() for k, v in batch.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        G.path1(static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        G.path1(static)
    graph.replay()
    arms["graph"] = (graph.replay,) + arms["device"][1:]
    names = ("step1", "step2_parity0", "step2_parity1")
    times = {a: {n: [] for n in names} for a in arms}
    for _ in range(args.rounds):
        for a, fns in arms.items():
            for n, fn in zip(names, fns):
                times[a][n].append(timed(fn, args.iters))
    ms = {a: {n: [round(statistics.median(v), 3), round(min(v), 3), round(max(v), 3)] for n, v in t.items()} for a, t in times.items()}

    from torch.profiler import ProfilerActivity, profile
    activities = {}
    for a, fns in arms.items():
        for n, fn in zip(names, fns):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            activities["%s/%s" % (a, n)] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    L = _lib.lib()
    L.smk_profiler_reset()
    L.smk_profiler_enable(1)
    for fn in arms["device"]:
        fn()
    torch.cuda.synchronize()
    L.smk_profiler_enable(0)
    rep = _lib.profiler_report()
    stage = {k: round(v["ms"], 4) for k, v in rep.items() if k.startswith(("mask_", "cycle_"))}
    top = dict(sorted(((k, round(v["ms"], 3)) for k, v in rep.items()), key=lambda kv: -kv[1])[:8])
    print(json.dumps(dict(gpu, ms_median_min_max=ms, cuda_activities_per_call=activities, device_step_stage_ms=stage,
                          device_step_top_tags_ms=top, trainer_step_ms_median_min_max=step_ms)))


def trainer_steps(tf, bases, B, args):
    """-> {arm: [median, min, max] ms per SmirkTrainer.step} of the step_host / step_live / step_graph arms."""
    from test_gpu_train_flow_live import Trainer
    data = [tf.make_batch(B, 70 + s) for s in range(2)]
    trainers = {"step_host": Trainer(tf.TrainFlow(bases, 3, seed=1)), "step_live": Trainer(tf.TrainFlow(bases, 3, seed=1)),
                "step_graph": Trainer(tf.TrainFlow(bases, 3, seed=1))}
    for name in ("step_live", "step_graph"):
        trainers[name].flow.enc.live_weights_(True)
        trainers[name].flow.gen.live_weights_(True)
    fns = {}
    for name in ("step_host", "step_live"):
        t = trainers[name]
        fns[name] = lambda t=t: (t.step(data[0], 0), t.step(data[1], 1))
    G = trainers["step_graph"]
    static = [{k: v.clone() for k, v in d.items()} for d in data]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for parity in (0, 1):
            G.step(static[parity], parity)
    torch.cuda.current_stream().wait_stream(s)
    graphs = []
    for parity in (0, 1):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=graphs[0].pool() if graphs else None):     # replayed in capture order
            G.step(static[parity], parity)
        graphs.append(g)
    fns["step_graph"] = lambda: (graphs[0].replay(), graphs[1].replay())
    for fn in fns.values():
        for _ in range(args.warmup):
            fn()
    times = {n: [] for n in fns}
    for _ in range(args.rounds):
        for n, fn in fns.items():
            times[n].append(timed(fn, args.iters) / 2)
    return {n: [round(statistics.median(v), 3), round(min(v), 3), round(max(v), 3)] for n, v in times.items()}


if __name__ == "__main__":
    main()
