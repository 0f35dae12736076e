"""Device time of the train-mode SmirkEncoder: the forward alone (batch-statistics BatchNorm, running-statistics update),
the backward alone (every parameter and the image get a gradient), and a pretraining-shaped step (encoder -> FLAME ->
Renderer -> landmark MSE + expression regularisation -> backward), at B = 32 and B = 256, precisions 3 and 0, next to the
eval forward and the grad-mode (input-gradient) forward.  CUDA-event mean over `--reps` iterations after warm-up; inputs
resident on the device.  Prints the card name and power limit read in the same run, the saved bytes per face, and the
per-kernel breakdown of one forward + backward from the library's event profiler."""
import argparse
import copy
import os
import subprocess
import sys
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_assets, synth_inputs  # noqa: E402


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--precisions", type=int, nargs="+", default=[3, 0])
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card: %s" % (q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()))
    os.chdir(synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_bench_train")))
    fl, rd = smirk_b200.FLAME().to(dev), smirk_b200.Renderer().to(dev)
    L = _lib.lib()
    base = smirk_b200.SmirkEncoder()
    base.load_state_dict(synth_inputs.random_state_dict(base.state_dict(), seed=7))
    for precision in a.precisions:
        ev = copy.deepcopy(base).eval().requires_grad_(False).to(dev)
        tm = copy.deepcopy(base).train().allow_train_mode_(True).to(dev)
        for m in (ev, tm, ev.pose_encoder, ev.shape_encoder, ev.expression_encoder, tm.pose_encoder, tm.shape_encoder, tm.expression_encoder):
            m.precision = precision
        params = list(tm.parameters())
        for B in a.batches:
            x = synth_inputs.images(B, 21).to(dev)
            xg = x.clone().requires_grad_()
            gen = torch.Generator().manual_seed(23)
            tgt = {"fan": (torch.rand(B, 68, 2, generator=gen) - 0.5).to(dev), "mp": (torch.rand(B, 105, 2, generator=gen) - 0.5).to(dev)}
            t_eval = timed(lambda: ev(x), a.reps)
            t_gfwd = timed(lambda: ev(xg), a.reps)
            with torch.no_grad():
                t_tfwd_ng = timed(lambda: tm(x), a.reps)
            t_tfwd = timed(lambda: tm(x), a.reps)
            out = tm(x)
            ys = [out[k] for k in sorted(out)]
            gys = [torch.randn(y.shape, generator=gen).to(dev) for y in ys]
            t_bwd = timed(lambda: torch.autograd.grad(ys, params, gys, retain_graph=True), a.reps)

            def step():
                o = tm(x)
                fo = fl(o)
                ro = rd(fo["vertices"], o["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
                loss = 100.0 * (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])) \
                    + 1e-2 * torch.sum(o["expression_params"] ** 2) / B
                torch.autograd.grad(loss, params)
            t_step = timed(step, a.reps)
            saved = L.smk_encoder_saved_bytes(tm._native.train_handle, B)
            print("precision %d B=%d  eval forward %.3f ms  grad-mode forward %.3f ms  train forward %.3f ms (no grad %.3f)  "
                  "train backward %.3f ms  pretrain step %.3f ms  saved %.1f MB/face" % (
                      precision, B, t_eval, t_gfwd, t_tfwd, t_tfwd_ng, t_bwd, t_step, saved / B / 1e6))
            del out, ys
            L.smk_profiler_reset()
            L.smk_profiler_enable(1)
            out = tm(x)
            torch.autograd.grad([out[k] for k in sorted(out)], params, gys)
            torch.cuda.synchronize()
            L.smk_profiler_enable(0)
            rep = _lib.profiler_report()
            print("    %d launches per train forward + backward" % sum(r["launches"] for r in rep.values()))
            for tag, r in sorted(rep.items(), key=lambda kv: -kv[1]["ms"]):
                print("    %-22s %4d launch  %8.3f ms  %7.1f GB/s  %7.2f TFLOP/s" % (
                    tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e9))
            del out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
