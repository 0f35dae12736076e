"""Device time of FLAME + Renderer forward + backward (the autograd route: FLAME -> Renderer with landmarks_fan /
landmarks_mp -> two landmark MSE losses + an L1 on rendered_img -> backward), and of the forward and the backward
alone, at B = 32 and B = 256, with the face-mask renderer or, with --full-head, Renderer(render_full_head=True).
CUDA-event mean over `--reps` iterations after warm-up; inputs resident on the device.  Prints the card name and
power limit read in the same run, then the per-kernel breakdown of one forward + backward from the library's event
profiler (smk_profiler_*)."""
import argparse
import os
import subprocess
import sys
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_assets, synth_inputs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--full-head", action="store_true", help="Renderer(render_full_head=True): 5023 vertices, 9976 faces")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card: %s" % (q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()))
    os.chdir(synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_bench_grad")))
    fl, rd = smirk_b200.FLAME().to(dev), smirk_b200.Renderer(render_full_head=a.full_head).to(dev)
    print("renderer: %s (%d faces)" % ("full head" if a.full_head else "face mask", rd.faces.shape[1]))
    L = _lib.lib()

    for B in a.batches:
        p = {k: v.to(dev).requires_grad_() for k, v in synth_inputs.flame_params(B, 11).items()}
        g = torch.Generator().manual_seed(12)
        tgt = {"fan": torch.randn(B, 68, 2, generator=g).to(dev), "mp": torch.randn(B, 105, 2, generator=g).to(dev),
               "img": torch.rand(B, 3, 224, 224, generator=g).to(dev)}

        def fwd():
            fo = fl(p)
            ro = rd(fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
            return (F.mse_loss(ro["landmarks_fan"][:, :17], tgt["fan"][:, :17]) + F.mse_loss(ro["landmarks_mp"], tgt["mp"])
                    + F.l1_loss(ro["rendered_img"], tgt["img"]))

        def step():
            torch.autograd.grad(fwd(), list(p.values()))

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            step()
        e1.record()
        torch.cuda.synchronize()
        t_step = e0.elapsed_time(e1) / a.reps
        e0.record()
        for _ in range(a.reps):                        # forward alone: the autograd route's forward, losses included
            fwd()
        e1.record()
        torch.cuda.synchronize()
        t_fwd = e0.elapsed_time(e1) / a.reps
        t_bwd = 0.0
        for _ in range(a.reps):                        # backward alone: events around torch.autograd.grad only
            loss = fwd()
            b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b0.record()
            torch.autograd.grad(loss, list(p.values()))
            b1.record()
            torch.cuda.synchronize()
            t_bwd += b0.elapsed_time(b1)
        t_bwd /= a.reps
        print("B=%d  forward+backward %.3f ms (%.0f faces/s)   forward alone %.3f ms   backward alone %.3f ms"
              % (B, t_step, B / t_step * 1e3, t_fwd, t_bwd))
        L.smk_profiler_reset()
        L.smk_profiler_enable(1)
        step()
        torch.cuda.synchronize()
        L.smk_profiler_enable(0)
        for tag, r in sorted(_lib.profiler_report().items(), key=lambda kv: -kv[1]["ms"]):
            print("    %-20s %3d launch  %8.3f ms  %7.1f GB/s  %7.1f GFLOP/s" % (
                tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e6))


if __name__ == "__main__":
    main()
