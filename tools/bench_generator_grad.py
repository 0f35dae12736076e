"""Device time of the SmirkGenerator forward alone, the grad-mode forward (which also stores the activations the
backward needs) and the input-gradient backward alone, frozen weights, at B = 32 and B = 256, by default precision 1 (TF32 wgmma)
and precision 0 (fp32 CUDA cores) for reference; `--precisions 3 1 0` adds the 3xTF32 tensor-core path.  CUDA-event mean over `--reps` iterations after warm-up; inputs resident
on the device.  Prints the card name and power limit read in the same run, then the per-kernel breakdown of one grad-mode
forward + backward from the library's event profiler (smk_profiler_*), with TFLOP/s per tag."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_inputs  # noqa: E402


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
    ap.add_argument("--precisions", type=int, nargs="+", default=[1, 0])
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card: %s" % (q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()))
    L = _lib.lib()
    for precision in a.precisions:
        g = smirk_b200.SmirkGenerator(6, 3, 32, 5)
        g.load_state_dict(synth_inputs.random_state_dict(g.state_dict(), seed=7))
        g.precision = precision
        g = g.eval().requires_grad_(False).to(dev)
        for B in a.batches:
            x = torch.cat([synth_inputs.images(B, 21), synth_inputs.masked_images(B, 22)], 1).to(dev)
            gy = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(23)).to(dev)
            xg = x.clone().requires_grad_()
            t_fwd = timed(lambda: g(x), a.reps)
            t_gfwd = timed(lambda: g(xg), a.reps)
            y = g(xg)
            t_bwd = timed(lambda: torch.autograd.grad(y, xg, gy, retain_graph=True), a.reps)
            mem = g._native_workspace("backward", 0, dev).numel() / 2 ** 20
            print("precision %d B=%d  forward %.3f ms   grad-mode forward %.3f ms   backward %.3f ms (%.2fx the forward)   "
                  "saved %.0f MB, backward workspace %.0f MB" % (precision, B, t_fwd, t_gfwd, t_bwd, t_bwd / t_fwd,
                                                                   L.smk_generator_saved_bytes(g._native.handle, B) / 2 ** 20, mem))
            del y
            L.smk_profiler_reset()
            L.smk_profiler_enable(1)
            torch.autograd.grad(g(xg), xg, gy)
            torch.cuda.synchronize()
            L.smk_profiler_enable(0)
            for tag, r in sorted(_lib.profiler_report().items(), key=lambda kv: -kv[1]["ms"]):
                print("    %-22s %3d launch  %8.3f ms  %7.1f GB/s  %7.2f TFLOP/s" % (
                    tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e9))
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
