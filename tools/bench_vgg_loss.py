"""Device time of smirk_b200.VGGPerceptualLoss at B = 32 and B = 256 (x and y [B,3,224,224] each), by default at precisions
3, 1 and 0: the no-grad forward, the grad-mode forward with x requiring grad (which also keeps x's activations and the sign
maps) and the backward to x alone.  CUDA-event mean over `--reps` iterations after warm-up, inputs resident on the device;
TFLOP/s from the FLOPs counted from the layer shapes (FLOPS_PER_IMAGE; the dgrad chain runs the same convolutions over x's
half only, less conv1_1's whose gradient is not needed past the input).  Comparison arm: the torch restatement
(tests/vgg_ref.py) on the same GPU in torch + cuDNN, fp32 and with cuDNN's TF32 allowed (the reference's default GPU
arithmetic), forward under no_grad.  Prints the card name, power limit and SM clock read in the same run, then the
per-kernel breakdown of one grad-mode forward + backward at the largest batch from the library's event profiler."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_inputs  # noqa: E402
import vgg_ref  # noqa: E402

# (S, Cin, Cout) of the ten 3x3 convolutions
LAYERS = [(224, 3, 64), (224, 64, 64), (112, 64, 128), (112, 128, 128), (56, 128, 256), (56, 256, 256), (56, 256, 256),
          (28, 256, 512), (28, 512, 512), (28, 512, 512)]
FLOPS_PER_IMAGE = sum(2.0 * S * S * 9 * ci * co for S, ci, co in LAYERS)       # 27.9 GFLOP (13.96 GMAC)
DGRAD_FLOPS_PER_IMAGE = sum(2.0 * S * S * 9 * ci * co for S, ci, co in LAYERS[1:]) + 2.0 * 224 * 224 * 9 * 64 * 3


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
    ap.add_argument("--precisions", type=int, nargs="+", default=[3, 1, 0])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card (name, power limit, SM clock, max SM clock): %s" % (q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()))
    L = _lib.lib()
    sd = vgg_ref.vgg_state_dict(smirk_b200.VGGPerceptualLoss(weights=None).state_dict(), seed=7)
    fwd_gf = lambda B: 2 * B * FLOPS_PER_IMAGE / 1e9
    for B in a.batches:
        x = (synth_inputs.images(B, 31) * 2 - 1).to(dev)
        y = (synth_inputs.images(B, 32) * 2 - 1).to(dev)
        sdd = {k: v.to(dev) for k, v in sd.items()}
        old = torch.backends.cudnn.allow_tf32
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            with torch.no_grad():
                t = timed(lambda: vgg_ref.vgg_loss_ref(sdd, x, y), a.reps)
            print("torch + cuDNN %-5s B=%d  forward %8.2f ms  %6.1f TFLOP/s" % ("tf32" if tf32 else "fp32", B, t, fwd_gf(B) / t))
        torch.backends.cudnn.allow_tf32 = old
        del sdd
        for precision in a.precisions:
            m = smirk_b200.VGGPerceptualLoss(weights=None)
            m.load_state_dict(sd)
            m.precision = precision
            m = m.to(dev)
            xg = x.clone().requires_grad_()
            t_fwd = timed(lambda: m(x, y), a.reps)
            t_gfwd = timed(lambda: m(xg, y), a.reps)
            loss = m(xg, y)
            t_bwd = timed(lambda: torch.autograd.grad(loss, xg, retain_graph=True), a.reps)
            saved = L.smk_vgg_loss_saved_bytes(m._native.handle, B, 1) / 2 ** 20
            print("precision %d B=%d  forward %8.2f ms %6.1f TFLOP/s   grad-mode forward %8.2f ms   backward (x) %8.2f ms %6.1f TFLOP/s"
                  "   saved %.0f MB" % (precision, B, t_fwd, fwd_gf(B) / t_fwd, t_gfwd, t_bwd, B * DGRAD_FLOPS_PER_IMAGE / 1e9 / t_bwd, saved))
            if B == max(a.batches):
                L.smk_profiler_reset()
                L.smk_profiler_enable(1)
                torch.autograd.grad(m(xg, y), xg)
                torch.cuda.synchronize()
                L.smk_profiler_enable(0)
                for tag, r in sorted(_lib.profiler_report().items(), key=lambda kv: -kv[1]["ms"]):
                    print("    %-24s %3d launch  %9.3f ms  %7.1f GB/s  %7.2f TFLOP/s" % (
                        tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e9))
            del loss, xg, m
            torch.cuda.empty_cache()
        del x, y
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
