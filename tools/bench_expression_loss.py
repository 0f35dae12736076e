"""Device time of smirk_b200.ExpressionLoss at B = 32 (the trainer's batch) and B = 256 (gen and tar [B,3,224,224] each),
by default at precisions 1, 3 and 0: the no-grad forward, the grad-mode forward with gen requiring grad (which also keeps
gen's activations) and the backward to gen alone, metric 'l2' with use_mean=False as the trainer calls it.  CUDA-event
mean over `--reps` iterations after warm-up, inputs resident on the device; TFLOP/s from the FLOPs counted from the layer
shapes (FLOPS_PER_IMAGE, two images per face).  Comparison arm: the torch restatement (tests/expression_ref.py) on the
same GPU in torch + cuDNN, with cuDNN's TF32 allowed (the reference's default GPU arithmetic) and in fp32, forward under
no_grad.  Prints the card name, power limit and SM clock read in the same run, the saved and workspace bytes per face,
then the per-kernel breakdown of one grad-mode forward + backward at the largest batch from the library's event
profiler."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib  # noqa: E402
import expression_ref  # noqa: E402


def conv_flops():
    """(S_out, K, N) of every convolution at 224^2 -> FLOPs per image."""
    f = 2.0 * 112 * 112 * 147 * 64
    for _, cin, planes, stride, ds in expression_ref.blocks():
        H = {64: 56, 256: 56, 512: 28, 1024: 14, 2048: 7}[cin]
        Ho = H // stride
        f += 2.0 * H * H * cin * planes + 2.0 * Ho * Ho * 9 * planes * planes + 2.0 * Ho * Ho * planes * 4 * planes
        if ds:
            f += 2.0 * Ho * Ho * cin * 4 * planes
    return f


FLOPS_PER_IMAGE = conv_flops()            # 8.17 GFLOP


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
    ap.add_argument("--precisions", type=int, nargs="+", default=[1, 3, 0])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card (name, power limit, SM clock, max SM clock): %s" % (q.stdout.strip() or "unknown (nvidia-smi: %s)" % q.stderr.strip()))
    print("FLOPs per image %.3f G, per face %.3f G" % (FLOPS_PER_IMAGE / 1e9, 2 * FLOPS_PER_IMAGE / 1e9))
    L = _lib.lib()
    sd = expression_ref.expression_state_dict(7)
    gf = lambda B: 2 * B * FLOPS_PER_IMAGE / 1e9             # noqa: E731
    for B in a.batches:
        gen = expression_ref.probe_images(B, 31).to(dev)
        tar = expression_ref.perturbed(expression_ref.probe_images(B, 31), 31).to(dev)
        sdd = {k: v.to(dev) for k, v in sd.items()}
        old = torch.backends.cudnn.allow_tf32
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            with torch.no_grad():
                t = timed(lambda: expression_ref.expression_loss_ref(sdd, gen, tar, False, "l2"), a.reps)
            print("torch + cuDNN %-5s B=%d  forward %8.2f ms  %6.1f TFLOP/s" % ("tf32" if tf32 else "fp32", B, t, gf(B) / t))
        torch.backends.cudnn.allow_tf32 = old
        del sdd
        torch.cuda.empty_cache()
        for precision in a.precisions:
            m = smirk_b200.ExpressionLoss(checkpoint=None)
            m.load_state_dict(sd)
            m.precision = precision
            m = m.to(dev)
            gg = gen.clone().requires_grad_()
            t_fwd = timed(lambda: m(gen, tar, use_mean=False), a.reps)
            t_gfwd = timed(lambda: m(gg, tar, use_mean=False), a.reps)
            loss = m(gg, tar, use_mean=False).mean()
            t_bwd = timed(lambda: torch.autograd.grad(loss, gg, retain_graph=True), a.reps)
            h = m._native.handle
            saved = L.smk_expression_loss_saved_bytes(h, B, 1) / B / 2 ** 20
            ws = L.smk_expression_loss_workspace_bytes(h, B) / B / 2 ** 20
            bws = L.smk_expression_loss_backward_workspace_bytes(h, B, 1) / B / 2 ** 20
            print("precision %d B=%d  forward %8.2f ms %6.1f TFLOP/s   grad-mode forward %8.2f ms   backward (gen) %8.2f ms %6.1f TFLOP/s"
                  "   per face: saved %.1f MB, forward workspace %.1f MB, backward workspace %.1f MB"
                  % (precision, B, t_fwd, gf(B) / t_fwd, t_gfwd, t_bwd, B * FLOPS_PER_IMAGE / 1e9 / t_bwd, saved, ws, bws))
            if B == max(a.batches):
                L.smk_profiler_reset()
                L.smk_profiler_enable(1)
                torch.autograd.grad(m(gg, tar, use_mean=False).mean(), gg)
                torch.cuda.synchronize()
                L.smk_profiler_enable(0)
                for tag, r in sorted(_lib.profiler_report().items(), key=lambda kv: -kv[1]["ms"]):
                    print("    %-30s %3d launch  %9.3f ms  %7.1f GB/s  %7.2f TFLOP/s" % (
                        tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e9))
            del loss, gg, m
            torch.cuda.empty_cache()
        del gen, tar
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
