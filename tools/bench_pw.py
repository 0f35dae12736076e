"""Micro-benchmark of the TF32 wgmma GEMM kernel (gemm_tc.cu) on the encoder's 1x1 projection shapes and the
generator's 3x3 convolution shapes.

    python tools/bench_pw.py [--batch 32] [--reps 20] [--only K72] [--gen]

Encoder shapes: (H, K=mid, N=Cout, residual) of the linear 1x1 projections of tf_mobilenetv3_{large,small}_
minimal_100 at 224x224 (reference src/smirk_encoder.py:7-12).  Generator shapes: (H, Cin, Cout) of the 3x3 convs
of the UNet (reference src/smirk_generator.py:56-76).  CUDA-event means with an L2 flush between launches.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from smirk_b200 import _lib  # noqa: E402

# (H, K, N, residual, launches per encoder pass)
PW = [
    (112, 16, 16, 1, 3), (56, 64, 24, 0, 2), (56, 72, 24, 1, 2), (28, 72, 40, 0, 2), (28, 120, 40, 1, 4),
    (14, 240, 80, 0, 2), (14, 200, 80, 1, 2), (14, 184, 80, 1, 4), (14, 480, 112, 0, 2), (14, 672, 112, 1, 2),
    (7, 672, 160, 0, 2), (7, 960, 160, 1, 4), (7, 160, 960, 0, 2),
    (28, 72, 24, 0, 1), (28, 88, 24, 1, 1), (14, 96, 40, 0, 1), (14, 240, 40, 1, 2), (14, 120, 48, 0, 1),
    (14, 144, 48, 1, 1), (7, 288, 96, 0, 1), (7, 576, 96, 1, 2), (7, 96, 576, 0, 1),
]
# (H, Cin, Cout) 3x3, zero padding
GEN = [(224, 32, 32), (224, 64, 32), (112, 64, 64), (112, 128, 64), (56, 128, 128), (56, 256, 128), (28, 256, 256),
       (28, 512, 256), (14, 512, 512)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--only", default="")
    ap.add_argument("--gen", action="store_true")
    a = ap.parse_args()
    lib = _lib.lib()
    dev = torch.device("cuda:0")
    P = lambda t: t.data_ptr() if t is not None else 0
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    tot = 0.0
    cases = [("pw", H, K, N, res, n) for (H, K, N, res, n) in PW]
    if a.gen:
        cases = [("c3", H, Cin, Cout, 0, 1) for (H, Cin, Cout) in GEN]
    for (kind, H, K, N, res, n) in cases:
        name = "%s_H%d_K%d_N%d%s" % (kind, H, K, N, "_res" if res else "")
        if a.only and a.only not in name:
            continue
        B = a.batch
        x = torch.randn(B, H, H, K, device=dev)
        Kg = K if kind == "pw" else 9 * K
        w = torch.randn(N, Kg, device=dev) / Kg ** 0.5
        sc, bi = torch.rand(N, device=dev) + 0.5, torch.randn(N, device=dev) * 0.2
        r = torch.randn(B, H, H, N, device=dev) if res else None
        out = torch.empty(B, H, H, N, device=dev)

        def run():
            rc = lib.smk_debug_conv_tc(P(x), K, B, H, H, K, P(w), P(sc), P(bi), N, Kg, 0 if kind == "pw" else 1, 0, P(r), N, 0,
                                       P(out), N, 0, st)
            assert rc == 0, lib.smk_last_error()

        for _ in range(3):
            run()
        torch.cuda.synchronize()
        ms = 0.0
        for _ in range(a.reps):
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ms += e0.elapsed_time(e1)
        us = ms / a.reps * 1e3
        nbytes = 4.0 * (x.numel() + out.numel() * (2 if res else 1) + w.numel())
        flops = 2.0 * B * H * H * N * Kg
        print("%-26s x%d  %7.1f us  %7.1f GB/s  %6.1f TFLOP/s  (%.1f MB)" % (name, n, us, nbytes / us * 1e-3, flops / us * 1e-6, nbytes / 1e6))
        tot += us * n
    print("sum: %.1f us" % tot)


if __name__ == "__main__":
    main()
