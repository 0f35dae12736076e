"""Experiment: the windowed 3x3 kernel (conv3_win_tc.cu) vs the im2col kernel (gemm_tc.cu), 224^2 x Cin -> 32.
tc_conv sends zero-padded 3x3 layers of this shape to the windowed kernel, so the im2col arm feeds gemm_tc an explicitly
zero-padded input (mode 2), which computes the same convolution.
    python tools/bench_win.py [--batch 256] [--cin 32]"""
import argparse, ctypes as C, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from smirk_b200 import _lib

ap = argparse.ArgumentParser(); ap.add_argument("--batch", type=int, default=256); ap.add_argument("--cin", type=int, default=32); a = ap.parse_args()
lib = _lib.lib(); vp, i = C.c_void_p, C.c_int
dev = torch.device("cuda:0"); B, H, Cin, N = a.batch, 224, a.cin, 32
x = torch.randn(B, H, H, Cin, device=dev); w = torch.randn(N, 9 * Cin, device=dev) / (9 * Cin) ** 0.5
sc, bi = torch.rand(N, device=dev) + 0.5, torch.randn(N, device=dev) * 0.1
xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1)).contiguous()
o1, o2 = torch.empty(B, H, H, N, device=dev), torch.empty(B, H, H, N, device=dev)
st = torch.cuda.current_stream().cuda_stream
P = lambda t: t.data_ptr()
def win(): assert lib.smk_debug_conv3_win(P(x), Cin, B, H, H, Cin, P(w), P(sc), P(bi), N, 1, P(o1), N, st) == 0, lib.smk_last_error()
def im2col():
    assert lib.smk_debug_conv_tc(P(xp), Cin, B, H, H, Cin, P(w), P(sc), P(bi), N, 9 * Cin, 2, 1, 0, N, 0, P(o2), N, 0, st) == 0, lib.smk_last_error()
for name, fn in (("win", win), ("im2col", im2col)):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): fn()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 5 * 1e3
    print("%-7s B=%d Cin=%d: %8.1f us  %6.1f TFLOP/s" % (name, B, Cin, us, 2.0 * B * H * H * N * 9 * Cin / us * 1e-6))
print("max |win - im2col| = %.3g" % float((o1 - o2).abs().max()))
