"""Device time of smirk_b200.MICA's forward at B = 32 and B = 256 (images [B,3,112,112]), by default at precisions 1, 3
and 0.  CUDA-event mean over `--reps` iterations after warm-up, inputs resident on the device; TFLOP/s from 24.18 GFLOP
per image (FLOPS_PER_IMAGE, counted from the layer shapes).  Comparison arm: the torch restatement (tests/mica_ref.py) on
the same GPU in torch + cuDNN, fp32 and with cuDNN's TF32 allowed (the reference's default GPU arithmetic), under no_grad.
Also: each precision's max-abs error over max-abs of shape_params and of the ArcFace features against the fp32
restatement at B = 32, with cuDNN TF32's own beside it; a pretraining-shaped step (train-mode encoder, FLAME, Renderer,
landmark + expression losses, SGD) at B = 32 with and without 10 * the MICA shape loss; and the per-kernel breakdown of
one forward at the largest batch from the library's event profiler.  Prints the card name, power limit and SM clock read
in the same run."""
import argparse
import os
import subprocess
import sys
import tempfile

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_assets, synth_inputs  # noqa: E402
import mica_ref  # noqa: E402


def _flops_per_image():
    f, S = 2.0 * 112 * 112 * 9 * 3 * 64, 112
    for _, cin, cout, stride in mica_ref.blocks():
        f += 2.0 * S * S * 9 * cin * cout                    # conv1 at the input size
        S //= stride
        f += 2.0 * S * S * 9 * cout * cout                   # conv2 at the output size
        if stride == 2:
            f += 2.0 * S * S * cin * cout                    # downsample
    return f + 2.0 * 25088 * 512 + 2.0 * (512 * 300 + 3 * 300 * 300 + 300 * 300)


FLOPS_PER_IMAGE = _flops_per_image()                     # 24.18 GFLOP (12.09 GMAC)


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


def err(a, ref):
    return ((a.double() - ref.double()).abs().max() / ref.double().abs().max()).item()


def make(sd, precision, dev):
    m = smirk_b200.MICA(checkpoint=None)
    m.load_state_dict(sd)
    for p in m.parameters():
        p.requires_grad = False
    m = m.eval().to(dev)
    m.precision = precision
    return m


def pretrain_step_ms(dev, mica_precision, reps):
    """Mean device time of one pretraining-shaped SGD step at B = 32, without (None) or with MICA at that precision."""
    old = os.getcwd()
    os.chdir(synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_bench_mica")))
    try:
        B = 32
        enc = smirk_b200.SmirkEncoder()
        enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
        enc = enc.to(dev).train().allow_train_mode_(True)
        fl, rd = smirk_b200.FLAME().to(dev), smirk_b200.Renderer().to(dev)
        mica = make(mica_ref.mica_state_dict(7, check=False), mica_precision, dev) if mica_precision is not None else None
        g = torch.Generator().manual_seed(5)
        tgt_fan, tgt_mp = (torch.rand(B, 68, 2, generator=g) - 0.5).to(dev), (torch.rand(B, 105, 2, generator=g) - 0.5).to(dev)
        img, img_mica = synth_inputs.images(B, 3).to(dev), mica_ref.probe_images(B, 4).to(dev)
        opt = torch.optim.SGD(enc.parameters(), lr=1e-7)

        def step():
            opt.zero_grad()
            out = enc(img)
            fo = fl(out)
            ro = rd(fo["vertices"], out["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
            loss = 100.0 * (F.mse_loss(ro["landmarks_fan"][:, :17, :2], tgt_fan[:, :17]) + F.mse_loss(ro["landmarks_mp"][..., :2], tgt_mp))
            loss = loss + 1e-2 * torch.sum(out["expression_params"] ** 2) / B
            if mica is not None:
                loss = loss + 10.0 * mica.calculate_mica_shape_loss(out["shape_params"], img_mica)
            loss.backward()
            opt.step()
        return timed(step, reps)
    finally:
        os.chdir(old)


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
    print("FLOP per image: %.2f G" % (FLOPS_PER_IMAGE / 1e9))
    L = _lib.lib()
    sd = mica_ref.mica_state_dict(7, check=False)
    sdd = {k: v.to(dev) for k, v in sd.items()}
    gf = lambda B: B * FLOPS_PER_IMAGE / 1e9                                              # noqa: E731
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    img = mica_ref.probe_images(32, 9).to(dev)
    with torch.no_grad():
        torch.backends.cudnn.allow_tf32 = False
        ref_s, ref_f = mica_ref.mica_ref(sdd, img)
        torch.backends.cudnn.allow_tf32 = True
        t_s, t_f = mica_ref.mica_ref(sdd, img)
    print("accuracy at B=32 vs the fp32 restatement (max-abs err / max-abs): cuDNN TF32 shape %.2e features %.2e"
          % (err(t_s, ref_s), err(t_f, ref_f)))
    for precision in a.precisions:
        m = make(sd, precision, dev)
        print("    precision %d: shape %.2e features %.2e" % (precision, err(m(img)["shape_params"], ref_s),
                                                               err(m.arcface_features(img), ref_f)))
        del m
    for B in a.batches:
        x = mica_ref.probe_images(B, 31).to(dev)
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            with torch.no_grad():
                t = timed(lambda: mica_ref.mica_ref(sdd, x), a.reps)
            print("torch + cuDNN %-5s B=%3d  forward %8.2f ms  %6.1f TFLOP/s" % ("tf32" if tf32 else "fp32", B, t, gf(B) / t))
        for precision in a.precisions:
            m = make(sd, precision, dev)
            t = timed(lambda: m(x), a.reps)
            print("precision %d   B=%3d  forward %8.2f ms  %6.1f TFLOP/s" % (precision, B, t, gf(B) / t))
            if B == max(a.batches):
                L.smk_profiler_reset()
                L.smk_profiler_enable(1)
                m(x)
                torch.cuda.synchronize()
                L.smk_profiler_enable(0)
                for tag, r in sorted(_lib.profiler_report().items(), key=lambda kv: -kv[1]["ms"]):
                    print("    %-24s %3d launch  %9.3f ms  %7.1f GB/s  %7.2f TFLOP/s" % (
                        tag, r["launches"], r["ms"], r["bytes"] / max(r["ms"], 1e-9) / 1e6, r["flops"] / max(r["ms"], 1e-9) / 1e9))
            del m
            torch.cuda.empty_cache()
        del x
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    del sdd
    torch.cuda.empty_cache()
    base = pretrain_step_ms(dev, None, a.reps)
    print("pretraining-shaped step B=32 (train-mode encoder, FLAME, Renderer, SGD): without MICA %.2f ms" % base)
    for precision in a.precisions:
        t = pretrain_step_ms(dev, precision, a.reps)
        print("    with 10 * MICA shape loss at precision %d: %.2f ms (MICA's share %.0f %%)" % (precision, t, 100.0 * (t - base) / t))


if __name__ == "__main__":
    main()
