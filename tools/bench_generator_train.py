"""Time the generator's train mode on one GPU: eval forward, train forward, train backward and one SGD step, at the trainer's
configuration (6, 3, 32, 5) and B = 32 (config_train's batch) and 64, precisions 0 and 3.  CUDA events over --iters
calls after --warmup; then one profiled step per case (the library's event profiler) for the largest tags and the 3x3
weight gradient's achieved FLOP/s (FLOPs from shapes, 2 M cout 9 cin per layer).  Prints one JSON line per case.
Per batch size one more line times the train-mode oracle (tests/generator_train_ref: oracle/generator_ref with torch's
train-mode BatchNorm) on torch + cuDNN on the same GPU, in fp32 (cuDNN's TF32 off) and with cuDNN's TF32: the train
forward and forward + backward, every parameter's gradient included.  The GPU's name and power limit go on every line.

    python tools/bench_generator_train.py [--iters 5] [--warmup 2] [--batch 32 64] [--precision 0 3]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit_w():
    """The GPU's power limit (nvidia-smi query), or None where it cannot be read."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--precision", type=int, nargs="+", default=[0, 3])
    args = ap.parse_args()
    import smirk_b200
    from smirk_b200 import _lib, synth_inputs
    assert torch.cuda.is_available(), "bench_generator_train needs a GPU"
    dev = "cuda"
    props = torch.cuda.get_device_properties(0)
    gpu = {"gpu": props.name, "power_limit_w": power_limit_w()}
    base = smirk_b200.SmirkGenerator(6, 3, 32, 5)
    base.load_state_dict(synth_inputs.random_state_dict(base.state_dict(), seed=7))
    for B in args.batch:
        x = torch.cat([synth_inputs.images(B, 1), synth_inputs.masked_images(B, 2)], 1).to(dev)
        gy = torch.randn(B, 3, 224, 224, device=dev)
        for precision in args.precision:
            g = copy.deepcopy(base).to(dev)
            g.precision = precision
            ev = g.eval()
            with torch.no_grad():
                t_eval = timed(lambda: ev(x), args.iters, args.warmup)
            g.train().allow_train_mode_(True)
            with torch.no_grad():
                t_fwd = timed(lambda: g(x), args.iters, args.warmup)
            params = list(g.parameters())
            holder = {}

            def fwd():
                holder["y"] = g(x)

            def bwd():
                torch.autograd.grad(holder["y"], params, gy)
            fwd()
            bwd()
            torch.cuda.synchronize()
            t_fb = timed(lambda: (fwd(), bwd()), args.iters, args.warmup)
            opt = torch.optim.SGD(params, lr=1e-4)

            def step():
                opt.zero_grad(set_to_none=True)
                (g(x) * gy).mean().backward()
                opt.step()
            t_step = timed(step, args.iters, args.warmup)
            torch.cuda.synchronize()
            L = _lib.lib()
            L.smk_profiler_reset()
            L.smk_profiler_enable(1)
            step()
            torch.cuda.synchronize()
            L.smk_profiler_enable(0)
            rep = _lib.profiler_report()
            total = sum(v["ms"] for v in rep.values())
            top = sorted(rep.items(), key=lambda kv: -kv[1]["ms"])[:8]
            wg = rep.get("conv3_wgrad", {"ms": 0.0, "flops": 0.0})
            print(json.dumps({
                **gpu, "B": B, "precision": precision,
                "eval_forward_ms": round(t_eval, 3), "train_forward_ms": round(t_fwd, 3),
                "train_backward_ms": round(t_fb - t_fwd, 3), "train_forward_backward_ms": round(t_fb, 3), "sgd_step_ms": round(t_step, 3),
                "profiled_step_ms": round(total, 3),
                "top_tags": {k: {"ms": round(v["ms"], 3), "share": round(v["ms"] / total, 4), "launches": v["launches"]} for k, v in top},
                "conv3_wgrad_tflops": round(wg["flops"] / (wg["ms"] * 1e-3) / 1e12, 2) if wg["ms"] else None,
            }), flush=True)
            del g, ev, opt, holder
        print(json.dumps({**gpu, "B": B, "arm": "torch + cuDNN train-mode oracle", **oracle_arm(base, x, gy, args)}), flush=True)


def oracle_arm(base, x, gy, args):
    """Train forward and forward + backward of the train-mode oracle on x's device, fp32 and cuDNN TF32."""
    import generator_train_ref as gtr
    out = {}
    old = torch.backends.cudnn.allow_tf32
    try:
        for name, tf32 in (("fp32", False), ("tf32", True)):
            torch.backends.cudnn.allow_tf32 = tf32
            sd = gtr.cpu_state(base, x.device)
            params = [v for v in sd.values() if v.requires_grad]
            with torch.no_grad():
                t_fwd = timed(lambda: gtr.generator_train_ref(sd, x, res_blocks=5), args.iters, args.warmup)
            t_fb = timed(lambda: torch.autograd.grad(gtr.generator_train_ref(sd, x, res_blocks=5), params, gy), args.iters, args.warmup)
            out[name] = {"train_forward_ms": round(t_fwd, 3), "train_backward_ms": round(t_fb - t_fwd, 3), "train_forward_backward_ms": round(t_fb, 3)}
    finally:
        torch.backends.cudnn.allow_tf32 = old
    return out


if __name__ == "__main__":
    main()
