"""configs[3]: the video demo's frame loop (demo_video.py [--crop] [--render_orig] [--use_smirk_generator]) at 1080p (or --frame-hw),
batch 64 frames per step, frame-sharded over the GPUs of a torchrun job (``shard_bounds``; each rank keeps its grids, no all-gather: their consumer
is the host video writer, and every GPU has its own PCIe link).  Prints one JSON line:

  device_fps     frames/s with the frames resident in HBM: graph replay over the lanes, CUDA events around exactly
                 --steps steps after --warmup, the slowest rank's time
  e2e_fps        frames/s from pinned host frames to pinned host grids (run_host), with the H2D / D2H bytes per frame
  stages         per-tag device time of one eager batch from the library's event profiler; GB/s of video_compose and of
                 the crop warp (warp_minmax + warp_bilinear) from their algorithmic bytes
  gpu            card name, power limit and SM clocks read in the same run (read-only nvidia-smi queries)
  cpu_baseline   the reference's per-frame loop on the host cores over --cpu-frames frames: crop and warp back with the
                 scikit-image restatement (oracle/warp_ref.py), or without the crop cv2.resize and torch's CPU F.interpolate;
                 the oracle port of encoder -> FLAME -> renderer, the grid

    python tools/bench_video.py [--render-orig] [--generator] [--no-crop] [--frame-hw 512x512]
    torchrun --nproc-per-node 2 tools/bench_video.py [--render-orig] [--generator]

The CPU baseline covers the loop without the generator (its hull mask and masking step are not timed there).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import smirk_b200  # noqa: E402
from smirk_b200 import _lib, synth_assets, synth_inputs, video  # noqa: E402
from smirk_b200.pipeline import SmirkPipeline, shard_bounds  # noqa: E402


def landmarks(rng, B, H, W):
    """Face-sized landmark clouds, placed as in a 1080 x 1920 frame scaled to H x W."""
    c = np.stack([rng.uniform(W * 500 / 1920, W * 1420 / 1920, B), rng.uniform(H * 300 / 1080, H * 780 / 1080, B)], 1)[:, None]
    return c + rng.normal(0, 1, (B, 478, 2)) * rng.uniform(40, 110, (B, 1, 1)) * (min(H, W) / 1080)


def cpu_baseline(root, frames, lm, render_orig, crop):
    """The reference's per-frame loop (demo_video.py:121-213) on the host: seconds per frame."""
    import torch.nn.functional as F
    from oracle import warp_ref, encoder_ref, flame_ref, render_ref
    st = bench._CPU_STATE
    if "enc_sd" not in st:
        st["enc_sd"] = synth_inputs.random_state_dict(smirk_b200.SmirkEncoder().state_dict(), seed=7)
        st["fc"], st["rc"] = flame_ref.FlameConstants(root), render_ref.RenderConstants(root)
    t0 = time.perf_counter()
    for f, l in zip(frames, lm):
        if crop:
            T = warp_ref.crop_face_ref(f.shape, l, 1.4, 224)
            c = warp_ref.warp_ref(f, np.linalg.inv(T), (224, 224))
        else:
            import cv2
            c = cv2.resize(cv2.cvtColor(f, cv2.COLOR_BGR2RGB), (224, 224))[..., ::-1]
        img = torch.from_numpy(np.ascontiguousarray(c[..., ::-1].transpose(2, 0, 1)))[None].float() / 255.0
        with torch.no_grad():
            p = {k: v for k, v in encoder_ref.encoder_forward_ref(st["enc_sd"], img).items() if not k.startswith("_")}
            fo = flame_ref.flame_forward_ref(st["fc"], p)
            r = render_ref.render_forward_ref(st["rc"], fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"],
                                              landmarks_mp=fo["landmarks_mp"])["rendered_img"][0].numpy()
        if render_orig and not crop:
            up = F.interpolate(torch.from_numpy(r)[None], f.shape[:2], mode='bilinear')[0].numpy()
            np.concatenate([f, ((up.transpose(1, 2, 0) * np.float32(255.0)).astype(np.uint8))[..., ::-1]], 1)
        elif render_orig:
            np.concatenate([f, warp_ref.warp_back_ref(r, T, f.shape[:2])[..., ::-1]], 1)
        else:
            np.concatenate([c, ((r.transpose(1, 2, 0) * np.float32(255.0)).astype(np.uint8))[..., ::-1]], 1)
    return (time.perf_counter() - t0) / len(frames)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64, help="frames per step over all GPUs")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--slots", type=int, default=2)
    ap.add_argument("--render-orig", action="store_true")
    ap.add_argument("--generator", action="store_true", help="--use_smirk_generator: hull mask, masking step, generator panel")
    ap.add_argument("--no-crop", action="store_true", help="demo_video.py without --crop: the whole frame resized")
    ap.add_argument("--frame-hw", default="1080x1920", help="frame height x width, e.g. 512x512 for pre-cropped clips")
    ap.add_argument("--cpu-frames", type=int, default=2)
    a = ap.parse_args()
    H, W = (int(v) for v in a.frame_hw.lower().split("x"))
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    root = synth_assets.materialize(os.path.join(tempfile.gettempdir(), "smk_assets_bench_video_%d" % rank))
    os.chdir(root)
    lo, hi = shard_bounds(a.batch, world, rank)
    B = hi - lo
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    enc = enc.eval().to(dev)
    enc.precision = 3
    stage = video.VideoStage((H, W), render_orig=a.render_orig, crop=not a.no_crop)
    fl = smirk_b200.FLAME().to(dev)
    gen = masking = None
    if a.generator:
        from smirk_b200.masking import MaskingStage
        gen = smirk_b200.SmirkGenerator(6, 3, 32, 5)
        gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
        gen = gen.eval().to(dev)
        gen.precision = 1
        masking = MaskingStage(fl.faces_tensor, synth_inputs.face_probabilities(fl.faces_tensor.shape[0]), seed=1234 + rank)
    pipe = SmirkPipeline(enc, fl, smirk_b200.Renderer().to(dev), gen, device=dev, slots=a.slots, masking=masking, video=stage)
    rng = np.random.default_rng(100 + rank)
    host = [torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).pin_memory() for _ in range(2)]
    lms = [landmarks(rng, B, H, W) for _ in range(2)]
    batches = [stage.prepare(l) if (a.generator or not a.no_crop) else stage.prepare(batch_size=B) for l in lms]
    frames = [h.to(dev) for h in host]                  # two 400 MB sets at 1080p: nothing of a step is still in the 50 MB L2
    for lane in range(pipe.slots):
        pipe.capture(B, lane)

    def barrier():
        torch.cuda.synchronize(dev)
        if dist is not None:
            dist.barrier()

    def timed(step):
        for i in range(a.warmup):
            step(i)
        pipe.join()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(a.steps):
            step(i)
        pipe.join()
        e1.record()
        torch.cuda.synchronize(dev)
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if dist is not None:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    sampler = bench.ClockSampler(local)
    sampler.start()
    ms_dev = timed(lambda i: pipe.submit(i, frames[i % 2], batches[i % 2]))
    keys = ("grid",)
    ms_e2e = timed(lambda i: pipe.run_host(host[i % 2], i, batches[i % 2], keys))
    clocks = sampler.stop()
    h2d, d2h = pipe.bytes_per_step(B, keys)

    L = _lib.lib()
    pipe.forward(frames[0], batches[0])
    torch.cuda.synchronize(dev)
    L.smk_profiler_reset(); L.smk_profiler_enable(1)
    pipe.forward(frames[0], batches[0])
    torch.cuda.synchronize(dev)
    rep = _lib.profiler_report()
    L.smk_profiler_enable(0); L.smk_profiler_reset()
    stages = {k: dict(ms=round(v["ms"], 4), launches=v["launches"]) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}
    gbs = lambda tags: round(sum(rep[t]["bytes"] for t in tags if t in rep) / max(1e-9, sum(rep[t]["ms"] for t in tags if t in rep)) / 1e6, 1)

    out = None
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                           capture_output=True, text=True).stdout.strip()
        cpu_s = cpu_baseline(root, [h.numpy() for h in host[0][:a.cpu_frames]], lms[0][:a.cpu_frames], a.render_orig, not a.no_crop)
        out = {
            "workload": "configs[3]: demo_video.py%s%s%s, %dx%d frames, batch %d (%d per GPU), %d GPU(s)"
                        % ("" if a.no_crop else " --crop", " --render_orig" if a.render_orig else "",
                           " --use_smirk_generator" if a.generator else "",
                           W, H, a.batch, B, world),
            "device_fps": round(a.batch * a.steps / ms_dev * 1e3, 1),
            "device_ms_per_step": round(ms_dev / a.steps, 3),
            "e2e_fps": round(a.batch * a.steps / ms_e2e * 1e3, 1),
            "e2e_ms_per_step": round(ms_e2e / a.steps, 3),
            "h2d_bytes_per_frame": h2d // B, "d2h_bytes_per_frame": d2h // B,
            "launches_per_step": pipe.launches_per_step(B),
            "stages_rank0_eager": stages,
            "video_compose_gbs": gbs(["video_minmax", "video_compose"]),
            "hull_mask_ms": round(rep["hull_mask"]["ms"], 4) if "hull_mask" in rep else None,
            "crop_warp_gbs": gbs(["warp_minmax", "warp_bilinear", "resize"]),
            "gpu": {"name_power_limit": q, "clocks": clocks},
            "command": " ".join(sys.argv),
            "cpu_baseline": {"frames_per_s": round(1.0 / cpu_s, 3), "frames": a.cpu_frames, "cores": os.cpu_count(),
                             "threads": torch.get_num_threads(),
                             "what": "oracle port (torch CPU) + %s, one frame at a time"
                                     % ("cv2.resize / F.interpolate" if a.no_crop else "warp_ref crop / warp back")},
            "steps": a.steps, "warmup": a.warmup, "slots": a.slots,
        }
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()
    if out is not None:
        print(json.dumps(out))


if __name__ == "__main__":
    main()
