"""Summarise an ncu CSV (--metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --csv) into
the per-kernel DRAM-traffic JSON that bench.py reads for `roofline.traffic`.

    ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none --csv \
        --log-file gpurun_out/ncu_dram.csv python tools/profile_layers.py --steps 1
    python tools/ncu_traffic.py gpurun_out/ncu_dram.csv profiles/r01_ncu_dram_traffic_c2_b32_tf32.json [--last-pass N]

Kernel function names are mapped to the profiler tags of the library (SMK_TAG in csrc/).  gemm_tc_kernel serves three
tags (1x1, 3x3, transposed conv); for the encoder-only workload it is all `pw_gemm_tc`.  With --last-pass N only the
last N launches of the capture are used (profile_layers.py runs warm-up passes first; pass the number of launches of
one forward pass, printed by bench.py as launches_per_step).
"""
import argparse
import csv
import json
import re

TAGS = [
    (r"xdw_kernel<\d+, *[123]>", "xdw_fused_tc3x"), (r"xdw_kernel", "xdw_fused_tc"),
    (r"gemm_tc_kernel<\d+, *\d+, *\d+, *(false|0), *[12]>", "pw_gemm_tc3x"),            # 3xTF32 variants (single-tile CTAs)
    (r"gemm_tc_kernel<\d+, *\d+, *\d+, *(true|1), *0>", "conv3x3_gemm_tc"),             # persistent CTAs: the generator's 3x3 convolutions
    (r"gemm_tc_kernel", "pw_gemm_tc"),                                                  # 1x1 convs / transposed convs
    (r"conv3_win_kernel", "conv3x3_win_tc"), (r"gap_head_kernel", "gap_head"), (r"mask_\w+_kernel", "masking"),
    (r"stem_ds_kernel", "stem_ds_fused"), (r"stem_conv3_kernel", "stem_conv3"), (r"stem_conv_kernel", "stem_conv"),
    (r"dwconv3x3", "dwconv3x3"), (r"conv_gemm_kernel", "conv_gemm_f32"), (r"raster_tile_kernel", "raster_tile"),
    (r"flame_verts_kernel", "flame_verts"), (r"flame_pose_kernel", "flame_pose"), (r"flame_landmarks_kernel", "flame_landmarks"),
    (r"tri_setup_kernel", "tri_setup"), (r"submesh_kernel", "submesh_normals"), (r"project_kernel", "project"),
    (r"reflect_halo_kernel", "reflect_halo"),
    (r"maxpool2x2_kernel", "maxpool2x2"), (r"nchw_to_nhwc_pad_kernel", "nchw_to_nhwc"), (r"conv1x1_sigmoid_kernel", "conv1x1_sigmoid"),
]
UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "usecond": 1.0, "nsecond": 1e-3, "ms": 1e3, "msecond": 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("out")
    ap.add_argument("--last-pass", type=int, default=0)
    ap.add_argument("--source", default="")
    ap.add_argument("--passes", type=int, default=1, help="forward passes covered by the selected launches (step traffic = total / passes)")
    a = ap.parse_args()
    rows = [r for r in csv.reader(open(a.csv, errors="replace")) if len(r) > 10]
    hdr = next(r for r in rows if r[0] == "ID")
    ix = {k: i for i, k in enumerate(hdr)}
    per_id = {}
    for r in rows:
        if r[0] == "ID" or not r[0].isdigit():
            continue
        d = per_id.setdefault(int(r[0]), {"name": r[ix["Kernel Name"]]})
        val = float(r[ix["Metric Value"]].replace(",", "")) * UNIT.get(r[ix["Metric Unit"]], 1.0)
        d[r[ix["Metric Name"]]] = val
    ids = sorted(per_id)
    lib = [i for i in ids if any(re.search(p, per_id[i]["name"]) for p, _ in TAGS)]
    if a.last_pass:
        lib = lib[-a.last_pass:]
    out = {}
    for i in lib:
        d = per_id[i]
        tag = next(t for p, t in TAGS if re.search(p, d["name"]))
        o = out.setdefault(tag, {"launches": 0, "dram_read_bytes": 0.0, "dram_write_bytes": 0.0, "ncu_us": 0.0})
        o["launches"] += 1
        o["dram_read_bytes"] += d.get("dram__bytes_read.sum", 0.0)
        o["dram_write_bytes"] += d.get("dram__bytes_write.sum", 0.0)
        o["ncu_us"] += d.get("gpu__time_duration.sum", 0.0)
    for o in out.values():
        o["traffic_bytes_per_launch"] = (o["dram_read_bytes"] + o["dram_write_bytes"]) / o["launches"]
    tot = sum(o["ncu_us"] for o in out.values())
    for o in out.values():
        o["share_of_ncu_time"] = o["ncu_us"] / tot
    step = sum(o["dram_read_bytes"] + o["dram_write_bytes"] for o in out.values()) / max(1, a.passes)
    json.dump({"source": a.source or ("ncu csv %s, last %d launches" % (a.csv, len(lib))), "launches": len(lib), "passes": a.passes,
               "step_traffic_bytes": step, "kernels": out}, open(a.out, "w"), indent=1)
    print("step DRAM traffic: %.1f MB over %d launches" % (step / 1e6, len(lib) // max(1, a.passes)))
    for t, o in sorted(out.items(), key=lambda kv: -kv[1]["ncu_us"]):
        print("%-18s x%-3d %9.1f us  share %.3f  dram/launch %8.2f MB" % (t, o["launches"], o["ncu_us"], o["share_of_ncu_time"], o["traffic_bytes_per_launch"] / 1e6))


if __name__ == "__main__":
    main()
