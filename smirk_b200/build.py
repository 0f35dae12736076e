"""Build recipe: smirk_b200/csrc/*.cu -> smirk_b200/libsmirk_b200.so (sm_90a only, in-tree).

nvcc cross-compiles without a GPU.  Objects are cached by mtime.  Per-file flags:
render.cu is compiled with -fmad=false so the rasteriser's fp32 arithmetic is never contracted into
FMAs (bit-exact face indices against the CPU oracle).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "build")
LIB = os.path.join(HERE, "libsmirk_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
BASE = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
PER_FILE = {"render.cu": ["-fmad=false"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    inc = os.path.join(HERE, "..", "include")
    hdrs += [os.path.join(inc, f) for f in os.listdir(inc) if f.endswith(".h")]
    hdr_m = max(os.path.getmtime(h) for h in hdrs)
    objs, rebuilt = [], False
    for s in sources():
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
            cmd = [NVCC] + BASE + PER_FILE.get(s, []) + ["-c", src, "-o", obj]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or r.returncode:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode:
                raise RuntimeError("nvcc failed on %s" % s)
            with open(obj + ".log", "w") as fh:
                fh.write(r.stdout + r.stderr)
            rebuilt = True
    if rebuilt or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-cudart", "static"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
