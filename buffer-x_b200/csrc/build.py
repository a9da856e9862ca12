"""Build libbufferx_b200.so (sm_90a, H100) with nvcc, in-tree.

    python buffer-x_b200/csrc/build.py [--force]

Two groups of translation units:
  EXACT  compiled with -fmad=false: every kernel whose result feeds an integer / index decision
         that must be bit-identical to the oracle (FPS, radius histogram, ball query, LRF, SPT,
         matching, consensus, RANSAC).
  FAST   compiled with FMA contraction: the convolution stacks (tolerance parity).
The shared object lands next to the package (buffer-x_b200/libbufferx_b200.so); it is git-ignored.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT = os.path.join(PKG, "libbufferx_b200.so")
OBJ = os.path.join(HERE, "_obj")

EXACT = ["bx_api.cu", "bx_fps.cu", "bx_radius.cu", "bx_patches.cu", "bx_spt.cu", "bx_match.cu", "bx_ransac.cu", "bx_neighbors.cu",
         "bx_bootstrap.cu", "bx_train.cu"]
FAST = ["bx_conv.cu", "bx_conv_tc.cu", "bx_conv_sd.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    # objects are only reusable for the flag set they were compiled with
    stamp, flags = os.path.join(OBJ, "flags.txt"), " ".join(ARCH + COMMON)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    headers = [os.path.join(HERE, "bx_common.cuh"), os.path.join(PKG, "..", "include", "bufferx_b200.h"),
               os.path.abspath(__file__)]
    headers += [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith(".cuh")]
    jobs = []
    for src, extra in [(s, ["-fmad=false"]) for s in EXACT] + [(s, []) for s in FAST]:
        sp = os.path.join(HERE, src)
        op = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(op, [sp] + headers):
            jobs.append([_nvcc()] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", op])
    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for log in ex.map(run, jobs):
            if verbose and log:
                print(log)
    with open(stamp, "w") as f:
        f.write(flags)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in EXACT + FAST]
    if force or jobs or _stale(OUT, objs):
        run([_nvcc()] + ARCH + ["-shared", "-o", OUT] + objs)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
