"""Build libvd3d.so in-tree with nvcc for sm_90a (no torch extension machinery:
the boundary is a plain C ABI).  Used by __graft_entry__.build()."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libvd3d.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-I", os.path.join(HERE, "..", "include")]

# (source, extra flags).  The DIBR kernels reproduce the reference's fp32 rounding one
# op at a time, so FMA contraction is off there and fused ops are spelled __fmaf_rn.
UNITS = [
    ("dibr_kernels.cu", ["-fmad=false"]),
    ("dibr_fast.cu", ["-fmad=false"]),
    ("vd3d_api.cu", ["-fmad=false"]),
    ("letterbox.cu", ["-fmad=false"]),
    ("sr_kernels.cu", ["-fmad=false"]),
    ("tiled_depth.cu", ["-fmad=false"]),
    ("depth_kernels.cu", []),
    ("depth_engine.cu", []),
]


def _stale(obj, deps):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(HERE, "..", "include", "vd3d.h"))
    objs = []
    for src, extra in UNITS:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        if force or _stale(obj, [sp] + hdrs):
            cmd = [nvcc] + ARCH + COMMON + extra + ["-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            subprocess.check_call(cmd)
        objs.append(obj)
    if force or _stale(LIB, objs):
        tmp = LIB + ".tmp"  # link next to the target, then rename: a concurrent reader never sees a half-written library
        cmd = [nvcc] + ARCH + ["-shared", "-o", tmp] + objs + ["-lcudart"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
