"""In-tree build of libchd_b200.so (hand-written CUDA for sm_90a, the H100 + the C ABI of include/chd_gpu.h,
include/chd_gpu_subs.h, include/chd_gpu_facing.h, include/chd_gpu_rings.h, include/chd_gpu_subs_sharded.h and include/chd_gpu_ring_bytes.h).

nvcc cross-compiles without a GPU.  The .so is a build product: git-ignored, rebuilt when a source is newer.
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libchd_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false",            # belt and braces: all parity-critical FP64 uses explicit _rn intrinsics anyway
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC,-O2,-Wall",
    "-shared", "-cudart", "shared",
    "-ldl",                   # NCCL is dlopen'ed on first multi-GPU use (chd_shard.cu): no link-time dependency on it
]


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu") or f.endswith(".cpp")]


def deps():
    out = [os.path.join(ROOT, "include", "chd_gpu.h"), os.path.join(ROOT, "include", "chd_gpu_subs.h"),
           os.path.join(ROOT, "include", "chd_gpu_facing.h"), os.path.join(ROOT, "include", "chd_gpu_rings.h"),
           os.path.join(ROOT, "include", "chd_gpu_subs_sharded.h"), os.path.join(ROOT, "include", "chd_gpu_ring_bytes.h"),
           os.path.abspath(__file__)]
    for f in os.listdir(CSRC):
        out.append(os.path.join(CSRC, f))
    return out


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in deps())


def build(force=False, verbose=False, extra_flags=(), out=None):
    """extra_flags / out: experiment builds, e.g. -DCHD_EMIT_ROWS=4 into another file; the product is LIB."""
    if out is None and not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = ([nvcc] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-I", os.path.join(ROOT, "include"), "-o", out or LIB]
           + sources())
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        sys.stderr.write(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return out or LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
