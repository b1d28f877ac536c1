"""Build libdensity_b200.so in-tree with nvcc for sm_90a, the H100 (no torch extension machinery: the library is a plain
C-ABI shared object, see include/density_b200.h)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libdensity_b200.so")
SOURCES = ["api.cu", "chameleon_encode.cu", "chameleon_decode.cu", "cheetah_encode.cu", "cl_decode.cu", "scalar_codec.cu", "decoded_size.cu",
           "decode_range.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--cudart", "static",
] + os.environ.get("DENSITY_B200_NVCC_EXTRA", "").split()


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if p and (os.path.sep not in p or os.path.exists(p)):
            return p
    return "nvcc"


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "density_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    objs = []
    bdir = os.path.join(HERE, "_obj")
    os.makedirs(bdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(bdir, src.replace(".cu", ".o"))
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        subprocess.check_call(cmd)
        objs.append(obj)
    tmp = SO + ".tmp"     # link next to the target, then rename: a snapshot of the tree never sees a half-written library
    cmd = [nvcc_path(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "--cudart", "static", "-o", tmp] + objs
    subprocess.check_call(cmd)
    os.replace(tmp, SO)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
