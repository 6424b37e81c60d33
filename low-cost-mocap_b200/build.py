"""Builds libmocap_b200.so in-tree with nvcc for sm_90a (H100); no JIT cache, the library is loaded from
the package directory."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmocap_b200.so")
SOURCES = ["api.cu", "blob_kernels.cu", "match_kernels.cu", "fused_kernel.cu", "tma_kernel.cu", "locate_kernels.cu", "preproc.cu", "calib_init.cu", "calib_ransac.cu", "calib_graph.cu", "ba.cu", "ba_dev.cu", "screen.cu", "track.cu", "live.cu", "jpeg.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--use_fast_math=false"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "mocap_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        subprocess.check_call(cmd)
        objs.append(obj)
    # link under a temporary name and rename: a reader (or a repository snapshot) never sees a half-written library
    tmp = LIB + ".tmp"
    subprocess.check_call([nvcc, "-shared"] + GENCODE + ["-o", tmp] + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
