"""Builds libpersia_b200.so in-tree with nvcc for H100 (sm_90a); no JIT cache: the .so travels with the repo."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libpersia_b200.so")
SOURCES = ["pb_index.cu", "pb_dedup.cu", "pb_reduce.cu", "pb_shard.cu", "pb_sort.cu", "pb_update.cu", "pb_raw.cu", "pb_launch.cu", "pb_api.cu"]
HEADERS = ["pb_common.cuh", "pb_kernels.cuh", "pb_device.cuh", "pb_group.cuh", "pb_probe.cuh", "pb_optim.cuh", "pb_batch.cuh", os.path.join(ROOT, "include", "persia_b200.h")]


def nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.abspath(__file__)] + [os.path.join(CSRC, s) for s in SOURCES] + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not stale():
        return SO
    cmd = [
        nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
        "--fmad=false",  # the optimizer reproduces the reference's fused / unfused structure explicitly
        "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared",
        "-I", os.path.join(ROOT, "include"), "-I", CSRC,
        "-Xlinker", "-rpath,/usr/local/cuda/lib64",
        "-o", SO,
    ] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    import sys

    print(build(force=True, verbose="-v" in sys.argv))
