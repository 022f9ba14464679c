"""Builds libybgpu.so (sm_90a, H100) in-tree with nvcc. Used by __graft_entry__.build()."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libybgpu.so")
SOURCES = ["engine.cu", "abi.cc", "host_sst.cc", "host_gen.cc", "subcompaction.cc", "numa.cc", "range_exchange.cc"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-msse4.2,-Wall", "--shared", "-cudart", "shared", "-ldl"]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "ybgpu_compaction.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = OUT + ".tmp%d" % os.getpid()          # written beside the target, then renamed: a snapshot of the tree never sees half a library
    cmd = [nvcc] + NVCC_FLAGS + ["-x", "cu"] + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", tmp]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    try:
        subprocess.check_call(cmd)
        os.replace(tmp, OUT)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
