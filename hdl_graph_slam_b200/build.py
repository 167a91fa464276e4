"""In-tree build of the engine's native libraries (no JIT cache: the .so files travel with the repo snapshot).

  _lib/libb200reg.so     CUDA engine + C ABI (sm_90a)                  <- csrc/api.cu
  _lib/libb2r_synth.so   synthetic LiDAR workload generator (C/OpenMP)  <- synth/lidar_synth.c
"""
import os
import subprocess
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_lib")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    # host code keeps a * b + c as two roundings on every target (the pose products of csrc/odometry_gate.cuh are compared bit for bit
    # with a float32 restatement); device code is not affected by this flag
    "--compiler-options=-ffp-contract=off",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _host_cc():
    for c in ("/usr/bin/gcc", shutil.which("gcc") or "gcc"):
        if os.path.exists(c):
            return c
    return "gcc"


def build_engine(force=False, verbose=False):
    os.makedirs(LIB, exist_ok=True)
    csrc = os.path.join(HERE, "csrc")
    srcs = [os.path.join(csrc, f) for f in sorted(os.listdir(csrc))] + [os.path.join(HERE, "..", "include", "b200reg.h")]
    out = os.path.join(LIB, "libb200reg.so")
    if force or _newer(out, srcs):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        tmp = out + f".tmp{os.getpid()}"  # link under another name, then rename: a reader (or a repo snapshot) never sees a half-written library
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
              "-o", tmp, os.path.join(csrc, "api.cu"), "-lnccl"]
        try:
            subprocess.check_call(cmd)
            os.replace(tmp, out)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    return out


def build_synth(force=False):
    os.makedirs(LIB, exist_ok=True)
    src = os.path.join(HERE, "synth", "lidar_synth.c")
    out = os.path.join(LIB, "libb2r_synth.so")
    if force or _newer(out, [src]):
        subprocess.check_call([_host_cc(), "-O2", "-fopenmp", "-fPIC", "-shared", "-o", out, src, "-lm"])
    return out


def build_all(force=False, verbose=False):
    return build_engine(force, verbose), build_synth(force)


if __name__ == "__main__":
    import sys
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
