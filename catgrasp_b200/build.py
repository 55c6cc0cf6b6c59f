"""Build recipe for libcatgrasp_b200.so: nvcc, sm_90a only, output inside the package tree."""
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libcatgrasp_b200.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-pthread", "--expt-relaxed-constexpr"]


if os.environ.get("CG_BUILD_EXPERIMENTS") == "1":   # developer builds only: the CG_FPS_CLUSTER switch
    NVCC_FLAGS.append("-DCG_EXPERIMENTS")


CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-pthread"]   # host-only sources (*.cpp): straight through g++


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    for src in sources():
        obj = os.path.join(obj_dir, os.path.splitext(os.path.basename(src))[0] + ".o")
        objs.append(obj)
        if src.endswith(".cpp"):
            cmd = [os.environ.get("CXX", "g++")] + CXX_FLAGS + ["-c", src, "-o", obj]
        else:
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"compiler failed on {src}")
    subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-pthread",
                           "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force=True, verbose="-v" in sys.argv))
