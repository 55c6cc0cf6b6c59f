"""Build recipe for oracle/_ref/libik_ref.so: oracle/ref_shim/ik_api.cpp linked against oracle/_ref/libmycpp_ref.so
(oracle/build_ref.py), which carries the reference's get_ik_within_limits (my_cpp/common.cpp:9-72) and its generated
ikfast solver for the KUKA iiwa14.  The shim exports every ikfast solution of a pose and ikfast's forward kinematics.

Like build_ref, it compiles only where /root/reference exists; the library goes to oracle/_ref/ (git-ignored).
"""
import os
import subprocess

from . import build_ref

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(build_ref.OUT_DIR, "libik_ref.so")
SRC = os.path.join(HERE, "ref_shim", "ik_api.cpp")


def available():
    return build_ref.available()


def build(force=False):
    if not build_ref.available():
        return LIB if os.path.exists(LIB) else None
    base = build_ref.build(force=force)
    mine = [SRC, os.path.abspath(__file__), base]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(s) for s in mine):
        return LIB
    ref = build_ref.REF
    eig = f"{ref}/PointGroup/lib/pointgroup_ops"
    inc = ["-I", os.path.join(HERE, "ref_shim"), "-I", f"{eig}/eigen3", "-I", eig, "-I", f"{ref}/my_cpp",
           "-I", f"{ref}/ikfast_pybind/src"]
    subprocess.check_call(["g++", "-O2", "-std=c++14", "-fPIC", "-shared", "-w", "-DIKFAST_HAS_LIBRARY"] + inc +
                          [SRC, "-o", LIB, "-L", build_ref.OUT_DIR, "-lmycpp_ref", "-Wl,-rpath,$ORIGIN"])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
