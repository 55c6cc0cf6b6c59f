"""Build recipe and ctypes wrapper of oracle/sdf_mesh_ref.c, and a float64 restatement of the mesh-SDF grid geometry --
ORACLE, test infrastructure only (the product is catgrasp_b200/csrc/cg_sdf_build.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "sdf_mesh_ref.c")
LIB = os.path.join(HERE, "_build", "libsdf_mesh_ref.so")

_lib = None


def build(force=False):
    """gcc with OpenMP and without FMA contraction: the point-triangle distance then rounds exactly like the kernel's,
    which spells out every float64 operation in the same order."""
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    subprocess.check_call(["gcc", "-O2", "-mfma", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", LIB, SRC,
                           "-lm"])
    return LIB


def _load():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.sdf_mesh_ref.restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def sdf_mesh_ref(vertices, faces, points, nthreads=0):
    """Signed distance (negative inside, by winding number) and winding number of every query point (Q,3)."""
    V = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
    F = np.ascontiguousarray(faces, dtype=np.int32).reshape(-1, 3)
    Q = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    sd = np.zeros(Q.shape[0])
    wind = np.zeros(Q.shape[0])
    _load().sdf_mesh_ref(_p(V), _p(F), C.c_int(F.shape[0]), _p(Q), C.c_long(Q.shape[0]), C.c_int(int(nthreads)),
                         _p(sd), _p(wind))
    return sd, wind


def grid_geometry(vertices, resolution, padding):
    """(dims (3,) int, origin (3,) float32, res float32) of the grid cg_sdf_from_mesh builds (include/catgrasp_b200.h)."""
    V = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    res = float(np.float32(resolution))
    lo, hi = V.min(0), V.max(0)
    dims = (np.ceil((hi - lo) / res - 1e-4) + 1 + 2 * padding).astype(np.int64)
    origin = (lo - padding * res).astype(np.float32)
    return dims, origin, np.float32(res)


def node_positions(origin, resolution, idx):
    """float64 positions origin + idx * res of integer node indices idx (..., 3), from the float32 origin and res."""
    return np.asarray(origin, np.float32).astype(np.float64) + np.asarray(idx, np.float64) * float(np.float32(resolution))
