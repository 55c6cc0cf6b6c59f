"""ctypes wrapper of oracle/_ref/libik_ref.so (oracle/build_ref_ik.py): the reference's own IK -- get_ik_within_limits
(my_cpp/common.cpp:9-72) over its generated ikfast solver for the KUKA iiwa14.  ORACLE, test infrastructure only."""
import ctypes as C
import os

import numpy as np

from . import build_ref_ik

_lib = None


def available():
    return build_ref_ik.available() or os.path.exists(build_ref_ik.LIB)


def _load():
    global _lib
    if _lib is None:
        path = build_ref_ik.build()
        if path is None:
            raise RuntimeError("oracle/_ref/libik_ref.so is not built and /root/reference is not present")
        _lib = C.CDLL(path)
        _lib.ref_ik_solutions.restype = C.c_int
        _lib.ref_ik_solutions.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        _lib.ref_ik_fk.restype = None
        _lib.ref_ik_fk.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def ik_solutions(ee_in_base):
    """All ikfast solutions (K,7) float64 of one (4,4) pose (narrowed to float32 as the reference's Matrix4f is), free
    joint 2 at 0, in ikfast's order."""
    lib = _load()
    m = np.ascontiguousarray(np.asarray(ee_in_base, dtype=np.float64).astype(np.float32)).reshape(16)
    out = np.zeros((64, 7), np.float64)
    n = lib.ref_ik_solutions(m.ctypes.data, out.ctypes.data, 64)
    assert n <= 64
    return out[:n].copy()


def ik_fk(q):
    """ikfast ComputeFk: (7,) joints -> (4,4) float64 end-effector pose in the base frame."""
    lib = _load()
    q = np.ascontiguousarray(q, dtype=np.float64).reshape(7)
    t = np.zeros(3, np.float64)
    r = np.zeros(9, np.float64)
    lib.ref_ik_fk(q.ctypes.data, t.ctypes.data, r.ctypes.data)
    T = np.eye(4)
    T[:3, :3] = r.reshape(3, 3)
    T[:3, 3] = t
    return T


def ik_within_limits(ee_in_base, upper, lower):
    """Solutions of get_ik_within_limits under the given limits (first 7 entries), as the reference keeps them."""
    s = ik_solutions(ee_in_base)
    up = np.asarray(upper, np.float64)[:7]
    lo = np.asarray(lower, np.float64)[:7]
    return s[~((s > up) | (s < lo)).any(axis=1)]
