"""IK feasibility of the KUKA iiwa14 on the GPU (csrc/cg_ik.cu): the closed-form replacement of the reference's
get_ik_within_limits (my_cpp/common.cpp:9-72) over its generated ikfast solver, free joint 2 fixed at 0."""
import numpy as np
import torch

from . import _lib

D_BS, D_SE, D_EW, D_WF = 0.36, 0.42, 0.40, 0.081


def joint_limits(upper, lower):
    """The first 7 entries of upper / lower as float64 (the reference indexes them by joint); fewer raise."""
    up = np.asarray(upper, dtype=np.float64).reshape(-1)
    lo = np.asarray(lower, dtype=np.float64).reshape(-1)
    if up.shape[0] < 7 or lo.shape[0] < 7:
        raise ValueError(f"upper / lower need at least 7 joint limits, got {up.shape[0]} / {lo.shape[0]}")
    return np.ascontiguousarray(up[:7]), np.ascontiguousarray(lo[:7])


def iiwa14_ik(ee_in_base, upper, lower, solutions=False):
    """ee_in_base (Q,4,4) (or one (4,4)) end-effector poses in the robot base frame, narrowed to float32 like the
    reference's Matrix4f -> count (Q,) int8 of solutions within [lower, upper] (both inclusive), and with
    ``solutions=True`` also (Q,8,7) float64 = every solution regardless of the limits in the slot order of
    include/catgrasp_b200.h (NaN where a branch has none).  numpy in -> numpy out; a CUDA tensor in -> CUDA tensors
    out on the same device and stream."""
    up, lo = joint_limits(upper, lower)
    ctx, ee = _lib.inputs(ee_in_base, dtype=torch.float32)
    ee = ee.reshape(-1, 16)
    Q = ee.shape[0]
    count = torch.empty((Q,), dtype=torch.int8, device=ee.device)
    sol = torch.empty((Q, 8, 7), dtype=torch.float64, device=ee.device) if solutions else None
    ctx.call("cg_iiwa14_ik_dev", ctx.h, ee, Q, up, lo, count, sol)
    return _lib.returned(ee_in_base, count, sol) if solutions else _lib.returned(ee_in_base, count)


def iiwa14_fk(q):
    """(..., 7) joint angles -> (..., 4, 4) float64 end-effector pose in the base frame (host, float64):
    Tz(0.36) Rz(q0) Ry(q1) Rz(q2) Tz(0.42) Ry(-q3) Rz(q4) Tz(0.40) Ry(q5) Rz(q6) Tz(0.081)."""
    q = np.asarray(q, dtype=np.float64)
    a = q.reshape(-1, 7)
    n = a.shape[0]

    def rot(axis, t, sign=1.0):
        c, s = np.cos(t), sign * np.sin(t)
        T = np.zeros((n, 4, 4))
        T[:, 3, 3] = 1.0
        if axis == "z":
            T[:, 0, 0], T[:, 0, 1], T[:, 1, 0], T[:, 1, 1], T[:, 2, 2] = c, -s, s, c, 1.0
        else:
            T[:, 0, 0], T[:, 0, 2], T[:, 2, 0], T[:, 2, 2], T[:, 1, 1] = c, s, -s, c, 1.0
        return T

    def tz(d):
        T = np.eye(4)
        T[2, 3] = d
        return T

    T = tz(D_BS) @ rot("z", a[:, 0]) @ rot("y", a[:, 1]) @ rot("z", a[:, 2]) @ tz(D_SE) @ rot("y", a[:, 3], -1.0) \
        @ rot("z", a[:, 4]) @ tz(D_EW) @ rot("y", a[:, 5]) @ rot("z", a[:, 6]) @ tz(D_WF)
    return T.reshape(q.shape[:-1] + (4, 4))
