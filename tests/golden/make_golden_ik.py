"""Golden vectors for the KUKA iiwa14 IK feasibility test, from the REFERENCE's own get_ik_within_limits
(my_cpp/common.cpp:9-72) over its generated ikfast solver, compiled by oracle/build_ref.py + oracle/build_ref_ik.py.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_golden_ik.py

Inputs are regenerated from seeds by ``inputs()`` (the tests call it too); ik_iiwa14.npz stores a SHA-256 of them so a
drifting generator is detected, plus what the reference computes:
  fk_q, fk_T             ComputeFk of 256 random configurations
  family                 per pose: 0 FK of a random configuration (16384), 1 random rigid pose (4096), 2 shoulder band,
                         3 wrist (q5) near 0, 4 elbow (q3) near 0, 5 reach boundary, 6 a joint 1e-4 rad from a limit
  nsol                   number of ikfast solutions of every pose (limits +-inf)
  count_a, count_b       in-limit counts under IK_UPPER / IK_LOWER of make_golden_mycpp.py and under +-90 degrees
  sol_index, sol         all ikfast solutions (float32) of the poses in sol_index (every special-family pose, the first
                         1024 FK and 512 rigid ones), concatenated in pose order
  shoulder_bisect        the wrist-centre radius (m) below which ikfast returns nothing, bisected at three arms
  filter_*               one filterGraspPose(filter_ik=True) case whose IK rejections include limit violations,
                         out-of-reach and shoulder-band poses: sorted survivor bit patterns and the four verbose
                         counters + survivor count the compiled reference printed
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, HERE)

from oracle.ik_ref import iiwa14_fk  # noqa: E402
from make_golden_mycpp import ik_frames  # noqa: E402  (this directory is on sys.path when run as a script)

IK_UPPER = np.deg2rad([170, 120, 170, 120, 170, 120, 175])     # make_golden_mycpp.py
IK_LOWER = -IK_UPPER
TIGHT_UPPER = np.full(7, np.pi / 2)
TIGHT_LOWER = -TIGHT_UPPER
N_FK, N_RIGID = 16384, 4096
SHOULDER_MM = [0.0, 0.5, 0.999, 1.001, 1.5, 5.0]
NEAR_ZERO = [0.0, 1e-8, 1e-7, 3e-7, 1e-6, 1e-5]
REACH_DELTA = [-1e-3, -1e-6, 1e-6, 1e-3]


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def random_rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3)


def pose_from_wrist(w, R):
    """End-effector pose whose wrist centre is w (base frame) for orientation R."""
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = w + 0.081 * R[:, 2]
    return T


def random_q(rng, n):
    q = rng.uniform(-2.5, 2.5, (n, 7))
    q[:, 2] = 0.0
    return q


def inputs():
    """(poses (N,4,4) float32, family (N,) int8, fk_q (256,7) float64)."""
    rng = np.random.RandomState(20261016)
    fk_q = random_q(rng, 256)
    poses, fam = [], []
    poses.append(iiwa14_fk(random_q(rng, N_FK))); fam += [0] * N_FK
    Rr = random_rotations(rng, N_RIGID)
    T = np.tile(np.eye(4), (N_RIGID, 1, 1))
    T[:, :3, :3] = Rr
    T[:, :3, 3] = rng.uniform([-1.1, -1.1, -0.4], [1.1, 1.1, 1.7], (N_RIGID, 3))
    poses.append(T); fam += [1] * N_RIGID
    fam2 = []
    for rho in SHOULDER_MM:
        for R in random_rotations(rng, 8):
            phi, h = rng.uniform(-np.pi, np.pi), rng.uniform(-0.6, 0.6)
            fam2.append(pose_from_wrist(np.array([1e-3 * rho * np.cos(phi), 1e-3 * rho * np.sin(phi), 0.36 + h]), R))
    poses.append(np.array(fam2)); fam += [2] * len(fam2)
    for joint, f in ((5, 3), (3, 4)):
        rows = []
        for v in NEAR_ZERO:
            for sign in (1.0, -1.0):
                q = random_q(rng, 4)
                q[:, joint] = sign * v
                rows.append(iiwa14_fk(q))
        poses.append(np.concatenate(rows)); fam += [f] * (len(rows) * 4)
    rows = []
    for d in REACH_DELTA:
        for R in random_rotations(rng, 8):
            u = rng.normal(size=3)
            u /= np.linalg.norm(u)
            rows.append(pose_from_wrist(np.array([0, 0, 0.36]) + (0.82 + d) * u, R))
    poses.append(np.array(rows)); fam += [5] * len(rows)
    rows = []
    for k in (0, 1, 3, 4, 5, 6):
        for lim in (IK_UPPER[k], IK_LOWER[k]):
            for d in (-1e-4, 1e-4):
                q = random_q(rng, 2)
                q[:, k] = lim + d
                rows.append(iiwa14_fk(q))
    poses.append(np.concatenate(rows)); fam += [6] * (len(rows) * 2)
    P = np.concatenate(poses).astype(np.float32)
    return P, np.array(fam, np.int8), fk_q


def filter_case():
    """One filterGraspPose(filter_ik=True) input set whose grasps are built from end-effector targets: reachable
    within the limits, beyond joint 3's limit (|q3| > 120 degrees on every branch), out of reach, in the shoulder band."""
    from catgrasp_b200 import synthetic
    rng = np.random.RandomState(7)
    p1, p2, _, _, _, _, g = synthetic.make_filter_case(43, 8, 1)
    cam, ee = ik_frames()
    q_ok = random_q(rng, 48)
    q_ok[:, 3] = rng.uniform(-1.5, 1.5, 48)
    q_lim = random_q(rng, 24)
    q_lim[:, 3] = rng.choice([-1, 1], 24) * rng.uniform(2.15, 2.5, 24)
    targets = [iiwa14_fk(q_ok), iiwa14_fk(q_lim)]
    far = iiwa14_fk(random_q(rng, 16))
    far[:, :3, 3] *= 1.6
    targets.append(far)
    band = [pose_from_wrist(np.array([4e-4 * np.cos(a), 4e-4 * np.sin(a), 0.36 + h]), R)
            for a, h, R in zip(rng.uniform(-np.pi, np.pi, 12), rng.uniform(-0.5, 0.5, 12), random_rotations(rng, 12))]
    targets.append(np.array(band))
    E = np.concatenate(targets)
    # grasp_in_cam = cam^-1 * ee_in_base * ee_in_grasp^-1 (common.cpp:216 solved for the grasp)
    grasps = np.linalg.inv(cam)[None] @ E @ np.linalg.inv(ee)[None]
    eye = np.eye(4)
    return dict(grasps=grasps, sym=eye[None], nocs_pose=eye, c2n=eye, gripper_in_grasp=g["gripper_in_grasp"], g=g,
                p1=p1, p2=p2, cam=cam, ee=ee)


def main():
    from oracle import mycpp_ref, mycpp_ref_ik
    P, fam, fk_q = inputs()
    out = {"inputs_sha": digest(P, fam, fk_q, IK_UPPER, IK_LOWER, TIGHT_UPPER, TIGHT_LOWER)}
    out["fk_q"] = fk_q
    out["fk_T"] = np.array([mycpp_ref_ik.ik_fk(q) for q in fk_q])
    sols = [mycpp_ref_ik.ik_solutions(T) for T in P]
    out["family"] = fam
    out["nsol"] = np.array([len(s) for s in sols], np.int8)
    inl = lambda s, up, lo: int((~((s > up) | (s < lo)).any(axis=1)).sum())       # noqa: E731  common.cpp:54-67
    out["count_a"] = np.array([inl(s, IK_UPPER, IK_LOWER) for s in sols], np.int8)
    out["count_b"] = np.array([inl(s, TIGHT_UPPER, TIGHT_LOWER) for s in sols], np.int8)
    idx = np.nonzero((fam >= 2) | (np.arange(len(fam)) < 1024) | ((fam == 1) & (np.arange(len(fam)) < N_FK + 512)))[0]
    out["sol_index"] = idx.astype(np.int32)
    out["sol"] = np.concatenate([sols[i] for i in idx] + [np.zeros((0, 7))]).astype(np.float32)
    # the shoulder band, bisected on the wrist-centre radius at three arms
    rng = np.random.RandomState(3)
    bis = []
    for R, h in zip(random_rotations(rng, 3), (-0.3, 0.1, 0.4)):
        lo, hi = 0.5e-3, 1.5e-3
        for _ in range(40):
            mid = 0.5 * (lo + hi)
            n = len(mycpp_ref_ik.ik_solutions(pose_from_wrist(np.array([mid, 0.0, 0.36 + h]), R)))
            lo, hi = (lo, mid) if n > 0 else (mid, hi)
        bis.append(hi)
    out["shoulder_bisect"] = np.array(bis)
    c = filter_case()
    surv, cnt = mycpp_ref.filterGraspPose(c["grasps"], c["sym"], c["nocs_pose"], c["c2n"], c["gripper_in_grasp"], False,
                                          False, 0, c["g"]["open"], c["p1"], c["g"]["enclosed"], c["p2"],
                                          cam_in_world=c["cam"], ee_in_grasp=c["ee"], filter_ik=True, upper=IK_UPPER,
                                          lower=IK_LOWER, counters=True)
    out["filter_survivors"] = mycpp_ref.sort_poses(surv).view(np.uint32)
    out["filter_counters"] = np.array([cnt["approach"], cnt["ik"], cnt["open"], cnt["close"], len(surv)], np.int64)
    out["filter_sha"] = digest(c["grasps"], c["p1"], c["p2"], c["cam"], c["ee"])
    np.savez_compressed(os.path.join(HERE, "ik_iiwa14.npz"), **out)
    print("poses", len(P), "solution sets stored", len(idx), "shoulder band", bis, "filter counters", out["filter_counters"])


if __name__ == "__main__":
    main()
