"""Closed-form inverse kinematics of the KUKA iiwa14 with joint 2 fixed at 0, in float64 numpy: the CPU twin of
catgrasp_b200/csrc/cg_ik.cu (same steps, same constants, same branch order), and a float64 forward kinematics.

The chain (measured from the reference's generated ikfast solver, tests/golden/make_golden_ik.py):
    base -> shoulder 0.36 m, shoulder -> elbow 0.42 m, elbow -> wrist 0.40 m, wrist -> end effector 0.081 m,
    joint axes z, +y, z, -y, z, +y, z; at q = 0 the end effector is at (0, 0, 1.261) with identity rotation.
With joint 2 = 0 the shoulder (joints 0, 1) and the wrist (joints 4, 5, 6) are spherical, so the wrist centre
p - 0.081 R z fixes q0, q1, q3 and R_03^T R the z-y-z wrist angles q4, q5, q6.

Branch slot b = 4*s + 2*e + w (8 slots, unused ones NaN):
    s = 0: q0 = atan2(y, x) of the wrist centre, s = 1: q0 + pi (the arm reaches over the base axis);
    e = 0: q3 = +acos(c3) >= 0, e = 1: q3 = -acos(c3);
    w = 0: q5 = acos(c5) >= 0 (ikfast reads q5 off the cosine), w = 1: the flipped wrist (q4 + pi, -q5, q6 + pi).
Every angle is wrapped to [-pi, pi].  The reference's special cases (bisected against ikfast; constants below):
    * no solution when the wrist centre is within SHOULDER_BAND of the joint-0 axis;
    * no solution when c3 lies outside [-1 - REACH_SLACK, 1 + REACH_SLACK]; inside that slack c3 is clamped;
    * e = 1 is dropped when the two elbow branches coincide (|sin q3| < ELBOW_MERGE / 2);
    * w = 1 is dropped when the wrist is singular (|sin q5| < WRIST_SINGULAR): then q5 = 0 or pi, q6 = 0 and q4
      carries q4 + q6 (or q4 - q6 at q5 = pi);
    * both wrist slots of an arm branch are dropped when WRIST_SINGULAR <= |sin q5| < WRIST_DROP.
Near the elbow and wrist thresholds ikfast's answer depends on the float32 rounding of the input (its consistency
checks compare against the un-orthonormal matrix); in_band() flags the poses where that happens, and the solver only
pins the behaviour outside them.
"""
import numpy as np

D_BS, D_SE, D_EW, D_WF = 0.36, 0.42, 0.40, 0.081

# ikfast returns nothing when the wrist centre's distance from the joint-0 axis is below 1 mm (bisected to 1e-3 m at
# several arm configurations; a reachable pose that the reference calls IK-infeasible)
SHOULDER_BAND = 1e-3
# the law-of-cosines value c3 is accepted up to 1e-7 beyond [-1, 1] and clamped (ikfast's IKFAST_SINCOS_THRESH)
REACH_SLACK = 1e-7
# two solutions whose sine and cosine differ by less than 1e-6 are one (ikfast's IKFAST_SOLUTION_THRESH); for the
# elbow pair +-q3 that is |2 sin q3| < 1e-6
ELBOW_MERGE = 1e-6
# below this |sin q5| ikfast takes the wrist as singular and returns one lumped solution per arm branch (most poses
# with q5 <= 3e-7 give 6 solutions; q5 = 1e-6 gives 6 or 4)
WRIST_SINGULAR = 1e-6
# between WRIST_SINGULAR and this |sin q5| ikfast returns neither wrist solution of the arm branch (its residual checks
# fail on the float32 input): over 60 random arms, the last q5 with a missing branch was 1.6e-3 .. 4.9e-3 (median
# 2.5e-3), and from 1e-5 to 2e-4 every arm lost the branch
WRIST_DROP = 2.5e-3
# ikfast checks each solution against the input matrix, which the reference passes unchecked (a float32 product, maybe
# of a scaled or sheared pose): a solution is kept only when its wrist rotation Rz(q4) Ry(q5) Rz(q6) reproduces
# R_03^T R to within this, entry by entry.  Tolerances from 1e-5 to 1e-4 all reproduce ikfast on the fixture and on
# the filter cases (whose non-orthonormal poses ikfast rejects); 3e-6 does not.
ROT_RESIDUAL = 3e-5

# Where ikfast's answer flickers with the input's rounding (in_band): |sin q5| below 1e-5 or in [2e-4, 6e-3];
# |sin q3| below 2e-2 (from 1e-9 to 1e-2 ikfast returns 0, 4 or 8 solutions for the same arm); and 1e-6 around the
# shoulder band and the reach boundary.
BAND_WRIST = ((0.0, 1e-5), (2e-4, 6e-3))
BAND_ELBOW = 2e-2
BAND_LINEAR = 1e-6


def _wrist_residual(q4, q5, q6, M):
    """max |Rz(q4) Ry(q5) Rz(q6) - M| over the 9 entries (M = R_03^T R)."""
    c4, s4, c5, s5, c6, s6 = np.cos(q4), np.sin(q4), np.cos(q5), np.sin(q5), np.cos(q6), np.sin(q6)
    W = [c4 * c5 * c6 - s4 * s6, -c4 * c5 * s6 - s4 * c6, c4 * s5,
         s4 * c5 * c6 + c4 * s6, -s4 * c5 * s6 + c4 * c6, s4 * s5,
         -s5 * c6, s5 * s6, c5]
    r = np.zeros_like(q4)
    for k in range(9):
        r = np.maximum(r, np.abs(W[k] - M[:, k // 3, k % 3]))
    return r


def _wrap(a):
    a = np.where(a > np.pi, a - 2.0 * np.pi, a)
    return np.where(a < -np.pi, a + 2.0 * np.pi, a)


def _rz(t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _ry(t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


def _tz(d):
    T = np.eye(4)
    T[2, 3] = d
    return T


def _r(R):
    T = np.eye(4)
    T[:3, :3] = R
    return T


def iiwa14_fk(q):
    """(..., 7) joint angles -> (..., 4, 4) float64 end-effector pose in the base frame."""
    q = np.asarray(q, np.float64)
    flat = q.reshape(-1, 7)
    out = np.empty((flat.shape[0], 4, 4))
    for n, a in enumerate(flat):
        T = _tz(D_BS) @ _r(_rz(a[0])) @ _r(_ry(a[1])) @ _r(_rz(a[2])) @ _tz(D_SE) @ _r(_ry(-a[3])) @ _r(_rz(a[4])) \
            @ _tz(D_EW) @ _r(_ry(a[5])) @ _r(_rz(a[6])) @ _tz(D_WF)
        out[n] = T
    return out.reshape(q.shape[:-1] + (4, 4))


def iiwa14_ik(ee_in_base, upper=None, lower=None):
    """ee_in_base (Q,4,4) (float32 values, widened to float64) -> (count (Q,) int8, solutions (Q,8,7) float64).
    count = number of valid slots with lower[i] <= q[i] <= upper[i] for all 7 joints (all valid slots when the limits
    are None)."""
    sol, _ = _solve(ee_in_base, False)
    valid = ~np.isnan(sol[:, :, 0])
    if upper is None:
        count = valid.sum(axis=1)
    else:
        up = np.asarray(upper, np.float64)[:7]
        lo = np.asarray(lower, np.float64)[:7]
        count = (valid & ((sol >= lo) & (sol <= up)).all(axis=2)).sum(axis=1)
    return count.astype(np.int8), sol


def in_band(ee_in_base):
    """(Q,) bool: the pose lies where ikfast's answer depends on the input's rounding (BAND_* above), so neither the
    solution set nor the count is pinned there."""
    return _solve(ee_in_base, True)[1]


def _solve(ee_in_base, want_band):
    T = np.asarray(ee_in_base).reshape(-1, 4, 4).astype(np.float64)
    Q = T.shape[0]
    sol = np.full((Q, 8, 7), np.nan)
    R = T[:, :3, :3]
    p = T[:, :3, 3]
    finite = np.isfinite(T[:, :3, :]).reshape(Q, -1).all(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        vx = p[:, 0] - D_WF * R[:, 0, 2]
        vy = p[:, 1] - D_WF * R[:, 1, 2]
        vz = (p[:, 2] - D_WF * R[:, 2, 2]) - D_BS
        rho = np.sqrt(vx * vx + vy * vy)
        c3 = ((vx * vx + vy * vy + vz * vz) - (D_SE * D_SE + D_EW * D_EW)) / (2.0 * D_SE * D_EW)
        ok = finite & (rho >= SHOULDER_BAND) & (c3 >= -1.0 - REACH_SLACK) & (c3 <= 1.0 + REACH_SLACK)
        band = None
        if want_band:
            reach = np.sqrt(vx * vx + vy * vy + vz * vz)
            band = finite & ((np.abs(rho - SHOULDER_BAND) < BAND_LINEAR) |
                             (np.abs(reach - (D_SE + D_EW)) < BAND_LINEAR) | (np.abs(reach - abs(D_SE - D_EW)) < BAND_LINEAR))
        c3 = np.clip(c3, -1.0, 1.0)
        s3 = np.sqrt(1.0 - c3 * c3)
        elbow_two = (2.0 * s3) >= ELBOW_MERGE
        if band is not None:
            band |= ok & (s3 < BAND_ELBOW)
        q0a = np.arctan2(vy, vx)
        for s in range(2):
            q0 = q0a if s == 0 else _wrap(q0a + np.pi)
            r = rho if s == 0 else -rho
            for e in range(2):
                q3 = np.arctan2(s3 if e == 0 else -s3, c3)
                ux = -D_EW * np.sin(q3)
                uz = D_SE + D_EW * np.cos(q3)
                q1 = _wrap(np.arctan2(r, vz) - np.arctan2(ux, uz))
                # M = R_03^T R with R_03 = Rz(q0) Ry(q1 - q3)
                c0, s0 = np.cos(q0), np.sin(q0)
                b = q1 - q3
                cb, sb = np.cos(b), np.sin(b)
                # rows of R_03^T: Ry(b)^T Rz(q0)^T
                a0 = np.stack([cb * c0, cb * s0, -sb * np.ones_like(c0)], axis=1)
                a1 = np.stack([-s0, c0, np.zeros_like(c0)], axis=1)
                a2 = np.stack([sb * c0, sb * s0, cb * np.ones_like(c0)], axis=1)
                M = np.stack([np.einsum("qk,qkc->qc", a, R) for a in (a0, a1, a2)], axis=1)
                s5 = np.sqrt(M[:, 0, 2] * M[:, 0, 2] + M[:, 1, 2] * M[:, 1, 2])
                c5 = M[:, 2, 2]
                sing = s5 < WRIST_SINGULAR
                q4g = np.arctan2(M[:, 1, 2], M[:, 0, 2])
                q5g = np.arccos(np.clip(c5, -1.0, 1.0))
                q6g = np.arctan2(M[:, 2, 1], -M[:, 2, 0])
                # singular: Rz(q4) Ry(0 or pi) Rz(q6) = Rz(q4 +- q6) (Ry(pi) flips the sense of the second z turn)
                q4s = np.where(c5 >= 0.0, np.arctan2(M[:, 1, 0], M[:, 0, 0]), np.arctan2(-M[:, 1, 0], -M[:, 0, 0]))
                q5s = np.where(c5 >= 0.0, 0.0, np.pi)
                drop = ~sing & (s5 < WRIST_DROP)
                if band is not None:
                    live = ok & (elbow_two | (e == 0))
                    band |= live & ((s5 < BAND_WRIST[0][1]) | ((s5 >= BAND_WRIST[1][0]) & (s5 < BAND_WRIST[1][1])))
                for w in range(2):
                    slot = 4 * s + 2 * e + w
                    valid = ok & (elbow_two | (e == 0)) & (~sing | (w == 0)) & ~drop
                    if w == 0:
                        q4 = np.where(sing, q4s, q4g)
                        q5 = np.where(sing, q5s, q5g)
                        q6 = np.where(sing, 0.0, q6g)
                    else:
                        q4, q5, q6 = _wrap(q4g + np.pi), -q5g, _wrap(q6g + np.pi)
                    valid = valid & (_wrist_residual(q4, q5, q6, M) <= ROT_RESIDUAL)
                    vals = np.stack([q0, q1, np.zeros_like(q0), q3, q4, q5, q6], axis=1)
                    sol[:, slot, :] = np.where(valid[:, None], vals, np.nan)
    return sol, band
