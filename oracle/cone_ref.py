"""CPU ORACLE (test infrastructure only): numpy restatement of the pose enumeration of
dexnet/grasping/grasp_sampler.py:266-286 (sample_one_surface_point) and :191-203 (center_ob_between_gripper).
PINNED: tests/test_cone_golden.py checks it against poses recorded from the reference's own sample_grasps
(tests/golden/make_golden_cone.py).  The rotation helpers it needs are restated here so that the oracle does not import
the product package.

Exact reference of csrc/cg_cone.cu (``exact_poses``, ``exact_center``)
----------------------------------------------------------------------
Both evaluate the operation on the float64 inputs exactly: ``fractions.Fraction`` for every product, sum and the 3x3
inverse, ``decimal`` at 80 digits for the square roots and quotients of the normalisation.  Each returns the exact
value rounded to the nearest float64 and a per-entry bound ``err`` on |kernel's float64 result - that value|, for the
kernel's own operation sequence.  u = 2^-53, g_n = n u / (1 - n u); |A| is the entrywise absolute value.  Every bound
also carries half an ulp of the rounded exact value, and is itself evaluated in float64 (relative error a few u, which
the factor 2 of ``encoder_ref.bound_ratio`` absorbs).

cone_pose_kernel, pose ((s * NR + r) * ND + k), NR = 1 + NS * NI:
  rotation   r >= 1: T = fl(R0 Rs), R^ = fl(T Ri), each entry a 3-term fma chain (products and sums rounded at most 3
             times in any order: |fl(x.y) - x.y| <= g_3 |x|.|y|).  With |T^| <= (1 + g_3) |R0||Rs|:
                 |R^ - R| <= eR = (2 g_3 + g_3^2) |R0||Rs||Ri|                       (r = 0: R = R0, eR = 0)
  normalise  column v (exact) -> q = v / ||v||.  For any w, ||w/||w|| - v/||v|| ||_2 <= 2 ||w - v||_2 / ||v||, so the
             kernel's input column moves q by at most 2 ||eR_col||_2 / ||v|| in every entry.  The kernel's norm
             sqrt(fl(fl(x^2 + y^2) + z^2)) of nonnegative terms is ||v^|| (1 + e), |e| <= en = g_3/2 (1 + g_3) + u (1 + g_3),
             and the quotient rounds once more:
                 eQ_i = 2 ||eR_col||_2 / ||v|| + (u + en) / (1 - en) (|q_i| + 2 ||eR_col||_2 / ||v||)
  translate  t_i = p_i + b a_i + a_i d (b = init_bite, a = q[:, 0]), three roundings of terms bounded by
             |p_i| + (|b| + |d|) |a^_i|, plus the propagated |a^_i - a_i| <= eQ_i0:
                 eT_i = (|b| + |d|) eQ_i0 + g_4 (|p_i| + (|b| + |d|) (|a_i| + eQ_i0))
  bottom row (0, 0, 0, 1) is exact.

center_grasp_kernel, given the float64 pose it centres (the uncentred kernel output):
  cofactor row  (ix, iy, iz) = (fg - di, ai - cg, cd - af) / det of R = [[a b c] [d e f] [g h i]].  A 2-term
             difference rounds at most twice, fma or not: |dn_k| <= g_2 N_k, N_k = |products|.  det = a m1 - b m2 + c m3
             over the three minors: |ddet| <= g_5 D, D = |a| M1 + |b| M2 + |c| M3.  Then
                 e_k = (g_2 N_k + |row_k| g_5 D) / (|det| - g_5 D),   eRow_k = e_k + u (|row_k| + e_k)
  each y_j   fma(iz, pz - tz, fma(iy, py - ty, ix (px - tx))): the differences round once (u |p - t|), the chain
             three times, and the row carries eRow:
                 eY_j = sum_k |p_jk - t_k| (eRow_k + g_4 (|row_k| + eRow_k))
  extent     fmin / fmax are exact, so max and min move by at most E = max_j eY_j (over all points); cy = fl(hi + lo) / 2:
                 eCY = E (1 + u) + u |cy|
  shift      t'_i = fma(T[i, 1], cy, t_i), one rounding:  eT'_i = |T[i, 1]| eCY + u (|t'_i| + |T[i, 1]| eCY)
             The rotation block and bottom row pass through unchanged (err 0).
``exact_center`` evaluates the y values exactly only for points within the bound of the float64 extremes (every point
whose interval [y - eY, y + eY] reaches past the best lower bound of the max, or of the min), which keeps it fast.
"""
import decimal
import math
from fractions import Fraction

import numpy as np


def _rot_x(a):
    si, ci = math.sin(a), math.cos(a)
    return np.array([[1.0, -(ci * 0.0), si * 0.0], [0.0, ci, -si], [-0.0, si, ci]])     # euler_matrix(a,0,0,'sxyz')[:3,:3]


def _normalize_cols(R):
    out = R.copy()
    out /= np.linalg.norm(R, axis=0).reshape(1, 3)
    return out


def _dir_to_rot(direction, ref):
    direction = direction / np.linalg.norm(direction)
    v = np.cross(direction, ref)
    if (v == 0).all():
        return np.eye(3)
    s = np.linalg.norm(v)
    c = direction.dot(ref)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    if s == 0:
        R = np.array([[1.0, 0, 0], [0, -1, 0], [0, 0, -1]])
    else:
        R = (np.identity(3) + K + K.dot(K) * (1 - c) / (s ** 2)).T
    return _normalize_cols(R)


def enumerate_poses(surface_pts, R0s, sphere_pts, hand_depth, approach_step, init_bite, points_for_center=None):
    poses = []
    for p, R0 in zip(surface_pts, R0s):
        Rs = [R0]
        for sp in sphere_pts:
            R_sphere = _dir_to_rot(sp.copy(), np.array([1, 0, 0]))
            for x_rot in np.arange(0, 180, 30):
                Rs.append(R0 @ R_sphere @ _rot_x(x_rot * np.pi / 180))
        for R in Rs:
            R = _normalize_cols(R)
            a = R[:, 0]
            for d in np.arange(0, hand_depth, approach_step):
                T = np.eye(4)
                T[:3, :3] = R
                T[:3, 3] = p + init_bite * a + a * d
                poses.append(T)
    poses = np.array(poses)
    if points_for_center is not None:
        homo = np.concatenate((points_for_center, np.ones((points_for_center.shape[0], 1))), axis=-1)
        for i in range(len(poses)):
            q = (np.linalg.inv(poses[i]) @ homo.T).T[:, :3]
            c = (q.max(axis=0) + q.min(axis=0)) / 2
            off = np.eye(4)
            off[:3, 3] = [0, c[1], 0]
            poses[i] = poses[i] @ off
    return poses


def poses_from_tables(surface_pts, R0s, R_sphere, R_inplane, depths, init_bite):
    """``enumerate_poses`` with the sphere and in-plane rotations given as tables (NS,3,3), (NI,3,3), in the kernel's
    pose order; numpy arithmetic, one rotation at a time."""
    NI = len(R_inplane)
    poses = []
    for p, R0 in zip(np.asarray(surface_pts, np.float64), np.asarray(R0s, np.float64)):
        Rs = [R0] + [R0 @ R_sphere[j // NI] @ R_inplane[j % NI] for j in range(len(R_sphere) * NI)]
        for R in Rs:
            R = _normalize_cols(R)
            a = R[:, 0]
            for d in depths:
                T = np.eye(4)
                T[:3, :3] = R
                T[:3, 3] = p + init_bite * a + a * d
                poses.append(T)
    return np.array(poses).reshape(-1, 4, 4)


U = 2.0 ** -53
_DEC = decimal.Context(prec=80)


def _g(n):
    return n * U / (1 - n * U)


def _frm(M):
    return [[Fraction(float(x)) for x in row] for row in M]


def _mm(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def _dec(f):
    return _DEC.divide(decimal.Decimal(f.numerator), decimal.Decimal(f.denominator))


def _half_ulp(x):
    return np.spacing(np.abs(x)) / 2


def exact_poses(surface_pts, R0s, R_sphere, R_inplane, depths, init_bite, index):
    """The poses ``index`` (flat, kernel order) of cone_pose_kernel's enumeration, exactly: returns (ref (n,4,4), the
    exact poses rounded to float64; err (n,4,4), the bound on the kernel's error in the module docstring).
    ``R_sphere`` may be empty (NS = 0)."""
    surf = np.asarray(surface_pts, np.float64).reshape(-1, 3)
    R0s = np.asarray(R0s, np.float64).reshape(-1, 3, 3)
    Rsph = np.asarray(R_sphere, np.float64).reshape(-1, 3, 3)
    Rinp = np.asarray(R_inplane, np.float64).reshape(-1, 3, 3)
    depths = np.asarray(depths, np.float64).reshape(-1)
    NS, NI, ND = len(Rsph), len(Rinp), len(depths)
    NR = 1 + NS * NI
    index = np.asarray(index, np.int64).reshape(-1)
    g3, g4 = _g(3), _g(4)
    en = g3 / 2 * (1 + g3) + U * (1 + g3)
    fsph, finp = [_frm(M) for M in Rsph], [_frm(M) for M in Rinp]
    b, bd = float(init_bite), decimal.Decimal(float(init_bite))
    rot = {}
    ref = np.zeros((len(index), 4, 4))
    err = np.zeros((len(index), 4, 4))
    for n, i in enumerate(index):
        s, r, k = int(i) // (NR * ND), int(i) // ND % NR, int(i) % ND
        if (s, r) not in rot:
            R = _frm(R0s[s])
            eR = np.zeros((3, 3))
            if r:
                js, ji = (r - 1) // NI, (r - 1) % NI
                R = _mm(_mm(R, fsph[js]), finp[ji])
                eR = (2 * g3 + g3 * g3) * ((np.abs(R0s[s]) @ np.abs(Rsph[js])) @ np.abs(Rinp[ji]))
            q = [[None] * 3 for _ in range(3)]
            eQ = np.zeros((3, 3))
            for c in range(3):
                nrm = _dec(R[0][c] ** 2 + R[1][c] ** 2 + R[2][c] ** 2).sqrt(_DEC)
                for j in range(3):
                    q[j][c] = _DEC.divide(_dec(R[j][c]), nrm)
                move = 2 * math.sqrt(float((eR[:, c] ** 2).sum())) / float(nrm)
                qf = np.array([abs(float(q[j][c])) for j in range(3)])
                eQ[:, c] = move + (U + en) / (1 - en) * (qf + move)
            rot[s, r] = q, eQ
        q, eQ = rot[s, r]
        d, dd = float(depths[k]), decimal.Decimal(float(depths[k]))
        for j in range(3):
            for c in range(3):
                ref[n, j, c] = float(q[j][c])
            a = q[j][0]
            t = _DEC.add(_DEC.add(decimal.Decimal(float(surf[s, j])), _DEC.multiply(bd, a)), _DEC.multiply(a, dd))
            ref[n, j, 3] = float(t)
            w = abs(b) + abs(d)
            err[n, j, 3] = w * eQ[j, 0] + g4 * (abs(surf[s, j]) + w * (abs(float(a)) + eQ[j, 0]))
        err[n, :3, :3] = eQ
        ref[n, 3, 3] = 1.0
    err[:, :3] += _half_ulp(ref[:, :3])
    return ref, err


def _cofactor_row(P):
    """Second row of inv(R) by cofactors for float64 poses (n,4,4), with its bound (module docstring): returns
    (row (n,3), eRow (n,3))."""
    a, b, c, d, e, f, g, h, i = (P[:, r, col] for r in range(3) for col in range(3))
    det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g)
    D = np.abs(a) * (np.abs(e * i) + np.abs(f * h)) + np.abs(b) * (np.abs(d * i) + np.abs(f * g)) + \
        np.abs(c) * (np.abs(d * h) + np.abs(e * g))
    num = np.stack([f * g - d * i, a * i - c * g, c * d - a * f], 1)
    N = np.stack([np.abs(f * g) + np.abs(d * i), np.abs(a * i) + np.abs(c * g), np.abs(c * d) + np.abs(a * f)], 1)
    row = num / det[:, None]
    den = np.abs(det) - _g(5) * D
    assert (den > 0).all(), "pose rotation too close to singular for the centring bound"
    ek = (_g(2) * N + np.abs(row) * _g(5) * D[:, None]) / den[:, None]
    # the float64 row here is itself within ek of the exact one: widen so that |row| bounds the exact row's magnitude
    return row, ek + U * (np.abs(row) + 2 * ek)


def exact_center(poses, points):
    """center_grasp_kernel on float64 poses (n,4,4) over object points (M,3), exactly: returns (ref, err) as
    ``exact_poses`` does.  Only the translation column changes; elsewhere ref = poses and err = 0."""
    P = np.asarray(poses, np.float64).reshape(-1, 4, 4)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    row, eRow = _cofactor_row(P)
    g4 = _g(4)
    ref, err = P.copy(), np.zeros_like(P)
    fp = [[Fraction(float(x)) for x in p] for p in pts]
    for n in range(len(P)):
        diff = pts - P[n, :3, 3]
        y = diff @ row[n]
        eY = (np.abs(diff) * (1 + U)) @ (eRow[n] + g4 * (np.abs(row[n]) + eRow[n]))
        E = float(eY.max())
        hi_c = np.nonzero(y + eY >= (y - eY).max())[0]
        lo_c = np.nonzero(y - eY <= (y + eY).min())[0]
        R = _frm(P[n, :3, :3])
        (a, b_, c), (d, e, f), (g, h, i) = R
        det = a * (e * i - f * h) - b_ * (d * i - f * g) + c * (d * h - e * g)
        rw = [(f * g - d * i) / det, (a * i - c * g) / det, (c * d - a * f) / det]
        t = [Fraction(float(x)) for x in P[n, :3, 3]]
        yx = {j: sum(rw[k] * (fp[j][k] - t[k]) for k in range(3)) for j in set(hi_c) | set(lo_c)}
        cy = (max(yx[j] for j in hi_c) + min(yx[j] for j in lo_c)) / 2
        eCY = E * (1 + U) + U * abs(float(cy))
        for k in range(3):
            col = float(P[n, k, 1])
            tn = t[k] + Fraction(col) * cy
            ref[n, k, 3] = float(tn)
            err[n, k, 3] = abs(col) * eCY + U * (abs(float(tn)) + abs(col) * eCY) + _half_ulp(ref[n, k, 3])
    return ref, err
