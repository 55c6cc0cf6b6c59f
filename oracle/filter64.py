"""Float64 restatement of the grasp-pose filter, with a rigorous bound on the float32 pipeline -- ORACLE, test only.

``filter64`` states filterGraspPose (my_cpp/common.cpp:159-299) plainly in float64 numpy, from the same float32-narrowed
inputs that the CUDA kernel (csrc/cg_collide.cu) and oracle/filter_ref.c get:

    g     = (nocs_pose @ canonical_to_nocs) @ (tf_j @ pose_i), first three columns divided by their norms
    approach test (filter_dir): reject when g's x axis points away from the camera, g[2,0] / |g[:3,0]| < 0
    offsets k = 0..4 (adjust) or k = 0: cur = g with t += step_k * g[:3,1], step_k = 0, +s1, -s1, +s2, -s2,
                s1 = 0.001f, s2 = 0.001f + 0.001f (the reference's float accumulator), first collision-free k wins
    gripper pose inv(cur @ gripper_in_grasp); a point p of either set sits at grid coordinates (inv p - origin) / res
    sd by oracle/sdf_ref.py (pinned to meshpy): signed_distance (trilinear, clamped; vectorised as trilinear64, which
    is pinned to it bit for bit), or signed_distance_nearest on the cells inside the grid (out-of-grid points are
    dropped, sdf.py:377-389); a point hits when sd < margin

For every (pose, offset, point set) it keeps m = min over the set of (sd - margin) in float64, and an interval
[lo, hi] that provably contains the minimum the float32 pipeline computes.  A set's verdict is decided when hi < 0
(certain hit) or lo >= 0 (certainly none); a pose is decided when its approach test (|dot| > its bound) and every
offset up to the winner are.  For trilinear lookups lo = m - tau and hi = m + tau, so decided means |m| > tau.

The bound.  Assumptions:
  * the float32 side evaluates the operation order of cg_collide.cu / filter_ref.c (mm4 without contraction,
    normalize_col, affine_inverse by cofactors, fold_grid, three fmas per coordinate, sdf_trilinear), each operation
    correctly rounded to nearest, subnormals kept;
  * u = 2^-24 per float32 rounding; an absolute 2^-140 per operation covers subnormal results; the float64 value of
    every intermediate carries a further 2^-50 relative per operation.
Coordinate error: that operation order is evaluated once more on (value, error) pairs (``_E``): a sum or product
propagates the input errors exactly (|a| db + da |b| + da db for a product, (da + |a/b| db) / (|b| - db) for a
quotient, da / (sqrt(a) + sqrt(a - da)) for a root) and adds one rounding u (|value| + propagated).  The value of that
chain must agree with the plain float64 statement above; their difference is added to the bound.
Trilinear lookup: the interpolant is continuous and, in grid units, Lipschitz along axis a with L_a = the largest
difference of two adjacent cells along a (clamping does not increase distances), so a coordinate error e moves sd by at
most sum_a L_a e_a.  The lookup's own rounding is at most 13 u max|cell| (per-axis weights 2^-25 each, two products
per corner, eight fmas; see shortcut_exact() in cg_collide.cu); 16 u max|cell| + 2^-140 is used.
Nearest lookup: the float32 coordinate rounds to one of the cells that round(c - e) .. round(c + e) reach per axis;
[lo, hi] spans those cells' values (+inf for a cell outside the grid).  Values are exact float32 grid entries.
"""
import numpy as np

from . import sdf_ref

U = 2.0 ** -24
U64 = 2.0 ** -50
TINY = 2.0 ** -140
LOOKUP_U = 16 * U
STEP1 = float(np.float32(0.001))
STEP2 = float(np.float32(np.float32(0.001) + np.float32(0.001)))
OFFSETS = [(0.0, 1.0), (STEP1, 1.0), (STEP1, -1.0), (STEP2, 1.0), (STEP2, -1.0)]   # (step, sign), k = 0..4


class _E:
    """A float64 value with a bound on |float32 pipeline result - value|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.asarray(e, np.float64) + np.zeros_like(self.v)

    @staticmethod
    def _rounded(v, p):
        return _E(v, p + (U + U64) * (np.abs(v) + p) + TINY)

    def __add__(a, b):
        return _E._rounded(a.v + b.v, a.e + b.e)

    def __sub__(a, b):
        return _E._rounded(a.v - b.v, a.e + b.e)

    def __mul__(a, b):
        return _E._rounded(a.v * b.v, np.abs(a.v) * b.e + a.e * np.abs(b.v) + a.e * b.e)

    def __truediv__(a, b):
        d = np.abs(b.v) - b.e
        if not (d > 0).all():
            raise ValueError("filter64: divisor not bounded away from 0")
        q = a.v / b.v
        return _E._rounded(q, (a.e + np.abs(q) * b.e) / d)

    def __neg__(a):
        return _E(-a.v, a.e)


def _sqrt(a):
    v = np.sqrt(a.v)
    lo = np.sqrt(np.maximum(a.v - a.e, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(v + lo > 0, a.e / (v + lo), np.sqrt(a.e))
    return _E._rounded(v, p)


def _fma(a, b, c):
    return _E._rounded(a.v * b.v + c.v, np.abs(a.v) * b.e + a.e * np.abs(b.v) + a.e * b.e + c.e)


def _const(x):
    return _E(np.float64(x))


def _mat(m):
    """(Q,4,4) or (4,4) exact inputs -> list of 16 _E (row-major)."""
    m = np.asarray(m, np.float64)
    return [_E(m[..., r, c]) for r in range(4) for c in range(4)]


def _mm4(A, B):
    out = []
    for r in range(4):
        for c in range(4):
            s = A[r * 4] * B[c]
            for k in (1, 2, 3):
                s = s + A[r * 4 + k] * B[k * 4 + c]
            out.append(s)
    return out


def _normalize_col(G, col):
    x, y, z = G[col], G[4 + col], G[8 + col]
    n = _sqrt((x * x + y * y) + z * z)
    G[col], G[4 + col], G[8 + col] = x / n, y / n, z / n


def _affine_inverse(A):
    a, b, c, d, e, f, g, h, i = A[0], A[1], A[2], A[4], A[5], A[6], A[8], A[9], A[10]
    c00 = e * i - f * h
    c01 = f * g - d * i
    c02 = d * h - e * g
    det = (a * c00 + b * c01) + c * c02
    r = _const(1.0) / det
    inv = [c00 * r, (c * h - b * i) * r, (b * f - c * e) * r, c01 * r, (a * i - c * g) * r, (c * d - a * f) * r,
           c02 * r, (b * g - a * h) * r, (a * e - b * d) * r]
    tx, ty, tz = A[3], A[7], A[11]
    for k in range(3):
        inv.append(-((inv[k * 3] * tx + inv[k * 3 + 1] * ty) + inv[k * 3 + 2] * tz))
    return inv


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def trilinear64(data, coords):
    """sdf_ref.signed_distance (sdf.py:292-343) with flat gathers instead of an (N, 8, 3) corner table: the same
    clamp, corner order, weights (1 - |corner - c|, multiplied x * y * z) and zero for out-of-grid corners.
    tests/test_filter_ref.py pins the two bit for bit."""
    data = np.asarray(data, np.float64)
    dims = np.array(data.shape)
    c = np.array(coords, np.float64).reshape(3, -1)
    for a in range(3):
        c[a] = np.clip(c[a], 0, dims[a] - 1)
    lo = np.floor(c)
    w = [(1 - np.abs(lo[a] - c[a]), 1 - np.abs(lo[a] + 1 - c[a])) for a in range(3)]
    i0 = lo.astype(np.int64)
    ok1 = [i0[a] + 1 < dims[a] for a in range(3)]
    flat = data.reshape(-1)
    sd = np.zeros(c.shape[1])
    for b in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (0, 1, 1), (1, 0, 1), (1, 1, 1)):   # sdf.py:217-225
        inb = np.ones(c.shape[1], bool)
        for a in range(3):
            if b[a]:
                inb &= ok1[a]
        ix, iy, iz = (np.where(inb, i0[a] + b[a], 0) for a in range(3))
        v = np.where(inb, flat[(ix * dims[1] + iy) * dims[2] + iz], 0.0)
        sd = sd + (w[0][b[0]] * w[1][b[1]]) * w[2][b[2]] * v
    return sd


class Grid:
    """One gripper SDF as the kernel sees it: float32 cells, origin and resolution."""

    def __init__(self, sdf):
        self.data = np.ascontiguousarray(sdf["sdf"], dtype=np.float32).astype(np.float64)
        self.origin = _f32(sdf["origin"]).reshape(3)
        self.res = float(np.float32(sdf["res"]))
        self.dims = np.array(self.data.shape)
        d = self.data
        self.lip = np.array([np.abs(np.diff(d, axis=a)).max() if d.shape[a] > 1 else 0.0 for a in range(3)])
        self.vmax = float(np.abs(d).max())

    def folded(self, invE, inv64):
        """fold_grid: camera -> grid map of the float32 side (12 _E, 3x3 then translation), checked against and
        re-centred on the plain float64 map (inv p - origin) / res, whose (3,4) form is returned alongside."""
        M = inv64[:, :3, :3] / self.res
        t = (inv64[:, :3, 3] - self.origin[None]) / self.res
        inv_res = _const(1.0) / _const(self.res)
        G = [invE[k] * inv_res for k in range(9)] + [(invE[9 + k] - _const(self.origin[k])) * inv_res for k in range(3)]
        plain = [M[:, k // 3, k % 3] for k in range(9)] + [t[:, k] for k in range(3)]
        out = []
        for g, p in zip(G, plain):
            dev = np.abs(g.v - p)
            if not (dev <= 1e-6 * (1.0 + np.abs(p))).all():
                raise AssertionError("filter64: the float32 operation chain and the plain statement disagree")
            out.append(_E(p, g.e + dev + 1e-12 * (1.0 + np.abs(p))))
        return out

    def set_minimum(self, GE, pts, mode, margin):
        """GE: 12 _E of shape (Q,) (from folded); pts (P,3) float32-exact.  Returns (m, lo, hi), each (Q,)."""
        Q = GE[0].v.shape[0]
        P = pts.shape[0]
        inf = np.full(Q, np.inf)
        if P == 0:
            return inf, inf.copy(), inf.copy()
        m, lo, hi = inf.copy(), inf.copy(), inf.copy()
        Mv = np.stack([g.v for g in GE[:9]], 1).reshape(Q, 3, 3)
        Me = np.stack([g.e for g in GE[:9]], 1).reshape(Q, 3, 3)
        tv = np.stack([g.v for g in GE[9:]], 1)
        te = np.stack([g.e for g in GE[9:]], 1)
        ax = np.abs(pts)
        qc = max(1, (1 << 18) // P)
        for q0 in range(0, Q, qc):
            sl = slice(q0, min(Q, q0 + qc))
            C = np.einsum("qaj,pj->aqp", Mv[sl], pts) + tv[sl].T[:, :, None]          # (3, q, P) grid units
            # fma(G2, z, fma(G1, y, fma(G0, x, t))): the map's error times |x|, plus three roundings, each at most
            # u (|G0 x| + |G1 y| + |G2 z| + |t| + the propagated error)
            prop = np.einsum("qaj,pj->aqp", Me[sl], ax) + te[sl].T[:, :, None]
            mag = np.einsum("qaj,pj->aqp", np.abs(Mv[sl]), ax) + np.abs(tv[sl]).T[:, :, None]
            Eg = prop + 3 * (U + U64) * (1 + 2 * U) * (mag + prop) + 3 * TINY + 1e-12
            if mode == 0:
                s = trilinear64(self.data, C.reshape(3, -1)).reshape(C.shape[1:])
                tau = np.einsum("a,aqp->qp", self.lip, Eg) + LOOKUP_U * self.vmax + TINY + 1e-14 * self.vmax
                s_lo, s_hi = s - tau, s + tau
            else:
                R = np.rint(C)
                s = self._nearest(R)
                r0, r1 = np.rint(C - Eg), np.rint(C + Eg)
                s_lo, s_hi = s.copy(), s.copy()
                amb = ((r0 != R) | (r1 != R)).any(0)    # a coordinate within its error of a cell boundary
                if amb.any():
                    r0, r1 = r0[:, amb], r1[:, amb]
                    a_lo, a_hi = s_lo[amb], s_hi[amb]
                    for cx in (r0[0], r1[0]):
                        for cy in (r0[1], r1[1]):
                            for cz in (r0[2], r1[2]):
                                v = self._nearest(np.stack([cx, cy, cz]))
                                a_lo, a_hi = np.minimum(a_lo, v), np.maximum(a_hi, v)
                    s_lo[amb], s_hi[amb] = a_lo, a_hi
            m[sl] = (s - margin).min(1)
            lo[sl] = (s_lo - margin).min(1)
            hi[sl] = (s_hi - margin).min(1)
        return m, lo, hi

    def _nearest(self, R):
        """sd at integer grid coordinates R (3, ...); +inf outside the grid (the point is dropped)."""
        shp = R.shape[1:]
        R = R.reshape(3, -1)
        inb = np.ones(R.shape[1], bool)
        for a in range(3):
            inb &= (R[a] >= 0) & (R[a] < self.dims[a])
        out = np.full(R.shape[1], np.inf)
        if inb.any():
            out[inb] = sdf_ref.signed_distance_nearest(self.data, R[:, inb])
        return out.reshape(shp)


def poses64(grasp_poses, symmetry_tfs, nocs_pose, canonical_to_nocs):
    """Plain float64 g (Q,4,4) and the same chain on _E in the kernel's order (16 _E of shape (Q,))."""
    gp = _f32(grasp_poses).reshape(-1, 4, 4)
    st = _f32(symmetry_tfs).reshape(-1, 4, 4)
    N, C = _f32(nocs_pose).reshape(4, 4), _f32(canonical_to_nocs).reshape(4, 4)
    G_, S_ = gp.shape[0], st.shape[0]
    gq = np.repeat(gp, S_, axis=0)                 # q = i * S + j
    sq = np.tile(st, (G_, 1, 1))
    c2c = N @ C
    g = np.einsum("ij,qjk->qik", c2c, np.einsum("qij,qjk->qik", sq, gq))
    g[:, :3, :3] /= np.linalg.norm(g[:, :3, :3], axis=1, keepdims=True)
    gE = _mm4(_mm4(_mat(N), _mat(C)), _mm4(_mat(sq), _mat(gq)))
    for col in range(3):
        _normalize_col(gE, col)
    return g, gE


def filter64(grasp_poses, symmetry_tfs, nocs_pose, canonical_to_nocs, gripper_in_grasp, filter_dir, adjust, sdf_mode,
             sdf_open, open_pts, sdf_encl, encl_pts, margin=0.0, split=False):
    """Same arguments as oracle.filter_ref.filter_ref.  Returns a dict:
    status (Q,) 0 / 1 / 3 / 4 as filter_ref, -1 where undecided; offset (Q,) winner or -1; poses (Q,4,4) float64
    (zero unless accepted); decided (Q,) bool; dot, dot_err (Q,); per set ``open`` / ``encl``: m, lo, hi (Q, 5), NaN
    where the pose never reached that test."""
    margin = float(np.float32(margin))
    g, gE = poses64(grasp_poses, symmetry_tfs, nocs_pose, canonical_to_nocs)
    Q = g.shape[0]
    gig = _f32(gripper_in_grasp).reshape(4, 4)
    gigE = _mat(np.broadcast_to(gig, (Q, 4, 4)))
    so = Grid(sdf_open)
    se = Grid(sdf_encl) if sdf_encl is not None else so
    p1 = _f32(open_pts).reshape(-1, 3)
    p2 = _f32(encl_pts).reshape(-1, 3)
    status = np.full(Q, -1, np.int64)
    offset = np.full(Q, -1, np.int64)
    out = np.zeros((Q, 4, 4))
    decided = np.zeros(Q, bool)
    rec = {s: {f: np.full((Q, 5), np.nan) for f in ("m", "lo", "hi")} for s in ("open", "encl")}

    # approach test: dot = z / |(x, y, z)| of the normalised x axis (the kernel's products by 0 and 1 are exact)
    x, y, z = gE[0], gE[4], gE[8]
    dE = z / _sqrt((x * x + y * y) + z * z)
    dot = g[:, 2, 0] / np.linalg.norm(g[:, :3, 0], axis=1)
    dot_err = dE.e + np.abs(dE.v - dot) + 1e-15
    active = np.ones(Q, bool)
    if filter_dir:
        rej = dot + dot_err < 0
        status[rej], decided[rej] = 1, True
        active = dot - dot_err >= 0                    # undecided approach tests stay undecided
    n_off = 5 if adjust else 1
    for k in range(n_off):
        idx = np.nonzero(active)[0]
        if idx.size == 0:
            break
        step, sign = OFFSETS[k]
        cur = g[idx].copy()
        cur[:, :3, 3] += step * sign * g[idx, :3, 1]
        curE = [_E(e.v[idx], e.e[idx]) for e in gE]
        for r in range(3):
            curE[r * 4 + 3] = curE[r * 4 + 3] + (_const(step) * curE[r * 4 + 1]) * _const(sign)
        inv64 = np.linalg.inv(cur @ gig)
        invE = _affine_inverse(_mm4(curE, [_E(e.v[idx]) for e in gigE]))
        verdict = np.zeros(idx.size, np.int64)        # 1 collides, 0 free, -1 undecided
        lo_o, hi_o = np.full(idx.size, np.inf), np.full(idx.size, np.inf)
        if p1.shape[0]:
            m, lo_o, hi_o = so.set_minimum(so.folded(invE, inv64), p1, sdf_mode, margin)
            rec["open"]["m"][idx, k], rec["open"]["lo"][idx, k], rec["open"]["hi"][idx, k] = m, lo_o, hi_o
        lo_e, hi_e = np.full(idx.size, np.inf), np.full(idx.size, np.inf)
        need = hi_o >= 0                               # the background decides unless the object set surely hits
        if p2.shape[0] and need.any():
            sub = np.nonzero(need)[0]
            GE = [_E(e.v[sub], e.e[sub]) for e in se.folded(invE, inv64)]
            m, lo_e[sub], hi_e[sub] = se.set_minimum(GE, p2, sdf_mode, margin)
            rec["encl"]["m"][idx[sub], k], rec["encl"]["lo"][idx[sub], k] = m, lo_e[sub]
            rec["encl"]["hi"][idx[sub], k] = hi_e[sub]
        verdict[(hi_o < 0) | (hi_e < 0)] = 1
        verdict[(lo_o >= 0) & (lo_e >= 0)] = 0
        verdict[~((hi_o < 0) | (hi_e < 0)) & ~((lo_o >= 0) & (lo_e >= 0))] = -1
        win = idx[verdict == 0]
        status[win], offset[win], decided[win], out[win] = 0, k, True, cur[verdict == 0]
        active[idx[verdict != 1]] = False
        if k == n_off - 1:
            lost = idx[verdict == 1]
            if split and not adjust:                   # 3 = the object set hits, 4 = only the background does
                o_hit, o_free = hi_o[verdict == 1] < 0, lo_o[verdict == 1] >= 0
                status[lost[o_hit]], decided[lost[o_hit]] = 3, True
                status[lost[o_free]], decided[lost[o_free]] = 4, True
            else:
                status[lost], decided[lost] = 3, True
    return {"status": status, "offset": offset, "poses": out, "decided": decided, "dot": dot, "dot_err": dot_err,
            "open": rec["open"], "encl": rec["encl"]}


def compare(res, status, offset, poses, pose_tol=1e-6):
    """Mismatches between a float32 filter result and ``res`` on the decided poses: (n_bad, n_undecided)."""
    d = res["decided"]
    bad = d & ((np.asarray(status) != res["status"]) | (np.asarray(offset) != res["offset"]))
    dp = np.abs(np.asarray(poses, np.float64).reshape(-1, 4, 4) - res["poses"]).reshape(len(d), -1).max(1)
    bad |= d & (dp > pose_tol)
    return int(bad.sum()), int((~d).sum())
