"""CPU ORACLE (test infrastructure only): one hypothesis of the 9-DoF RANSAC (aligning.py:36-67) in high precision,
with signed gate margins and error bounds, so that the CUDA kernel (csrc/cg_ransac.cu) can be checked hypothesis by
hypothesis.

Per hypothesis (ids -> four (double)(float)-narrowed points, as cv2.estimateAffine3D narrows them to CV_32F):

* The affine [A | t].  cv2 solves the 12x12 system of 4 points (M = [p_i, 1] in three diagonal blocks, so M's
  singular values each appear three times) with DECOMP_SVD.  It drops singular values <= 2 DBL_EPSILON * (sum of
  the 12) = 6 DBL_EPSILON * sum_j sigma_j(M): bisecting on the smallest singular value of a 4-point system with
  OpenCV 4.13 puts the cut at 1.996 * DBL_EPSILON * (sum of the 12).  A nonsingular system is solved exactly
  (fractions); an exactly singular one (exact rational determinant 0) gets the minimum-norm solution pinv(M) B.  A
  nonsingular system whose smallest singular value lies within [0.8, 1.25] x the cut is *undecided*: cv2 computes
  its singular values to ~u sigma_max, about a tenth of the cut.  tests/test_ransac_ref.py checks the cut against
  cv2 on subsets at 0.7x and 1.4x of it.
  The kernel switches to its minimum-norm solve on an absolute LU pivot < 1e-12, not on cv2's relative cut, so a
  nonsingular system below 1.25 x the cut whose pivots all stay >= 1e-12 (possible only with large coordinates;
  NOCS coordinates lie in the unit cube) is solved by LU there: info["lu_may_differ"] marks such systems, and the
  kernel tests count them as undecided.
* Every gate quantity with its signed margin (>= 0 passes, as in the kernel and aligning.py): the column norms
  against min_scale / max_scale, the singular values of R = A / scales against 0.8 / 1.2, det(U V^T), the canonical
  extents of the target (true inverse S^-1 Ro^T) against max_dims.
* valid, T = [U V^T diag(s) | t] and the inlier count as an interval [lo, hi].
* ``bound``: a per-hypothesis bound on |T_kernel - T| (elementwise).  A gate whose margin lies inside the error
  its quantity inherits from this bound is undecided, and so is the hypothesis unless another gate fails outright.

The error bound.  The kernel solves M X = B by LU with partial pivoting in float64 (unit roundoff u = 2^-53).
Higham (Accuracy and Stability, Thm 9.4 and 7.2): the computed X solves (M + dM) X = B with
|dM| <= gamma_3n |L||U|, and ||X - X*|| / ||X|| <= kappa(M) ||dM|| / ||M|| / (1 - ...).  With n = 4,
||  |L||U| || <= n * rho * ||M|| and growth rho <= 2^(n-1) = 8, so ||dM|| / ||M|| <= 3n * n * 8 u = 384 u:
C_SOLVE = 384.  The minimum-norm path (one-sided Jacobi SVD, backward stable at a few u per rotation) obeys Wedin's
least-squares bound ||dX|| <= kappa u c (2 ||X|| + (kappa + 1) ||r|| / ||M||), r = B - M X; the same C_SOLVE
covers it (on 3000 random singular subsets the kernel's routine on the host, and cv2, stay below 1x of
u kappa^2 ||X||).  kappa is sigma_max / sigma_min over the kept singular values.  cv2 solves the same system by
SVD with an error of the same form, so decisions are compared only where both sit outside the bound.
The steps after the solve are well conditioned on a valid hypothesis (scales >= min_scale > 0, singular values of R
in [0.8, 1.2]): a column norm moves by at most sqrt(3) dX, R = A / s by (dX + ds) / s_min per entry, the polar factor
by ||dR||_F / sigma_min(R) (Higham, Thm 8.9), T's linear part by d(Ro) s_max + ds; 64 u of slack covers the
kernel's own float64 arithmetic after the solve (Jacobi 3x3, products of O(1) numbers).

Inlier count.  The kernel forms e = |T [s, 1] - tgt| with FMA-contracted rows, then sqrt, in float64.  A point is
decided when |e - thr| exceeds sqrt(3) * bound * (|s|_1 + 1) + 32 u * (|T| |[s, 1]| + |tgt|): the first term is the
kernel's T error, the second both sides' rounding of the residual.  lo counts decided inliers, hi adds the
undecided ones.
"""
from fractions import Fraction

import mpmath as mp
import numpy as np

U = 2.0 ** -53
EPS = 2.0 ** -52
C_SOLVE = 384.0
CV2_CUT = 6.0 * EPS            # relative to sum_j sigma_j(M)
SV_LO, SV_HI = 0.8, 1.2
DPS = 50


def narrow(src, tgt, ids):
    """(H,4,3) float64 sample points after the float32 round trip that cv2 and the kernel apply."""
    ids = np.asarray(ids).reshape(-1, 4)
    s = np.asarray(src, np.float64)[ids].astype(np.float32).astype(np.float64)
    d = np.asarray(tgt, np.float64)[ids].astype(np.float32).astype(np.float64)
    return s, d


def _det4(rows):
    """Exact determinant of a 4x4 matrix of Fractions (fraction-free expansion by Gaussian elimination)."""
    m = [r[:] for r in rows]
    det = Fraction(1)
    for c in range(4):
        p = next((r for r in range(c, 4) if m[r][c] != 0), None)
        if p is None:
            return Fraction(0)
        if p != c:
            m[c], m[p] = m[p], m[c]
            det = -det
        det *= m[c][c]
        for r in range(c + 1, 4):
            f = m[r][c] / m[c][c]
            if f:
                for k in range(c, 4):
                    m[r][k] -= f * m[c][k]
    return det


def _solve_exact(M, B):
    """Exact solution of the nonsingular 4x4 system M X = B (Fractions, three right-hand sides)."""
    M = [r[:] for r in M]
    B = [r[:] for r in B]
    for c in range(4):
        p = next(r for r in range(c, 4) if M[r][c] != 0)
        M[c], M[p], B[c], B[p] = M[p], M[c], B[p], B[c]
        for r in range(c + 1, 4):
            f = M[r][c] / M[c][c]
            if f:
                for k in range(c, 4):
                    M[r][k] -= f * M[c][k]
                for k in range(3):
                    B[r][k] -= f * B[c][k]
    X = [[None] * 3 for _ in range(4)]
    for k in range(3):
        for c in range(3, -1, -1):
            X[c][k] = (B[c][k] - sum(M[c][j] * X[j][k] for j in range(c + 1, 4))) / M[c][c]
    return X


def solve_affine(s4, d4):
    """cv2.estimateAffine3D on 4 narrowed points: exact, or pinv at 50 digits.  Returns (X (4x3 mp), info) with
    info = {kappa, sigma_max, resid, singular, cut_undecided, lu_may_differ (bools)}."""
    with mp.workdps(DPS):
        M = mp.matrix([[mp.mpf(float(v)) for v in p] + [mp.mpf(1)] for p in s4])
        B = mp.matrix([[mp.mpf(float(v)) for v in p] for p in d4])
        exact_singular = _det4([[Fraction(float(v)) for v in p] + [Fraction(1)] for p in s4]) == 0
        sig64 = np.linalg.svd(np.c_[np.asarray(s4, np.float64), np.ones(4)], compute_uv=False)
        if exact_singular or sig64[-1] < 1e-9 * sig64[0]:
            U_, S, V = mp.svd_r(M)
            sig = [S[i] for i in range(4)]
        else:                   # float64 singular values are accurate to ~u sigma_max: enough for kappa and the cut
            sig = [mp.mpf(float(v)) for v in sig64]
        cut = CV2_CUT * sum(sig)
        smin = min(sig)
        cut_undecided = (not exact_singular) and 0.8 * cut <= smin <= 1.25 * cut
        lu_may_differ = (not exact_singular) and smin <= 1.25 * cut
        truncate = exact_singular or smin < cut
        if not truncate:
            Xq = _solve_exact([[Fraction(float(v)) for v in p] + [Fraction(1)] for p in s4],
                              [[Fraction(float(v)) for v in p] for p in d4])
            X = mp.matrix([[mp.mpf(x.numerator) / x.denominator for x in row] for row in Xq])
            kept = sig
        else:
            # pinv(M) B = V diag(1/sigma_kept) U^T B  (svd_r: M = U diag(S) V, V's rows are the right vectors)
            X = mp.matrix(4, 3)
            kept = [s for s in sig if s > cut]
            for i in range(4):
                if not sig[i] > cut:
                    continue
                for k in range(3):
                    proj = sum(U_[r, i] * B[r, k] for r in range(4)) / sig[i]
                    for j in range(4):
                        X[j, k] += V[i, j] * proj
        R = M * X - B
        resid = max(abs(R[i, k]) for i in range(4) for k in range(3))
        info = {"kappa": float(max(kept) / min(kept)), "sigma_max": float(max(sig)), "resid": float(resid),
                "singular": bool(truncate), "cut_undecided": bool(cut_undecided), "lu_may_differ": bool(lu_may_differ)}
        return X, info


def column_scales(A):
    """Per-axis scales = column norms of the affine's linear part (aligning.py:41)."""
    return [mp.sqrt(sum(A[i, j] ** 2 for i in range(3))) for j in range(3)]


def polar_det(Ro):
    """det(U V^T): +-1 on a well-defined polar factor; aligning.py:52 rejects < 0."""
    return mp.det(Ro)


def canonical_inverse(Ro, sc, t):
    """inv(T) = [S^-1 Ro^T | -S^-1 Ro^T t] (3,4) float64, the map of the target into the canonical frame (aligning.py:59)."""
    Ti = np.zeros((3, 4))
    for i in range(3):
        for j in range(3):
            Ti[i, j] = float(Ro[j, i] / sc[i])
        Ti[i, 3] = float(-(sum(Ro[j, i] / sc[i] * t[j] for j in range(3))))
    return Ti


def _decide(margin, band):
    """True / False / None (undecided) for a gate that passes at margin >= 0."""
    if margin > band:
        return True
    if margin < -band:
        return False
    return None


def hypothesis(s4, d4, target, thr, min_scale, max_scale, max_dims, source=None):
    """One hypothesis.  Returns a dict: valid (True/False/None), T (4,4) float64 or None, bound, lo, hi (counts, when
    source is given and T exists), gates {name: (margin, band)}, info."""
    min_scale = np.asarray(min_scale, np.float64)
    max_scale = np.asarray(max_scale, np.float64)
    X, info = solve_affine(s4, d4)
    k = info["kappa"]
    xmax = float(max(abs(X[j, c]) for j in range(4) for c in range(3)))
    dX = C_SOLVE * U * k * (2 * xmax + (k + 1) * info["resid"] / info["sigma_max"]) + 4 * U * xmax
    gates = {}
    out = {"info": info, "T": None, "bound": np.inf, "lo": None, "hi": None, "gates": gates}
    with mp.workdps(DPS):
        A = mp.matrix([[X[j, i] for j in range(3)] for i in range(3)])       # A[i][j] = X[j][i]
        t = [X[3, i] for i in range(3)]
        sc = column_scales(A)
        ds = 2.0 * dX + 4 * U * float(max(sc))
        for j in range(3):
            gates[f"min_scale{j}"] = (float(sc[j] - min_scale[j]), ds)
            gates[f"max_scale{j}"] = (float(max_scale[j] - sc[j]), ds)
        smin_sc = float(min(sc))
        if any(_decide(m, b) is False for m, b in gates.values()):
            pass                # decided invalid: the later gates cannot change that
        elif smin_sc > 4 * ds:
            R = mp.matrix([[A[i, j] / sc[j] for j in range(3)] for i in range(3)])
            dR = (dX + ds) / (smin_sc - ds)
            w, Vm = mp.eigsy(R.T * R)
            sv = [mp.sqrt(max(w[i], mp.mpf(0))) for i in range(3)]
            dsv = 3 * dR + 64 * U
            gates["sv_min"] = (float(min(sv) - SV_LO), dsv)
            gates["sv_max"] = (float(SV_HI - max(sv)), dsv)
            if float(min(sv)) > 4 * dsv and _decide(*gates["sv_min"]) is not False and _decide(*gates["sv_max"]) is not False:
                Q = Vm * mp.diag([1 / s for s in sv]) * Vm.T
                Ro = R * Q
                dRo = 3 * dR / (float(min(sv)) - dsv) + 64 * U
                gates["det"] = (float(polar_det(Ro)), 6 * dRo)
                T = np.eye(4)
                for i in range(3):
                    for j in range(3):
                        T[i, j] = float(Ro[i, j] * sc[j])
                    T[i, 3] = float(t[i])
                bound = max(dRo * float(max(sc)) + ds, dX) + 64 * U * max(1.0, float(max(sc)))
                out["T"], out["bound"] = T, bound
                if max_dims is not None:
                    Ti = canonical_inverse(Ro, sc, t)
                    tg = np.asarray(target, np.float64)
                    c = tg @ Ti[:, :3].T + Ti[:, 3]
                    ext = c.max(axis=0) - c.min(axis=0)
                    tmax = float(np.abs(tg).sum(axis=1).max())
                    dTi = (dRo + ds / smin_sc) / smin_sc
                    dext = 2 * (dTi * tmax + dTi * float(np.abs(T[:3, 3]).sum()) + np.abs(Ti[:, :3]).max() * 3 * dX) \
                        + 64 * U * (np.abs(Ti[:, :3]).sum(axis=1).max() * tmax + np.abs(Ti[:, 3]).max())
                    for j in range(3):
                        gates[f"dims{j}"] = (float(max_dims[j] - ext[j]), float(dext))
    decisions = [_decide(m, b) for m, b in gates.values()]
    if info["cut_undecided"]:
        decisions.append(None)
    if any(d is False for d in decisions):
        valid = False
    elif out["T"] is None or any(d is None for d in decisions):
        valid = None
    else:
        valid = True
    out["valid"] = valid
    if source is not None and out["T"] is not None:
        out["lo"], out["hi"] = inlier_interval(out["T"], out["bound"], source, target, thr)
    return out


def inlier_interval(T, bound, source, target, thr):
    """[lo, hi] of the kernel's inlier count for a transform within ``bound`` of T (see the module docstring)."""
    src = np.asarray(source, np.float64)
    tgt = np.asarray(target, np.float64)
    sh = np.c_[src, np.ones(len(src))]
    e = np.linalg.norm(sh @ T[:3].T - tgt, axis=1)
    l1 = np.abs(sh).sum(axis=1)
    slack = np.sqrt(3.0) * bound * l1 + 32 * U * (np.abs(sh) @ np.abs(T[:3]).T).max(axis=1) \
        + 32 * U * (np.abs(tgt).max(axis=1) + thr)
    lo = int(np.count_nonzero(e <= thr - slack))
    hi = int(np.count_nonzero(e <= thr + slack))
    return lo, hi


def evaluate(source, target, ids, thr, min_scale, max_scale, max_dims, stop_at_full=False):
    """All hypotheses of ``ids`` (H,4).  With stop_at_full, stops after the first decided-valid hypothesis whose
    count is decided at N (nothing later can beat it under the first-maximum rule)."""
    s, d = narrow(source, target, ids)
    N = len(source)
    res = []
    for h in range(len(s)):
        r = hypothesis(s[h], d[h], target, thr, min_scale, max_scale, max_dims, source=source)
        res.append(r)
        if stop_at_full and r["valid"] is True and r["lo"] == N:
            break
    return res


def replay_winner(res):
    """aligning.py:105-117 over the oracle's decisions: the first maximum of the inlier count among valid hypotheses.
    Returns the winning index, or None when no hypothesis is valid.  Raises if an undecided hypothesis (valid or
    count) could change the winner."""
    best, best_lo = None, -1
    for h, r in enumerate(res):
        if r["valid"] is True and r["lo"] == r["hi"] and r["lo"] > best_lo:
            best, best_lo = h, r["lo"]
    for h, r in enumerate(res):
        if r["valid"] is False or h == best:
            continue
        hi = r["hi"] if r["hi"] is not None else np.inf
        if r["valid"] is None or r["lo"] != r["hi"]:
            if hi > best_lo or (hi == best_lo and (best is None or h < best)):
                raise AssertionError(f"hypothesis {h} is undecided and could change the winner {best}")
    return best
