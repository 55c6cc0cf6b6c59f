"""numpy restatement of catgrasp_b200/csrc/cg_meanshift.cu: sklearn's MeanShift(bandwidth, seeds=None,
bin_seeding=False, cluster_all=True) with the kernel's arithmetic, and the composition of PointGroupPredictor.predict
around it (predicter.py:308-338).

Neighbour sets are cKDTree candidates (radius widened by 1e-9 relative) filtered by the exact rule
d2 = (dx*dx + dy*dy) + dz*dz <= bw*bw in float64, each operation a separate ufunc.  Sums are int64 fixed point:
q = rint(ldexp(p - origin, 41 - E)), origin = min_bound - bw/2, E = ceil(log2(max(p - origin) + bw)), and the mean
is dtype(ldexp(sum) / n + origin) in X's dtype.  The post-processing is sklearn's own (_mean_shift.py, fit): a dict of
centres keyed by value, sorted by (count, centre) descending, greedy suppression within bw, nearest kept centre with
ties to the smaller index.

step_bruteforce and modes_bruteforce restate one ascent step and the post-processing with no tree at all: every
(centre, point) and every (mode, mode) pair is compared.  They pin the tree-based ascent / modes above, and they let a
test feed the kernel's own intermediate results (a run stopped at max_iter k, the kernel's seed centres) through one
more step or through the post-processing.
"""
import math

import numpy as np
from scipy.spatial import cKDTree

QBITS = 41
SLACK = 1 + 1e-9


def _ceil_log2(v):
    f, e = np.frexp(v)
    return int(e - 1 if f == 0.5 else e)


def quantise(X64, bw):
    """(origin, E, q): the fixed-point image of the points."""
    origin = X64.min(axis=0) - bw * 0.5
    u = X64 - origin
    E = _ceil_log2(float(u.max()) + bw)
    return origin, E, np.rint(np.ldexp(u, QBITS - E)).astype(np.int64)


def _d2(a, b):
    dx = a[:, 0] - b[:, 0]
    dy = a[:, 1] - b[:, 1]
    dz = a[:, 2] - b[:, 2]
    return (dx * dx + dy * dy) + dz * dz


def _balls(tree, pts, queries, r, chunk=1 << 16):
    """Yields (rows, cols, d2) for every (query, point) pair with d2 <= r*r, per chunk of queries; r may be per query."""
    r = np.broadcast_to(np.asarray(r, np.float64), (len(queries),))
    for s in range(0, len(queries), chunk):
        q = queries[s:s + chunk]
        lists = tree.query_ball_point(q, r[s:s + chunk] * SLACK, workers=-1)
        lens = np.fromiter((len(x) for x in lists), np.int64, len(lists))
        rows = np.repeat(np.arange(len(q)), lens)
        cols = np.concatenate([np.asarray(x, np.int64) for x in lists]) if len(rows) else np.zeros(0, np.int64)
        d2 = _d2(q[rows], pts[cols])
        keep = d2 <= r[s:s + chunk][rows] * r[s:s + chunk][rows]
        yield s + rows[keep], cols[keep], d2[keep]


def nearest(ref, query):
    """Index of the nearest ref point for every query (float64 d2, ties to the smaller index)."""
    ref = np.asarray(ref, np.float64)
    query = np.asarray(query, np.float64)
    tree = cKDTree(ref)
    dk, _ = tree.query(query, k=1)
    out = np.empty(len(query), np.int64)
    for rows, cols, d2 in _balls(tree, ref, query, dk * SLACK):      # a superset of the exact minimum's ties
        o = np.lexsort((cols, d2, rows))
        first = np.ones(len(o), bool)
        first[1:] = rows[o][1:] != rows[o][:-1]
        out[rows[o][first]] = cols[o][first]
    return out


def ascent(X, bw, max_iter=300):
    """Per seed (every row of X): (centre in X's dtype, final set size, completed steps)."""
    X = np.asarray(X)
    T = X.dtype.type
    X64 = X.astype(np.float64)
    origin, E, q = quantise(X64, bw)
    unscale = np.ldexp(1.0, E - QBITS)
    stop = 1e-3 * bw
    tree = cKDTree(X64)
    P = len(X)
    m = X.copy()
    n = np.zeros(P, np.int64)
    it = np.zeros(P, np.int64)
    active = np.arange(P)
    while active.size:
        cnt = np.zeros(len(active), np.int64)
        sums = np.zeros((len(active), 3), np.int64)
        for rows, cols, _ in _balls(tree, X64, m[active].astype(np.float64), bw):
            cnt += np.bincount(rows, minlength=len(active))
            np.add.at(sums, rows, q[cols])
        n[active] = cnt
        full = cnt > 0
        new = m[active].copy()
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = (sums.astype(np.float64) * unscale) / cnt[:, None].astype(np.float64) + origin
        new[full] = mean[full].astype(T)
        d = (new - m[active]).astype(np.float64)
        step = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        m[active] = new
        done = ~full | (step <= stop) | (it[active] == max_iter)
        it[active[~done]] += 1
        active = active[~done]
    return m, n, it


def modes(centres, counts, bw):
    """sklearn's post-processing up to the kept centres (in X's dtype, (count, x, y, z) descending)."""
    T = centres.dtype.type
    d = {}
    for c, k in zip(centres, counts):
        if k:
            d[tuple(c)] = int(k)              # equal by value (-0.0 == 0.0): first key, last count
    srt = sorted(d.items(), key=lambda t: (t[1], t[0]), reverse=True)
    sc = np.array([t[0] for t in srt], T).reshape(-1, 3)
    sc64 = sc.astype(np.float64)
    nbr = [[] for _ in range(len(sc))]
    for rows, cols, _ in _balls(cKDTree(sc64), sc64, sc64, bw):
        sel = cols > rows                     # earlier modes are already decided
        for r, c in zip(rows[sel].tolist(), cols[sel].tolist()):
            nbr[r].append(c)
    unique = np.ones(len(sc), bool)
    for i in range(len(sc)):
        if unique[i]:
            unique[nbr[i]] = False
    return sc[unique]


def frame(X, bw):
    """(origin, E) of the kernel's fixed point (cg_meanshift.cu's header): origin = min_bound - bw/2 per axis, the
    origin of the cell index over X, and E the smallest integer with 2^E >= max(p - origin) + bw."""
    X64 = np.asarray(X, np.float64)
    origin = X64.min(axis=0) - bw * 0.5
    umax = max(float(X64[:, a].max()) - float(origin[a]) for a in range(3))
    m, e = math.frexp(umax + bw)
    return origin, e - 1 if m == 0.5 else e


def step_bruteforce(X, bw, M, chunk=1 << 22):
    """One ascent step from every centre of M (rows in X's dtype) over all points of X, pair by pair:
    (new centre in X's dtype, set size, the set's mean in float64 as sklearn defines it).

    Membership is d2 = (dx*dx + dy*dy) + dz*dz <= bw*bw, each operation rounded on its own; the new centre is
    dtype(float(sum q) * 2^(E-41) / n + origin) with q the int64 fixed-point image of each point.  The mean is summed
    in extended precision, so it is within an ulp of the exact mean of the set.  A centre with an empty set keeps its
    value, count 0 and a NaN mean.  Works through chunks of about `chunk` pairs."""
    X = np.asarray(X)
    T = X.dtype.type
    X64 = X.astype(np.float64)
    M = np.asarray(M, T).reshape(-1, 3)
    M64 = M.astype(np.float64)
    origin, E = frame(X64, bw)
    q = np.rint((X64 - origin) * math.ldexp(1.0, QBITS - E)).astype(np.int64)
    bw2 = bw * bw
    new = M.copy()
    n = np.zeros(len(M), np.int64)
    mean = np.full((len(M), 3), np.nan)
    rows = max(1, chunk // len(X))
    for s in range(0, len(M), rows):
        m = M64[s:s + rows]
        dx = m[:, None, 0] - X64[None, :, 0]
        dy = m[:, None, 1] - X64[None, :, 1]
        dz = m[:, None, 2] - X64[None, :, 2]
        r, c = np.nonzero((dx * dx + dy * dy) + dz * dz <= bw2)
        if not len(r):
            continue
        cnt = np.bincount(r, minlength=len(m))
        full = np.flatnonzero(cnt)
        starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])[full]
        sums = np.add.reduceat(q[c], starts, axis=0)                           # int64: below 2^62 for P <= 2^21
        ext = np.add.reduceat(X64[c].astype(np.longdouble), starts, axis=0)
        n[s + full] = cnt[full]
        mean[s + full] = (ext / cnt[full, None].astype(np.longdouble)).astype(np.float64)
        for i, k in enumerate(full.tolist()):
            for a in range(3):
                v = float(int(sums[i, a])) * math.ldexp(1.0, E - QBITS) / float(cnt[k]) + float(origin[a])
                new[s + k, a] = T(v)
    return new, n, mean


def bound_ratio(centre, mean, E):
    """|centre - mean| over its bound, per entry, for a centre from the fixed-point step and its set's mean (NaN rows,
    empty sets, give 0).  Each q is within half a quantum 2^(E-41) of fl(p - origin), itself within 2^(E-53) of
    p - origin; the int64 -> double conversion and the division add 2^(E-53) each; adding the origin rounds by half
    an ulp of the centre in float64, narrowing by half an ulp in the centre's dtype; the mean is good to an ulp."""
    c = np.asarray(centre)
    c64 = c.astype(np.float64)
    bound = (0.5 * math.ldexp(1.0, E - QBITS) + 3 * math.ldexp(1.0, E - 53) + np.spacing(np.abs(c64)) / 2
             + np.spacing(np.abs(c)).astype(np.float64) / 2 + np.spacing(np.abs(np.nan_to_num(mean))))
    return np.nan_to_num(np.abs(c64 - mean) / bound)


def modes_bruteforce(seed_centres, seed_counts, bw):
    """sklearn's post-processing with no tree: seeds with a non-empty set in a dict keyed by centre value (-0.0 ==
    0.0; the first key, the last count), sorted by (count, x, y, z) descending, then greedy suppression in that order
    over all later pairs with d2 = (dx*dx + dy*dy) + dz*dz <= bw*bw.  The kept centres in the seeds' dtype."""
    c = np.asarray(seed_centres)
    T = c.dtype.type
    d = {}
    for key, k in zip(c.astype(np.float64).tolist(), np.asarray(seed_counts).tolist()):
        if k:
            d[tuple(key)] = k
    ranked = sorted(d.items(), key=lambda t: (t[1], t[0][0], t[0][1], t[0][2]), reverse=True)
    sc = np.array([t[0] for t in ranked], np.float64).reshape(-1, 3)
    keep = np.ones(len(sc), bool)
    bw2 = bw * bw
    for i in range(len(sc)):
        if keep[i]:
            dx = sc[i, 0] - sc[i + 1:, 0]
            dy = sc[i, 1] - sc[i + 1:, 1]
            dz = sc[i, 2] - sc[i + 1:, 2]
            keep[i + 1:] &= ~((dx * dx + dy * dy) + dz * dz <= bw2)
    return sc[keep].astype(T)


def fit(X, bw, max_iter=300):
    """dict(seed_centres, seed_counts, seed_iters, centres, labels, n_iter) as the kernel computes them."""
    X = np.asarray(X)
    if X.dtype not in (np.float32, np.float64):
        X = X.astype(np.float64)
    c, n, it = ascent(X, bw, max_iter)
    kept = modes(c, n, bw)
    labels = nearest(kept, X)
    return {"seed_centres": c, "seed_counts": n, "seed_iters": it, "centres": kept, "labels": labels,
            "n_iter": int(it.max())}


def pointgroup_labels(xyz_original_all, pt_offsets, cloud_xyz, bandwidth):
    """predicter.py:308-338 on arrays: (labels_all int64, xyz_shifted float32)."""
    from oracle import cloud_ref
    xo = np.asarray(xyz_original_all, np.float32)
    off = np.asarray(pt_offsets, np.float32)
    down, _ = cloud_ref.voxel_down_sample(xo, 0.002)
    ids = nearest(xo, down)
    xyz_down = xo[ids]
    xyz_shifted = xyz_down + off[ids]
    labels = fit(xyz_shifted, bandwidth)["labels"]
    return labels[nearest(xyz_down, cloud_xyz)], xyz_shifted
