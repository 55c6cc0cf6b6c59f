"""numpy restatement of catgrasp_b200/csrc/cg_meanshift.cu: sklearn's MeanShift(bandwidth, seeds=None,
bin_seeding=False, cluster_all=True) with the kernel's arithmetic, and the composition of PointGroupPredictor.predict
around it (predicter.py:308-338).

Neighbour sets are cKDTree candidates (radius widened by 1e-9 relative) filtered by the exact rule
d2 = (dx*dx + dy*dy) + dz*dz <= bw*bw in float64, each operation a separate ufunc.  Sums are int64 fixed point:
q = rint(ldexp(p - origin, 41 - E)), origin = min_bound - bw/2, E = ceil(log2(max(p - origin) + bw)), and the mean
is dtype(ldexp(sum) / n + origin) in X's dtype.  The post-processing is sklearn's own (_mean_shift.py, fit): a dict of
centres keyed by value, sorted by (count, centre) descending, greedy suppression within bw, nearest kept centre with
ties to the smaller index.
"""
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
