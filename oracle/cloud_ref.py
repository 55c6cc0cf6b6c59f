"""numpy float64 restatement of the point-cloud preparation contracts (catgrasp_b200/csrc/cg_cloud.cu).

Distances: d2 = (dx*dx + dy*dy) + dz*dz, each operation a separate numpy ufunc (so rounded like scipy's
sqeuclidean_distance_double, without FMA).  Neighbour sets are brute force.  Voxel sums are sequential in ascending
point index: vectorised over voxels, looped over the rank within a voxel.  Normals come from numpy.linalg.eigh, with
an error bound from the eigengap; a normal whose bound exceeds NORMAL_DECIDED is undecided.
"""
import numpy as np

U = 2.0 ** -53
NORMAL_BOUND_C = 64.0       # c in c * u * ||C|| / (lambda_2 - lambda_1)
NORMAL_DECIDED = 1e-6       # radians: larger bounds leave the normal undecided


def _d2(q, p):
    """(Q,P) d2 between every query and every point, scipy's operation order."""
    dx = q[:, None, 0] - p[None, :, 0]
    dy = q[:, None, 1] - p[None, :, 1]
    dz = q[:, None, 2] - p[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def _chunks(Q, P, budget=1 << 22):
    step = max(1, budget // max(P, 1))
    for s in range(0, Q, step):
        yield s, min(Q, s + step)


def depth2xyzmap(depth, K):
    """Utils.py:239-251: float64 (u - cx) * z / fx left to right, narrowed to float32; depth < 0.1 -> 0 (compared in
    the depth's own dtype, as numpy compares an array with a Python float)."""
    K = np.asarray(K, np.float64)
    H, W = depth.shape[:2]
    vs, us = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    z = depth.reshape(-1).astype(np.float64)
    xs = (us.reshape(-1) - K[0, 2]) * z / K[0, 0]
    ys = (vs.reshape(-1) - K[1, 2]) * z / K[1, 1]
    out = np.stack([xs, ys, z], 1).reshape(H, W, 3).astype(np.float32)
    out[depth < depth.dtype.type(0.1)] = 0
    return out


def voxel_cells(pts, voxel):
    """Cell of every point: floor((p - (min_bound - voxel*0.5)) / voxel)."""
    pts = np.asarray(pts, np.float64)
    origin = pts.min(axis=0) - voxel * 0.5
    return np.floor((pts - origin) / voxel).astype(np.int64)


def voxel_down_sample(pts, voxel, normals=None):
    """Voxel means (and normalised normal sums) in ascending (ix, iy, iz) order; also returns each point's voxel."""
    pts = np.asarray(pts, np.float64)
    c = voxel_cells(pts, voxel)
    order = np.lexsort((np.arange(len(pts)), c[:, 2], c[:, 1], c[:, 0]))
    cs = c[order]
    head = np.ones(len(pts), bool)
    head[1:] = (cs[1:] != cs[:-1]).any(axis=1)
    vid_sorted = np.cumsum(head) - 1
    V = int(vid_sorted[-1]) + 1
    starts = np.nonzero(head)[0]
    counts = np.diff(np.append(starts, len(pts)))
    rank = np.arange(len(pts)) - starts[vid_sorted]
    sums = np.zeros((V, 3))
    nsum = np.zeros((V, 3))
    for r in range(int(counts.max())):
        sel = rank == r
        sums[vid_sorted[sel]] = sums[vid_sorted[sel]] + pts[order[sel]]
        if normals is not None:
            nsum[vid_sorted[sel]] = nsum[vid_sorted[sel]] + np.asarray(normals, np.float64)[order[sel]]
    means = sums / counts[:, None].astype(np.float64)
    voxel_of = np.empty(len(pts), np.int64)
    voxel_of[order] = vid_sorted
    if normals is None:
        return means, voxel_of
    q = (nsum[:, 0] * nsum[:, 0] + nsum[:, 1] * nsum[:, 1]) + nsum[:, 2] * nsum[:, 2]
    n = np.sqrt(q)
    nz = q > 0
    nsum[nz] = nsum[nz] / n[nz, None]
    return means, nsum, voxel_of


def nearest(ref, query, max_dist):
    """Brute-force cKDTree.query within max_dist: (dists, idx), first minimum (smallest index) on a tie, -1 / inf
    where sqrt(d2) > max_dist."""
    ref = np.asarray(ref, np.float64)
    query = np.asarray(query, np.float64)
    idx = np.full(len(query), -1, np.int64)
    dist = np.full(len(query), np.inf)
    for s, e in _chunks(len(query), len(ref)):
        d2 = _d2(query[s:e], ref)
        i = np.argmin(d2, axis=1)
        d = np.sqrt(d2[np.arange(e - s), i])
        ok = d <= max_dist
        idx[s:e] = np.where(ok, i, -1)
        dist[s:e] = np.where(ok, d, np.inf)
    return dist, idx


def within(ref, query, r, compare_sqrt):
    """True where some ref point has d2 <= r*r (query_ball_point) or sqrt(d2) <= r (the crop's dists <= R)."""
    ref = np.asarray(ref, np.float64)
    query = np.asarray(query, np.float64)
    out = np.zeros(len(query), bool)
    if len(ref) == 0:
        return out
    # queries farther than r (1 + 1e-9) from ref's bounding box on some axis cannot be within r in either form
    slack = r * (1 + 1e-9)
    near = np.nonzero(((query >= ref.min(0) - slack) & (query <= ref.max(0) + slack)).all(axis=1))[0]
    qn = query[near]
    for s, e in _chunks(len(qn), len(ref)):
        d2 = _d2(qn[s:e], ref)
        out[near[s:e]] = (np.sqrt(d2) <= r).any(axis=1) if compare_sqrt else (d2 <= r * r).any(axis=1)
    return out


def cloudA_minus_cloudB(ptsA, ptsB, thres):
    keep = np.nonzero(~within(ptsB, ptsA, thres, compare_sqrt=False))[0]
    return ptsA[keep], keep


def neighbours(pts, radius, max_nn):
    """(N, max_nn) int64 neighbour lists (-1 padded) and sizes: the max_nn smallest (d2, index) with d2 <= r*r."""
    pts = np.asarray(pts, np.float64)
    N = len(pts)
    nbr = np.full((N, max_nn), -1, np.int64)
    cnt = np.zeros(N, np.int64)
    r2 = radius * radius
    for s, e in _chunks(N, N):
        d2 = _d2(pts[s:e], pts)
        for i in range(e - s):
            cand = np.nonzero(d2[i] <= r2)[0]
            o = np.lexsort((cand, d2[i, cand]))[:max_nn]
            nbr[s + i, :len(o)] = cand[o]
            cnt[s + i] = len(o)
    return nbr, cnt


def covariances(pts, nbr, cnt):
    """Two-pass float64 covariance about the mean, neighbours summed in list order, divided by the count."""
    pts = np.asarray(pts, np.float64)
    N, M = nbr.shape
    n = np.maximum(cnt, 1).astype(np.float64)
    s = np.zeros((N, 3))
    for t in range(M):
        a = t < cnt
        s[a] = s[a] + pts[nbr[a, t]]
    mean = s / n[:, None]
    c = np.zeros((N, 6))            # xx xy xz yy yz zz
    pairs = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    for t in range(M):
        a = t < cnt
        d = pts[nbr[a, t]] - mean[a]
        for k, (i, j) in enumerate(pairs):
            c[a, k] = c[a, k] + d[:, i] * d[:, j]
    c = c / n[:, None]
    C = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)
    return C


def orient(pts, normals, view_port=(0.0, 0.0, 0.0)):
    """Utils.py:205-213 correct_pcd_normal_direction on arrays."""
    view_dir = np.asarray(view_port, np.float64).reshape(-1, 3) - np.asarray(pts, np.float64)
    view_dir = view_dir / np.linalg.norm(view_dir, axis=1).reshape(-1, 1)
    normals = np.asarray(normals, np.float64) / (np.linalg.norm(np.asarray(normals, np.float64), axis=1) + 1e-10).reshape(-1, 1)
    dots = (view_dir * normals).sum(axis=1)
    indices = np.where(dots < 0)
    normals[indices, :] = -normals[indices, :]
    return normals


def estimate_normals(pts, radius, max_nn, view_port=(0.0, 0.0, 0.0)):
    """Returns (oriented normals (N,3), bound (N,) radians, neighbour lists, sizes).  Normals with fewer than 3
    neighbours or a zero covariance are (0,0,1) before orientation, with bound 0; elsewhere the bound is
    NORMAL_BOUND_C * u * ||C||_2 / (lambda_2 - lambda_1) (inf for a zero gap)."""
    pts = np.asarray(pts, np.float64)
    nbr, cnt = neighbours(pts, radius, max_nn)
    C = covariances(pts, nbr, cnt)
    w, v = np.linalg.eigh(C)
    n = v[:, :, 0].copy()
    gap = w[:, 1] - w[:, 0]
    norm = np.abs(w).max(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        bound = np.where(gap > 0, NORMAL_BOUND_C * U * norm / gap, np.inf)
    fixed = (cnt < 3) | (C.reshape(-1, 9) == 0).all(axis=1)
    n[fixed] = [0.0, 0.0, 1.0]
    bound[fixed] = 0.0
    return orient(pts, n, view_port), bound, nbr, cnt


def prepare_object(ob_pts, ob_normals, scene_pts, gripper_diameter):
    """run_grasp_simulation.py:113-138, :171-175 up to the occupancy call: returns None below 100 voxels, else
    (data, occupancy input (voxel-down-sampled background), points_for_sample, normals_for_sample)."""
    ob64 = np.asarray(ob_pts, np.float64)
    down, _ = voxel_down_sample(ob64, 0.0005)
    if len(down) < 100:
        return None
    _, ids = nearest(ob64, down, np.inf)
    data = {"cloud_xyz": ob_pts[ids].reshape(-1, 3), "cloud_normal": ob_normals[ids].reshape(-1, 3)}
    keep = np.nonzero(within(ob64, scene_pts, gripper_diameter / 2, compare_sqrt=True))[0]
    background = scene_pts[keep]
    background, _ = cloudA_minus_cloudB(background, ob64, 0.005)
    occ_in = voxel_down_sample(background, 0.001)[0] if len(background) else np.zeros((0, 3))
    xyz = data["cloud_xyz"]
    voxel_size = float(np.linalg.norm(xyz.max(axis=0) - xyz.min(axis=0)) / 10.0)
    pfs, nfs, _ = voxel_down_sample(xyz, voxel_size, normals=data["cloud_normal"])
    return data, occ_in, pfs, nfs
