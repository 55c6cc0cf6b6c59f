"""Point-cloud preparation on the device (csrc/cg_cloud.cu): the open3d and scipy calls that feed the ported stages.

Each function replaces one reference call site and takes numpy arrays or CUDA tensors (numpy in, numpy out; see
_lib).  Points are float64 (scipy works in float64 and open3d stores Vector3d); float32 input is widened exactly.
Distances are float64 ``(dx*dx + dy*dy) + dz*dz``, bit-equal to scipy's cKDTree; a tie goes to the smaller point index.

Voxel outputs come in ascending (ix, iy, iz) voxel order.  open3d returns them in the iteration order of its hash
map, which is not reproducible, so callers must not depend on the order.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


def _offsets(off, n, what):
    """``off`` as an int32 numpy array of S + 1 >= 2 ascending offsets from 0 to n; ValueError otherwise."""
    o = np.asarray(off, dtype=np.int64).reshape(-1)
    if len(o) < 2 or o[0] != 0 or o[-1] != n or (np.diff(o) < 0).any():
        raise ValueError(f"{what}: need S + 1 >= 2 ascending offsets from 0 to {n}, got {o.tolist()}")
    return o.astype(np.int32)


class CloudIndex:
    """Points binned into cells of size ``cell`` (origin min_bound - cell/2) and sorted by (cell, index); built once
    and shared by every query on the same cloud and cell size.  Holds its own copy of the points.

    With ``set_offsets`` (S + 1 ints from 0 to the point count) the points are S sets laid end to end, set s the rows
    [set_offsets[s], set_offsets[s + 1]), each binned as a one-set index over it alone would bin it (its own origin);
    ``cell_offsets`` then gives each set's cells, ``voxel_means`` comes out set-major, and ``nearest_many`` and
    ``normals_many`` search each point's own set.  A set with no points raises ValueError; a batch whose cell keys need
    more than 63 bits raises CgError.  ``nearest``, ``within`` and ``normals`` need a one-set index."""

    def __init__(self, pts, cell, device=None, set_offsets=None):
        self.ctx, p = _lib.inputs(pts, dtype=torch.float64, ctx=None if device is None else _lib.Context.get(device))
        p = p.reshape(-1, 3)
        self.device = self.ctx.device
        if p.shape[0] == 0:
            raise ValueError("CloudIndex needs at least one point")
        h = C.c_void_p()
        if set_offsets is None:
            self.ctx.call("cg_cloud_index_create", self.ctx.h, p, p.shape[0], float(cell), C.byref(h))
        else:
            off = _offsets(set_offsets, p.shape[0], "CloudIndex")
            if (np.diff(off) < 1).any():
                raise ValueError(f"CloudIndex: every set needs at least one point, got offsets {off.tolist()}")
            self.ctx.call("cg_cloud_index_create_many", self.ctx.h, p, off, len(off) - 1, float(cell), C.byref(h))
        self.h = h
        n, u, S = C.c_int(), C.c_int(), C.c_int()
        self.ctx.call("cg_cloud_index_info", h, C.byref(n), C.byref(u), None, None)
        self.n_points, self.n_cells = n.value, u.value
        self.ctx.call("cg_cloud_index_sets", h, C.byref(S), None)
        self.n_sets = S.value
        coff = np.zeros(self.n_sets + 1, np.int32)
        self.ctx.call("cg_cloud_index_sets", h, None, coff)
        self.set_offsets = np.array([0, self.n_points]) if set_offsets is None else off.astype(np.int64)
        self.cell_offsets = coff.astype(np.int64)     # set s's cells (and voxel means): [cell_offsets[s], [s + 1])

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            self.ctx.call("cg_cloud_index_destroy", h)
            self.h = None

    def _query(self, query):
        return _lib.inputs(query, dtype=torch.float64, ctx=self.ctx)[1].reshape(-1, 3)

    def _empty(self, *shape, dtype=torch.float64):
        return torch.empty(shape, dtype=dtype, device=torch.device("cuda", self.device))

    def voxel_means(self, normals=None):
        """open3d VoxelDownSample with voxel_size = cell: (U,3) means (and (U,3) normals) as device tensors."""
        out = self._empty(self.n_cells, 3)
        nrm = None if normals is None else self._query(normals)
        out_n = None if normals is None else torch.empty_like(out)
        self.ctx.call("cg_voxel_down_sample_dev", self.h, nrm, out, out_n)
        return out, out_n

    def nearest(self, query, max_dist):
        q = self._query(query)
        idx = self._empty(q.shape[0], dtype=torch.int32)
        dist = self._empty(q.shape[0])
        self.ctx.call("cg_cloud_nearest_dev", self.h, q, q.shape[0], float(max_dist), idx, dist)
        return dist, idx

    def nearest_many(self, query, query_offsets, max_dist):
        """nearest per set: the queries [query_offsets[s], query_offsets[s + 1]) search set s only.  (dists (Q,)
        float64, indices (Q,) int32 into the whole index, -1 / inf where set s has no point within max_dist)."""
        q = self._query(query)
        off = _offsets(query_offsets, q.shape[0], "CloudIndex.nearest_many")
        if len(off) != self.n_sets + 1:
            raise ValueError(f"CloudIndex.nearest_many: {len(off) - 1} query ranges for {self.n_sets} sets")
        idx = self._empty(q.shape[0], dtype=torch.int32)
        dist = self._empty(q.shape[0])
        self.ctx.call("cg_cloud_nearest_many_dev", self.h, q, off, q.shape[0], float(max_dist), idx, dist)
        return dist, idx

    def within(self, query, r, compare_sqrt):
        """uint8 mask: some indexed point has d2 <= r*r (compare_sqrt False) or sqrt(d2) <= r (True)."""
        q = self._query(query)
        mask = self._empty(q.shape[0], dtype=torch.uint8)
        self.ctx.call("cg_cloud_radius_mask_dev", self.h, q, q.shape[0], float(r), int(bool(compare_sqrt)), mask)
        return mask

    def normals(self, radius, max_nn, view_port=(0.0, 0.0, 0.0), neighbours=False):
        """Oriented normals of the indexed points (N,3); with neighbours=True also the (N,max_nn) int32 neighbour
        lists in (d2, index) order, -1 padded, and their (N,) sizes."""
        out = self._empty(self.n_points, 3)
        nbr = self._empty(self.n_points, max_nn, dtype=torch.int32) if neighbours else None
        cnt = self._empty(self.n_points, dtype=torch.int32) if neighbours else None
        vp = np.ascontiguousarray(view_port, dtype=np.float64).reshape(3)
        self.ctx.call("cg_cloud_normals_dev", self.h, float(radius), int(max_nn), vp, out, nbr, cnt)
        return (out, nbr, cnt) if neighbours else out

    def normals_many(self, radius, max_nn, view_port=(0.0, 0.0, 0.0), neighbours=False):
        """normals per set, one view point for all: set s's rows are what ``normals`` gives on a one-set index of
        set s alone, bit for bit, whatever either index's cell; neighbour ids index the whole index (set s's first
        point added, -1 padding kept)."""
        out = self._empty(self.n_points, 3)
        nbr = self._empty(self.n_points, max_nn, dtype=torch.int32) if neighbours else None
        cnt = self._empty(self.n_points, dtype=torch.int32) if neighbours else None
        vp = np.ascontiguousarray(view_port, dtype=np.float64).reshape(3)
        self.ctx.call("cg_cloud_normals_many_dev", self.h, float(radius), int(max_nn), vp, out, nbr, cnt)
        return (out, nbr, cnt) if neighbours else out


def _query_cell(pts, r):
    """Cell size for an index queried at radius r: r itself, but no finer than 1/2^20 of the cloud's largest extent
    (an index holds fewer than 2^21 cells per axis)."""
    p = pts.reshape(-1, 3)
    if isinstance(p, torch.Tensor):
        span = float((p.amax(0) - p.amin(0)).max()) if p.shape[0] else 0.0
    else:
        span = float((p.max(0) - p.min(0)).max()) if p.shape[0] else 0.0
    return max(float(r), span / 2.0 ** 20, 1e-12)


def _query_cell_many(p, off, r):
    """The largest of the non-empty sets' _query_cell: every set of ``p`` (N,3), rows [off[s], off[s + 1]), then spans
    fewer than 2^21 cells per axis.  One read of the spans on a CUDA tensor, whatever the number of sets."""
    rows = [(a, b) for a, b in zip(off[:-1], off[1:]) if b > a]
    if isinstance(p, torch.Tensor):
        span = float(torch.stack([(p[a:b].amax(0) - p[a:b].amin(0)).max() for a, b in rows]).max())
    else:
        span = max(float((p[a:b].max(0) - p[a:b].min(0)).max()) for a, b in rows)
    return max(float(r), span / 2.0 ** 20, 1e-12)


def depth2xyzmap(depth, K, out=None):
    """Utils.py:239-251 (called at run_grasp_simulation.py:198): (H,W) depth, float32 or float64 -> (H,W,3) float32
    camera-frame points; pixels with depth < 0.1 are (0,0,0).  ``out``: a contiguous float32 CUDA tensor of H*W*3
    elements on the depth's device to write the points into (a frame's slice of a buffer shared by several frames),
    returned as it is."""
    d = depth if isinstance(depth, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(depth))
    ctx, d = _lib.inputs(d, dtype=d.dtype if d.dtype in (torch.float32, torch.float64) else torch.float64)
    H, W = d.shape[:2]
    if out is not None:
        if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == H * W * 3):
            raise ValueError(f"depth2xyzmap: out must be a contiguous float32 CUDA tensor of {H * W * 3} elements")
        ctx.call("cg_depth2xyz_dev", ctx.h, d, int(d.dtype == torch.float64), H, W,
                 np.ascontiguousarray(K, dtype=np.float64).reshape(9), out)
        return out
    out = torch.empty((H, W, 3), dtype=torch.float32, device=d.device)
    ctx.call("cg_depth2xyz_dev", ctx.h, d, int(d.dtype == torch.float64), H, W,
             np.ascontiguousarray(K, dtype=np.float64).reshape(9), out)
    return _lib.returned(depth, out)


def voxel_down_sample(pts, voxel_size, normals=None):
    """open3d ``PointCloud.voxel_down_sample(voxel_size)`` (run_grasp_simulation.py:97, :114, :137, :173, :246):
    voxel means (and normalised summed normals when ``normals`` is given), in ascending (ix, iy, iz) order."""
    if pts.shape[0] == 0:
        z = np.zeros((0, 3))
        z = torch.from_numpy(z).to(pts.device) if getattr(pts, "is_cuda", False) else z
        return z if normals is None else (z, z)
    p, nrm = CloudIndex(pts, voxel_size).voxel_means(normals)
    return _lib.returned(pts, p) if normals is None else _lib.returned(pts, p, nrm)


def nearest(ref_pts, query_pts, max_dist):
    """``cKDTree(ref_pts).query(query_pts)`` (run_grasp_simulation.py:120, :131) for answers within ``max_dist``:
    (dists (Q,) float64, indices (Q,) int64), -1 / inf where no point lies within max_dist (inclusive)."""
    d, i = CloudIndex(ref_pts, _query_cell(ref_pts, max_dist)).nearest(query_pts, max_dist)
    return _lib.returned(query_pts, d, i.to(torch.int64))


def cloudA_minus_cloudB(ptsA, ptsB, thres):
    """Utils.py:482-488 (called at run_grasp_simulation.py:135): the points of A with no point of B within ``thres``
    (``query_ball_point``: d2 <= thres*thres).  Returns (ptsA[keep_ids], keep_ids), keep_ids ascending int64."""
    like = isinstance(ptsA, torch.Tensor)
    nA = ptsA.shape[0]
    if nA == 0 or ptsB.shape[0] == 0:
        keep = torch.arange(nA, device="cuda") if like else np.arange(nA)
        return ptsA[keep], keep
    idx = CloudIndex(ptsB, _query_cell(ptsB, thres))
    mark = idx.within(ptsA, thres, compare_sqrt=False)
    keep = torch.nonzero(mark == 0).reshape(-1)
    if like:
        return ptsA[keep.to(ptsA.device)], keep
    keep = keep.cpu().numpy()
    return ptsA[keep], keep


def estimate_normals(pts, radius, max_nn, view_port=(0.0, 0.0, 0.0)):
    """open3d ``estimate_normals(KDTreeSearchParamHybrid(radius, max_nn))`` followed by Utils.py:205-213
    ``correct_pcd_normal_direction(pcd, view_port)`` (run_grasp_simulation.py:209-210, :247-248): (N,3) float64."""
    if pts.shape[0] == 0:
        z = np.zeros((0, 3))
        return torch.from_numpy(z).to(pts.device) if getattr(pts, "is_cuda", False) else z
    return _lib.returned(pts, CloudIndex(pts, _query_cell(pts, radius)).normals(radius, max_nn, view_port))


def estimate_normals_many(pts, set_offsets, radius, max_nn, view_port=(0.0, 0.0, 0.0)):
    """estimate_normals per set, in one index build: ``pts`` (N,3) holds S sets laid end to end, set s the rows
    [set_offsets[s], set_offsets[s + 1]) (S + 1 ascending offsets from 0 to N; a set may be empty).  Returns (N,3)
    float64, set s's rows equal to estimate_normals on set s alone, bit for bit.  Synchronises three times whatever S
    is (the cell size, the index build's two).  One view point serves every set."""
    off = _offsets(set_offsets, pts.shape[0], "estimate_normals_many").astype(np.int64)
    if pts.shape[0] == 0:
        z = np.zeros((0, 3))
        return torch.from_numpy(z).to(pts.device) if getattr(pts, "is_cuda", False) else z
    kept = np.concatenate([[0], np.cumsum(np.diff(off)[np.diff(off) > 0])])    # empty sets have no rows to index
    p = pts.reshape(-1, 3)
    cell = _query_cell_many(p, off, radius)
    return _lib.returned(pts, CloudIndex(p, cell, set_offsets=kept).normals_many(radius, max_nn, view_port))


def prepare_object(ob_pts, ob_normals, scene_pts, gripper_diameter, octo_resolution=0.001, K=None):
    """run_grasp_simulation.py:113-139 and :171-175 (compute_candidate_grasp_one_ob) in one call: numpy in, numpy out;
    CUDA tensors in, CUDA tensors out.

    Returns None when fewer than 100 voxels survive the 0.5 mm down-sampling (:116-118); otherwise a dict with
    ``data`` ({'cloud_xyz', 'cloud_normal'}: each voxel mean snapped to its nearest object point, duplicates kept,
    :119-126), ``background_pts`` (the occupancy samples of the scene around the object, :130-139),
    ``points_for_sample`` and ``normals_for_sample`` (:171-175).  ``K`` is handed to makeOccupancyGridFromCloudScan,
    which does not use it.  The object and scene points stay on the device either way; the occupancy grid is built
    by the host entry of makeOccupancyGridFromCloudScan."""
    from .my_cpp import makeOccupancyGridFromCloudScan
    like = ob_pts
    ob_pts, ob_normals, scene_pts = (a if isinstance(a, torch.Tensor) else np.asarray(a)
                                     for a in (ob_pts, ob_normals, scene_pts))
    ctx, ob_pts, ob_normals, scene_pts = _lib.inputs(
        ob_pts, ob_normals, scene_pts,
        dtype=tuple(torch.float32 if str(a.dtype).endswith("float32") else torch.float64
                    for a in (ob_pts, ob_normals, scene_pts)))
    ob_pts, ob_normals, scene_pts = ob_pts.reshape(-1, 3), ob_normals.reshape(-1, 3), scene_pts.reshape(-1, 3)
    dev = ctx.device
    ob_index = CloudIndex(ob_pts, 0.0005, dev)
    n_down = ob_index.n_cells                                                          # :113-115
    if n_down < 100:                                                                   # :116-118
        return None
    down, _ = ob_index.voxel_means()
    del ob_index
    # :119-122 snap: a voxel mean and its members share a voxel, so the nearest member is within the diagonal; the
    # bound is widened by 1e-9 relative so rounding at a voxel face cannot exclude it
    snap_bound = 0.0005 * np.sqrt(3.0) * (1 + 1e-9)
    _, ids = CloudIndex(ob_pts, snap_bound, dev).nearest(down, snap_bound)
    if bool((ids < 0).any()):
        raise _lib.CgError("prepare_object: a voxel mean has no object point within its voxel's diagonal")
    ids = ids.to(torch.int64)
    xyz, nrm = ob_pts[ids], ob_normals[ids]
    # :130-134 crop: scene points whose nearest object point is within gripper_diameter/2 (sqrt(d2) <= R)
    R = gripper_diameter / 2
    keep = torch.nonzero(CloudIndex(ob_pts, _query_cell(ob_pts, R), dev).within(scene_pts, R, compare_sqrt=True))
    background = scene_pts[keep.reshape(-1)]
    background, _ = cloudA_minus_cloudB(background, ob_pts, thres=0.005)               # :135
    if background.shape[0]:
        background = voxel_down_sample(background, 0.001).cpu().numpy()              # :136-137
        background_pts = makeOccupancyGridFromCloudScan(background, np.eye(3) if K is None else K, octo_resolution)
    else:
        background_pts = np.zeros((0, 3), np.float32)
    # :172, in the cloud's dtype (the extent is exact; the norm is numpy's)
    ext = (xyz.amax(0) - xyz.amin(0)).cpu().numpy()
    voxel_size = float(np.linalg.norm(ext) / 10.0)
    pfs, nfs = voxel_down_sample(xyz, voxel_size, normals=nrm)                         # :171-175
    background_pts = torch.from_numpy(background_pts).to(xyz.device)
    xyz, nrm, background_pts, pfs, nfs = _lib.returned(like, xyz, nrm, background_pts, pfs, nfs)
    return {"data": {"cloud_xyz": xyz, "cloud_normal": nrm}, "background_pts": background_pts,
            "points_for_sample": pfs, "normals_for_sample": nfs}
