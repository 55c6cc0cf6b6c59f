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


class CloudIndex:
    """Points binned into cells of size ``cell`` (origin min_bound - cell/2) and sorted by (cell, index); built once
    and shared by every query on the same cloud and cell size.  Holds its own copy of the points."""

    def __init__(self, pts, cell, device=None):
        self.ctx, p = _lib.inputs(pts, dtype=torch.float64, ctx=None if device is None else _lib.Context.get(device))
        p = p.reshape(-1, 3)
        self.device = self.ctx.device
        if p.shape[0] == 0:
            raise ValueError("CloudIndex needs at least one point")
        h = C.c_void_p()
        self.ctx.call("cg_cloud_index_create", self.ctx.h, p, p.shape[0], float(cell), C.byref(h))
        self.h = h
        n, u = C.c_int(), C.c_int()
        self.ctx.call("cg_cloud_index_info", h, C.byref(n), C.byref(u), None, None)
        self.n_points, self.n_cells = n.value, u.value

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


def _query_cell(pts, r):
    """Cell size for an index queried at radius r: r itself, but no finer than 1/2^20 of the cloud's largest extent
    (an index holds fewer than 2^21 cells per axis)."""
    p = pts.reshape(-1, 3)
    if isinstance(p, torch.Tensor):
        span = float((p.amax(0) - p.amin(0)).max()) if p.shape[0] else 0.0
    else:
        span = float((p.max(0) - p.min(0)).max()) if p.shape[0] else 0.0
    return max(float(r), span / 2.0 ** 20, 1e-12)


def depth2xyzmap(depth, K):
    """Utils.py:239-251 (called at run_grasp_simulation.py:198): (H,W) depth, float32 or float64 -> (H,W,3) float32
    camera-frame points; pixels with depth < 0.1 are (0,0,0)."""
    d = depth if isinstance(depth, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(depth))
    ctx, d = _lib.inputs(d, dtype=d.dtype if d.dtype in (torch.float32, torch.float64) else torch.float64)
    H, W = d.shape[:2]
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


def prepare_object(ob_pts, ob_normals, scene_pts, gripper_diameter, octo_resolution=0.001, K=None):
    """run_grasp_simulation.py:113-139 and :171-175 (compute_candidate_grasp_one_ob) in one call, numpy in and out.

    Returns None when fewer than 100 voxels survive the 0.5 mm down-sampling (:116-118); otherwise a dict with
    ``data`` ({'cloud_xyz', 'cloud_normal'}: each voxel mean snapped to its nearest object point, duplicates kept,
    :119-126), ``background_pts`` (the occupancy samples of the scene around the object, :130-139),
    ``points_for_sample`` and ``normals_for_sample`` (:171-175).  ``K`` is handed to makeOccupancyGridFromCloudScan,
    which does not use it."""
    from .my_cpp import makeOccupancyGridFromCloudScan
    ob_pts = np.asarray(ob_pts)
    ob_normals = np.asarray(ob_normals)
    scene_pts = np.asarray(scene_pts)
    ob_index = CloudIndex(ob_pts, 0.0005)
    down, _ = ob_index.voxel_means()                                                   # :113-115
    if down.shape[0] < 100:                                                            # :116-118
        return None
    del ob_index
    # :119-122 snap: a voxel mean and its members share a voxel, so the nearest member is within the diagonal; the
    # bound is widened by 1e-9 relative so rounding at a voxel face cannot exclude it
    snap_bound = 0.0005 * np.sqrt(3.0) * (1 + 1e-9)
    index = CloudIndex(ob_pts, snap_bound)
    _, ids = index.nearest(down, snap_bound)
    ids = ids.cpu().numpy().astype(np.int64)
    if (ids < 0).any():
        raise _lib.CgError("prepare_object: a voxel mean has no object point within its voxel's diagonal")
    data = {"cloud_xyz": ob_pts[ids].reshape(-1, 3), "cloud_normal": ob_normals[ids].reshape(-1, 3)}
    # :130-134 crop: scene points whose nearest object point is within gripper_diameter/2 (sqrt(d2) <= R)
    R = gripper_diameter / 2
    crop_index = CloudIndex(ob_pts, _query_cell(ob_pts, R))
    keep = torch.nonzero(crop_index.within(scene_pts, R, compare_sqrt=True)).reshape(-1).cpu().numpy()
    background = scene_pts[keep]
    background, _ = cloudA_minus_cloudB(background, ob_pts, thres=0.005)               # :135
    if background.shape[0]:
        background = voxel_down_sample(background, 0.001)                             # :136-137
        background_pts = makeOccupancyGridFromCloudScan(background, np.eye(3) if K is None else K, octo_resolution)
    else:
        background_pts = np.zeros((0, 3), np.float32)
    xyz = data["cloud_xyz"]
    voxel_size = float(np.linalg.norm(xyz.max(axis=0) - xyz.min(axis=0)) / 10.0)       # :172, in the cloud's dtype
    pfs, nfs = voxel_down_sample(xyz, voxel_size, normals=data["cloud_normal"])         # :171-175
    return {"data": data, "background_pts": background_pts, "points_for_sample": pfs, "normals_for_sample": nfs}
