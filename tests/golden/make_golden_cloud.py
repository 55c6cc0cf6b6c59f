"""Golden vectors for the point-cloud preparation (catgrasp_b200/cloud.py), produced by EXECUTING THE REFERENCE's
Utils.depth2xyzmap (:239-251), Utils.cloudA_minus_cloudB (:482-488) and Utils.correct_pcd_normal_direction (:205-213),
and the two cKDTree.query lines of run_grasp_simulation.py::compute_candidate_grasp_one_ob as the reference writes
them (:119-121, the snap of the voxel means, and :130-133, the crop), with the real scipy cKDTree.

Run in the authoring container only (needs the reference checkout):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cloud.py

Input: a depth image rendered by synthetic.render_depth from a seeded pile at the reference K (config.yml:1-3)
scaled down by 6 (344 x 257 pixels) so that the fixture stays small, with pixels set to 0, just below 0.1 and
exactly float32(0.1).  The voxel means that the snap queries come from oracle/cloud_ref.py (open3d is absent).

Import-only stubs: open3d (see below), trimesh and transformations.  Two stand-ins:
- installed scipy has removed ``n_jobs`` from query_ball_point, so the cKDTree that Utils uses passes it on as
  ``workers``;
- ``open3d`` is a numpy point-cloud object with ``points`` / ``normals`` attributes and a Vector3dVector that copies
  to float64, which is all that correct_pcd_normal_direction reads and writes.
"""
import os
import sys
import types

import numpy as np
from scipy.spatial import cKDTree

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, "/root/reference")


class _Stub(types.ModuleType):
    __all__ = []
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


for _m in ["trimesh", "transformations"]:
    sys.modules[_m] = _Stub(_m)


class _PointCloud:
    def __init__(self):
        self.points = np.zeros((0, 3))
        self.normals = np.zeros((0, 3))


_o3d = types.ModuleType("open3d")
_o3d.geometry = types.SimpleNamespace(PointCloud=_PointCloud)
_o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64))
sys.modules["open3d"] = _o3d

import Utils as ref_utils   # noqa: E402  the reference itself


class _CKDTreeWorkers(cKDTree):
    def query_ball_point(self, x, r, n_jobs=1, **kw):
        return super().query_ball_point(x, r, workers=n_jobs, **kw)


ref_utils.cKDTree = _CKDTreeWorkers

from catgrasp_b200 import synthetic   # noqa: E402
from oracle import cloud_ref            # noqa: E402

K_FULL = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)
SCALE = 6
GRIPPER_DIAMETER = 0.05


def inputs():
    K = K_FULL.copy()
    K[:2] /= SCALE
    H, W = 1544 // SCALE, 2064 // SCALE
    depth, ids = synthetic.render_depth(K, H, W, n_objects=8, seed=21)
    rng = np.random.RandomState(22)
    flat = depth.reshape(-1)
    pick = rng.choice(flat.size, 300, replace=False)
    flat[pick[:100]] = 0.0
    flat[pick[100:200]] = np.float32(0.1)
    flat[pick[200:]] = np.nextafter(np.float32(0.1), np.float32(0))
    ids.reshape(-1)[pick] = -2
    return K, depth, ids


def main():
    K, depth, ids = inputs()
    xyz_map = ref_utils.depth2xyzmap(depth, K)
    scene_pts = xyz_map[xyz_map[:, :, 2] >= 0.1].reshape(-1, 3)           # run_grasp_simulation.py:199
    ob_id = int(np.bincount(ids[ids >= 0]).argmax())
    ob_pts = xyz_map[ids == ob_id].reshape(-1, 3)

    # :119-121 with the oracle's voxel means standing in for open3d's
    ob_pts_down, _ = cloud_ref.voxel_down_sample(ob_pts, 0.0005)
    kdtree = cKDTree(ob_pts)
    dists, indices = kdtree.query(ob_pts_down)
    snap_idx = indices
    # :130-133
    kdtree = cKDTree(ob_pts)
    dists, indices = kdtree.query(scene_pts)
    keep_ids = np.where(dists <= GRIPPER_DIAMETER / 2)[0]
    background_pts = scene_pts[keep_ids]
    # :135
    minus_pts, minus_ids = ref_utils.cloudA_minus_cloudB(background_pts, ob_pts, thres=0.005)

    # orientation of arbitrary normals, some zero, some perpendicular to the view ray
    rng = np.random.RandomState(23)
    orient_ids = np.sort(rng.choice(len(scene_pts), 6000, replace=False))
    pts = scene_pts[orient_ids].astype(np.float64)
    nrm = rng.normal(size=pts.shape)
    nrm[:50] = 0.0
    nrm[50:100] = np.cross(-pts[50:100], rng.normal(size=(50, 3)))
    pcd = _PointCloud()
    pcd.points = pts
    pcd.normals = nrm.copy()
    oriented = np.asarray(ref_utils.correct_pcd_normal_direction(pcd).normals)
    view_port = np.array([0.01, -0.02, 0.03])
    pcd.normals = nrm.copy()
    oriented_vp = np.asarray(ref_utils.correct_pcd_normal_direction(pcd, view_port=view_port).normals)

    np.savez_compressed(os.path.join(HERE, "cloud_prep.npz"), K=K, depth=depth, ids=ids, xyz_map=xyz_map, ob_id=ob_id,
                        gripper_diameter=GRIPPER_DIAMETER, ob_pts_down=ob_pts_down, snap_idx=snap_idx,
                        crop_keep_ids=keep_ids, minus_pts=minus_pts, minus_ids=minus_ids, orient_ids=orient_ids, normals_in=nrm,
                        oriented=oriented, view_port=view_port, oriented_vp=oriented_vp)
    print("cloud golden:", depth.shape, "scene", len(scene_pts), "object", len(ob_pts), "voxels", len(ob_pts_down),
          "crop", len(keep_ids), "minus", len(minus_ids), "minus ascending", bool((np.diff(minus_ids) > 0).all()))


if __name__ == "__main__":
    main()
