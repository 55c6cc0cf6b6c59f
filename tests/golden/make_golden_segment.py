"""Golden vectors for the segmentation's clustering, produced by EXECUTING THE REFERENCE's own
PointGroupPredictor.predict (predicter.py:232-338) with the real sklearn MeanShift and scipy cKDTree.

Run in the authoring container only (needs the reference checkout at /root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_segment.py

The sparse-conv network is out of scope, so the parts around it are stand-ins: spconv and pointgroup_ops are stub
modules (voxelization_idx returns placeholders the fake model ignores), the model returns fixed float32 offsets
(each point pulled toward its object's centre, plus seeded noise), Tensor.cuda is the identity, and open3d is a stub
whose PointCloud.voxel_down_sample is oracle.cloud_ref.voxel_down_sample.  Everything from the network's output to
the labels (:305-338) is the reference's code, unmodified.

The pile is thinned so that no two points lie within a 2 mm voxel's diagonal (see run()).

segment.npz holds, per class (prefix hnm_, nut_, screw_): cloud_xyz (the predict input, float32), xyz_original_all
and pt_offsets (what the network saw and returned), labels_all and xyz_shifted (the reference's results).
"""
import os
import sys
import types

import numpy as np
import torch

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, "/root/reference")

from oracle import cloud_ref                 # noqa: E402
from catgrasp_b200 import synthetic          # noqa: E402


class _Any:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Any()

    def __getattr__(self, n):
        return _Any()


class _Stub(types.ModuleType):
    __all__ = []
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        full = self.__name__ + "." + name
        if full in sys.modules:
            return sys.modules[full]
        return type(name, (_Any,), {})


_ABSENT = ["open3d", "trimesh", "transformations", "autolab_core", "spconv", "spconv.modules", "matplotlib",
           "matplotlib.pyplot", "pybullet",
           "dexnet", "dexnet.grasping", "dexnet.grasping.grasp", "dexnet.grasping.gripper",
           "dexnet.grasping.grasp_sampler",
           "PointGroup", "PointGroup.data", "PointGroup.data.dataset_seg", "PointGroup.model",
           "PointGroup.model.pointgroup", "PointGroup.model.pointgroup.pointgroup", "PointGroup.lib",
           "PointGroup.lib.pointgroup_ops", "PointGroup.lib.pointgroup_ops.functions",
           "PointGroup.lib.pointgroup_ops.functions.pointgroup_ops", "PointGroup.util", "PointGroup.util.config"]
for _m in _ABSENT:
    sys.modules[_m] = _Stub(_m)
torch.Tensor.cuda = lambda self, *a, **k: self


class _PointCloud:
    """open3d.geometry.PointCloud with the one method predict uses, voxel_down_sample = the oracle's."""

    def __init__(self):
        self.points = np.zeros((0, 3))

    def voxel_down_sample(self, voxel_size):
        out = _PointCloud()
        out.points = cloud_ref.voxel_down_sample(np.asarray(self.points, np.float64), voxel_size)[0]
        return out


o3d = sys.modules["open3d"]
o3d.geometry = types.SimpleNamespace(PointCloud=_PointCloud)
o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64).copy())
pg_ops = sys.modules["PointGroup.lib.pointgroup_ops.functions.pointgroup_ops"]
pg_ops.voxelization_idx = lambda locs, *a: (locs, torch.zeros(1), torch.zeros(1))
pg_ops.voxelization = lambda feats, *a: feats

import predicter as ref_predicter            # noqa: E402  the reference itself

THIN = 0.002 * np.sqrt(3.0) * 1.01


class _FakeModel:
    """Returns fixed float32 offsets: each point pulled `pull` of the way to its object's centre, plus noise that
    depends on the point's coordinates alone."""

    prepare_epochs = 1

    def __init__(self, scene_xyz, centre_of, pull, noise, seed):
        from scipy.spatial import cKDTree
        self.tree, self.centre_of, self.pull, self.noise, self.seed = cKDTree(scene_xyz), centre_of, pull, noise, seed
        self.seen = None

    def __call__(self, input_, p2v_map, coords_float, *a, **k):
        x = coords_float.numpy().astype(np.float64)
        _, i = self.tree.query(x)
        # repeated points (the first snap keeps duplicates) get one offset, so the snap's choice among them is moot
        _, first, inv = np.unique(x, axis=0, return_index=True, return_inverse=True)
        noise = np.random.RandomState(self.seed).normal(0, self.noise, (len(first), 3))[inv.reshape(-1)]
        off = (self.pull * (self.centre_of[i] - x) + noise).astype(np.float32)
        self.seen = (coords_float.numpy().copy(), off)
        return {"pt_offsets": torch.from_numpy(off)}


def thin(xyz, spacing):
    """Greedy subset with no two points within `spacing` (ascending index order)."""
    from scipy.spatial import cKDTree
    nbrs = cKDTree(xyz).query_ball_point(xyz, spacing)
    keep = np.ones(len(xyz), bool)
    for i in range(len(xyz)):
        if keep[i]:
            keep[[j for j in nbrs[i] if j > i]] = False
    return np.nonzero(keep)[0]


def run(class_name, n_points, n_objects, seed, pull, noise):
    scene = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    # no two points share a 2 mm voxel, so no voxel mean is equidistant from two points: cKDTree answers a tie with
    # whichever point its traversal meets, which no other implementation can reproduce
    sel = thin(scene["cloud_xyz"], THIN)
    xyz = scene["cloud_xyz"][sel].astype(np.float32)
    centre_of = scene["object_poses"][:, :3, 3][scene["object_id"][sel]]
    p = ref_predicter.PointGroupPredictor.__new__(ref_predicter.PointGroupPredictor)
    p.class_name = class_name
    p.n_slice_per_side = 1
    p.cfg = {"downsample_size": 0.0005}                                   # config_pointgroup.yaml:13
    p.cfg_pg = types.SimpleNamespace(use_coords=True, mode=4, batch_size=1)
    p.dataset = types.SimpleNamespace(scale=500, full_scale=[128, 999999], mode=4)
    p.model = _FakeModel(xyz.astype(np.float64), centre_of, pull, noise, seed + 100)
    data = {"cloud_xyz": xyz.copy(), "cloud_normal": scene["cloud_normal"][sel].astype(np.float32),
            "cloud_rgb": np.zeros_like(xyz, dtype=np.uint8)}
    labels_all = p.predict(data)
    xo, off = p.model.seen
    return {"cloud_xyz": xyz, "xyz_original_all": xo, "pt_offsets": off,
            "labels_all": np.asarray(labels_all, np.int64), "xyz_shifted": np.asarray(p.xyz_shifted, np.float32)}


def main():
    out = {}
    for class_name, n, k, seed, pull, noise in (("hnm", 30000, 16, 41, 0.85, 0.0008),
                                                ("nut", 40000, 24, 42, 0.6, 0.001),
                                                ("screw", 30000, 16, 43, 0.3, 0.001)):
        r = run(class_name, n, k, seed, pull, noise)
        for key, v in r.items():
            out[f"{class_name}_{key}"] = v
        print(class_name, "points", len(r["cloud_xyz"]), "shifted", len(r["xyz_shifted"]), "clusters",
              len(np.unique(r["labels_all"])))
    np.savez_compressed(os.path.join(HERE, "segment.npz"), **out)


if __name__ == "__main__":
    main()
