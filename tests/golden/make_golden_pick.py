"""Golden vectors for the control flow of the per-pick call (catgrasp_b200/pick.py), produced by EXECUTING THE
REFERENCE's own run_grasp_simulation.py::compute_candidate_grasp (:188-329) with its collaborators replaced:

- ``seg_predicter.predict`` returns fixed labels, one per no-background point;
- ``compute_candidate_grasp_one_ob`` records the seg id, ``ob_pts`` and ``scene_pts`` it receives and the numpy
  generator's state, and returns fixed grasps with fixed ``p_T_given_G`` (none for some objects);
- ``grasp_predicter.predict_batch`` returns fixed probabilities: softmax rows of logits drawn from N(0, 30^2), where
  numpy's pairwise sum and a left-to-right sum disagree, with exact ties and zeros of both signs in p_T_given_G.

Run in the authoring container only (needs the reference checkout):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_pick.py

run_grasp_simulation.py imports the simulator, dexnet, open3d and the networks at module level; none of them runs in
compute_candidate_grasp once the collaborators above are replaced, so they are empty stub modules for the import only.
Utils is the reference's own (depth2xyzmap, toOpen3dCloud, correct_pcd_normal_direction).  open3d is the numpy
point-cloud stand-in of make_golden_cloud.py, extended with the calls compute_candidate_grasp makes: estimate_normals
(normals (0, 0, 1): nothing downstream of the replaced collaborators reads them), voxel_down_sample (oracle/cloud_ref)
and io.write_point_cloud (a no-op).

Scenes (a depth frame, the simulator's id map and the fixed labels):
  mixed      small segments (< 500 points), a low-density segment spread over the frame, two segments of equal count,
             a segment on one image row at one depth (zero extents: density inf, an inlier) and ordinary segments, with labels in
             shuffled order; one of the kept objects returns no grasps
  equal      four segments of equal count: the visit order is descending label
  none       no inlier: the generator ends after the segment stage
"""
import os
import sys
import types

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, "/root/reference")

from oracle import cloud_ref   # noqa: E402


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


class _PointCloud:
    def __init__(self):
        self.points = np.zeros((0, 3))
        self.normals = np.zeros((0, 3))
        self.colors = np.zeros((0, 3))

    def estimate_normals(self, search_param=None):
        self.normals = np.tile([0.0, 0.0, 1.0], (len(self.points), 1))

    def voxel_down_sample(self, voxel_size):
        out = _PointCloud()
        out.points, _ = cloud_ref.voxel_down_sample(np.asarray(self.points), voxel_size)
        return out


_o3d = types.ModuleType("open3d")
_o3d.geometry = types.SimpleNamespace(PointCloud=_PointCloud, KDTreeSearchParamHybrid=lambda **k: None)
_o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64))
_o3d.io = types.SimpleNamespace(write_point_cloud=lambda *a, **k: None)
sys.modules["open3d"] = _o3d

_ABSENT = ["trimesh", "transformations", "autolab_core", "pybullet", "pybullet_data", "pybullet_tools",
           "pybullet_tools.utils", "dexnet", "dexnet.grasping", "dexnet.grasping.grasp",
           "dexnet.grasping.grasp_sampler", "dexnet.grasping.gripper", "data_reader", "pybullet_env",
           "pybullet_env.env_base", "pybullet_env.env_grasp", "pybullet_env.env", "pybullet_env.utils_pybullet",
           "pybullet_env.env_semantic_grasp", "pointnet2", "aligning", "dataset_nunocs", "dataset_grasp", "predicter",
           "my_cpp"]
for _m in _ABSENT:
    sys.modules[_m] = _Stub(_m)

import run_grasp_simulation as RGS   # noqa: E402  the reference itself

H, W = 40, 640
K = np.array([[600.0, 0, 320.0], [0, 600.0, 20.0], [0, 0, 1]])
BG_BODY = 100          # the simulator id of the bin (an environment body)
N_CLASSES = 11         # config_grasp.yml classes


def _scene(name, rng):
    """(depth (H,W) float32, sim id map (H,W), labels of the no-background points, grasps per label)."""
    depth = np.full((H, W), 0.7, np.float32) - rng.uniform(0, 0.05, (H, W)).astype(np.float32)
    seg = np.full((H, W), BG_BODY, np.int64)
    lab = np.full((H, W), -1, np.int64)

    def put(label, rows, cols):
        seg[rows, cols] = 1000 + label
        lab[rows, cols] = label

    if name == "mixed":
        put(0, slice(0, 20), slice(0, 40))                # 800, inlier
        put(1, slice(20, 40), slice(0, 40))               # 800, equal to 0
        put(2, slice(0, 10), slice(40, 60))               # 200, small
        put(3, 5, slice(60, 640))                         # 580 on one row at one depth: zero y and z extents
        depth[5, 60:640] = np.float32(0.69)
        put(4, slice(0, 40), slice(100, 130))             # 1200
        put(5, slice(10, 15), slice(60, 100))             # 200, small
        put(6, slice(20, 40), slice(140, 170))            # 600
        # low density: 700 pixels scattered over the frame, far in depth
        free = np.argwhere(lab == -1)
        pick = free[rng.choice(len(free), 700, replace=False)]
        lab[pick[:, 0], pick[:, 1]] = 7
        seg[pick[:, 0], pick[:, 1]] = 1007
        depth[pick[:, 0], pick[:, 1]] = rng.uniform(0.3, 1.5, len(pick)).astype(np.float32)
        depth[10, 200] = 0.05                             # below 0.1: background by depth
        perm = np.array([3, 6, 0, 7, 2, 5, 1, 4])         # labels as MeanShift numbers them: arbitrary
        lab = np.where(lab >= 0, perm[np.maximum(lab, 0)], -1)
        no_grasp = [int(perm[6])]
    elif name == "equal":
        for k in range(4):
            put(k, slice(0, 20), slice(60 * k, 60 * k + 30))   # 600 each
        put(4, slice(20, 25), slice(0, 50))                     # 250, small
        no_grasp = []
    else:
        put(0, slice(0, 10), slice(0, 40))
        put(1, slice(10, 20), slice(0, 40))
        no_grasp = []
    return depth, seg, lab, no_grasp


class _Grasp:
    def __init__(self, pose, p, idx):
        self.pose, self.p_T_given_G, self.idx = pose, p, idx

    def get_grasp_pose_matrix(self):
        return self.pose


def run(name, rng):
    depth, seg, lab_img, no_grasp = _scene(name, rng)
    bg = (depth < 0.1) | (seg == BG_BODY)
    labels = lab_img[bg == 0].reshape(-1)
    assert (labels >= 0).all()
    rec = {"ob_pts": [], "scene_pts": None, "state": None, "probs": [], "p_T_given_G": []}
    visits = []

    class Seg:
        def predict(self, data):
            self.xyz_shifted = data["cloud_xyz"]
            return labels.copy()

    def one_ob(ags, ob_pts, ob_normals, open_gripper_collision_pts, scene_pts, **kw):
        if rec["state"] is None:                          # the generator's state after the segment stage
            rec["state"] = np.random.get_state()
        rec["ob_pts"].append(np.array(ob_pts))
        rec["scene_pts"] = np.array(scene_pts)
        # the label of these points (the caller selected them with scene_seg == seg_id)
        hit = np.nonzero((xyz_nobg == ob_pts[:1]).all(-1))[0]
        sid = int(labels[hit[0]])
        visits.append(sid)
        if sid in no_grasp:
            return [], None
        G = int(rng.randint(5, 40))
        p = rng.uniform(0, 1, G)
        p[: G // 4] = p[G // 4: 2 * (G // 4)]             # exact ties
        p[-3:] = [0.0, -0.0, 0.0]                         # zeros of both signs
        rec["p_T_given_G"].append(p)
        return [_Grasp(np.eye(4), float(p[i]), i) for i in range(G)], {"seg_id": sid}

    class Q:
        def predict_batch(self, data, grasp_poses):
            G = len(grasp_poses)
            z = rng.normal(0, 30, (G, N_CLASSES - 1))
            z[::5] = 0.0                                  # some rows exactly uniform: equal p_G
            e = np.exp(z - z.max(1, keepdims=True))
            probs = (e / e.sum(1, keepdims=True)).astype(np.float32)
            rec["probs"].append(probs)
            return [[int(pr.argmax()), pr.max(), pr] for pr in probs]

    xyz_nobg = RGS.depth2xyzmap(depth, K)[bg == 0].reshape(-1, 3)
    env = types.SimpleNamespace(env_body_ids=[BG_BODY])
    RGS.cfg = {"K": K.reshape(-1).tolist()}
    RGS.cfg_grasp = {"classes": list(np.linspace(0, 1, N_CLASSES))}
    RGS.debug_dir = "/nonexistent"
    RGS.seg_predicter, RGS.grasp_predicter = Seg(), Q()
    RGS.nocs_predicter = RGS.gripper = RGS.canonical = None
    RGS.compute_candidate_grasp_one_ob = one_ob
    np.random.seed(1234)
    out = RGS.compute_candidate_grasp(np.zeros((H, W, 3), np.uint8), depth, seg, 0, env, None, [np.eye(4)])
    yielded = []
    if out is not None:
        for grasps in out:
            yielded.append(grasps)
    if rec["state"] is None:
        rec["state"] = np.random.get_state()
    res = {f"{name}_depth": depth, f"{name}_seg": seg, f"{name}_bg": bg, f"{name}_labels": labels,
           f"{name}_cloud_xyz": xyz_nobg, f"{name}_visits": np.array(visits, np.int64),
           f"{name}_rng_key": rec["state"][1], f"{name}_rng_pos": np.int64(rec["state"][2]),
           f"{name}_n_yield": np.int64(len(yielded))}
    for k, pts in enumerate(rec["ob_pts"]):
        res[f"{name}_ob_pts_{k}"] = pts
    if rec["scene_pts"] is not None:
        res[f"{name}_scene_pts"] = rec["scene_pts"]
    for k, grasps in enumerate(yielded):
        res[f"{name}_probs_{k}"] = rec["probs"][k]
        res[f"{name}_p_T_given_G_{k}"] = rec["p_T_given_G"][k]
        res[f"{name}_order_{k}"] = np.array([g.idx for g in grasps], np.int64)
        res[f"{name}_p_G_{k}"] = np.array([g.p_G for g in grasps])
        res[f"{name}_p_T_G_{k}"] = np.array([g.p_T_G for g in grasps])
        res[f"{name}_seg_id_{k}"] = np.int64(grasps[0].seg_id)
    print(f"{name}: {len(xyz_nobg)} points, visits {visits}, {len(yielded)} yields")
    return res


def main():
    rng = np.random.RandomState(77)
    res = {"K": K, "n_classes": np.int64(N_CLASSES), "seed": np.int64(1234)}
    for name in ("mixed", "equal", "none"):
        res.update(run(name, rng))
    np.savez_compressed(os.path.join(HERE, "pick_control.npz"), **res)


if __name__ == "__main__":
    main()
