"""Time the point-cloud preparation of one pick on a full-resolution rendered pile (2064 x 1544, the reference camera
of config.yml:1-3): back-projection, the two scene normal passes (run_grasp_simulation.py:208-210 on the
non-background scene, :245-248 after the 1 mm scene voxel pass), the scene voxel pass itself, and prepare_object per
object (:113-139, :171-175).  CUDA events after warm-up; the card's name and power limit are printed with the numbers.

For context the same steps are timed with scipy on the host where scipy has them (cKDTree queries, query_ball_point,
numpy back-projection).  open3d's voxel_down_sample and estimate_normals are not installed here: not measured.

    python scripts/time_cloud_prep.py [--objects 8] [--reps 5] [--out results/time_cloud_prep.json]
"""
import _harness
import argparse
import json
import os

import numpy as np
import torch

from catgrasp_b200 import cloud, synthetic

K = _harness.REFERENCE_K


def gpu_ms(fn, reps):
    return float(np.median(_harness.synced_ms(fn, reps, 1)))


def host_ms(fn, reps):
    return float(np.median(_harness.wall_ms(fn, reps, 0)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": _harness.card(), "frame": list(_harness.REFERENCE_HW)}
    print("card:", res["card"])
    depth, ids = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=a.objects, seed=0, bin_size=0.2)
    d_dev = torch.from_numpy(depth).cuda()

    xyz_dev = cloud.depth2xyzmap(d_dev, K)
    xyz = xyz_dev.cpu().numpy()
    valid = xyz[:, :, 2] >= 0.1
    scene_pts = xyz[valid].reshape(-1, 3)
    no_bg = xyz[(ids >= 0) & (depth >= 0.1)].reshape(-1, 3)      # the id map stands in for PointGroup's masks
    res["scene_points"], res["no_bg_points"] = int(len(scene_pts)), int(len(no_bg))
    no_bg_dev = torch.from_numpy(no_bg.astype(np.float64)).cuda()
    scene_dev = torch.from_numpy(scene_pts.astype(np.float64)).cuda()

    res["gpu_ms"] = {
        "depth2xyzmap": gpu_ms(lambda: cloud.depth2xyzmap(d_dev, K), a.reps),
        "normals_no_bg_r2mm": gpu_ms(lambda: cloud.estimate_normals(no_bg_dev, 0.002, 30), a.reps),
        "scene_voxel_1mm": gpu_ms(lambda: cloud.voxel_down_sample(scene_dev, 0.001), a.reps),
    }
    scene_down = cloud.voxel_down_sample(scene_dev, 0.001)
    res["scene_voxels"] = int(scene_down.shape[0])
    res["gpu_ms"]["normals_scene_r3mm"] = gpu_ms(lambda: cloud.estimate_normals(scene_down, 0.003, 30), a.reps)
    scene_down_np = scene_down.cpu().numpy()
    obs = []
    for k in np.unique(ids[ids >= 0]):
        ob = xyz[(ids == k) & valid].reshape(-1, 3)
        ob_n = cloud.estimate_normals(ob, 0.002, 30)
        obs.append((ob, ob_n))
    res["object_points"] = [int(len(o[0])) for o in obs]
    per = [gpu_ms(lambda o=o: cloud.prepare_object(o[0], o[1], scene_down_np, 0.2), a.reps) for o in obs]
    res["gpu_ms"]["prepare_object_per_object"] = per
    res["gpu_ms"]["prepare_object_all"] = float(sum(per))

    from scipy.spatial import cKDTree
    from oracle import cloud_ref

    def host_prepare(ob):
        down, _ = cloud_ref.voxel_down_sample(ob, 0.0005)        # numpy stand-in for open3d (not open3d)
        cKDTree(ob).query(down)
        d, _ = cKDTree(ob).query(scene_down_np)
        bg = scene_down_np[d <= 0.1]
        cKDTree(bg).query_ball_point(ob, r=0.005, workers=-1) if len(bg) else None

    res["host_ms"] = {
        "depth2xyzmap_numpy": host_ms(lambda: cloud_ref.depth2xyzmap(depth, K), 2),
        "prepare_object_scipy_queries_all": float(sum(host_ms(lambda o=o: host_prepare(o[0]), 2) for o in obs)),
        "open3d_voxel_down_sample": "not measured",
        "open3d_estimate_normals": "not measured",
    }
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
