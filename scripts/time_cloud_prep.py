"""Time the point-cloud preparation of one pick on a full-resolution rendered pile (2064 x 1544, the reference camera
of config.yml:1-3): back-projection, the two scene normal passes (run_grasp_simulation.py:208-210 on the
non-background scene, :245-248 after the 1 mm scene voxel pass), the scene voxel pass itself, and prepare_object per
object (:113-139, :171-175).  CUDA events after warm-up; the card's name and power limit are printed with the numbers.

For context the same steps are timed with scipy on the host where scipy has them (cKDTree queries, query_ball_point,
numpy back-projection).  open3d's voxel_down_sample and estimate_normals are not installed here: not measured.

    python scripts/time_cloud_prep.py [--objects 8] [--reps 5] [--out results/time_cloud_prep.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from catgrasp_b200 import cloud, synthetic   # noqa: E402

K = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def gpu_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps):
        s.record()
        fn()
        e.record()
        e.synchronize()
        out.append(s.elapsed_time(e))
    return float(np.median(out))


def host_ms(fn, reps):
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append(1e3 * (time.perf_counter() - t))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    depth, ids = synthetic.render_depth(K, 1544, 2064, n_objects=a.objects, seed=0, bin_size=0.2)
    d_dev = torch.from_numpy(depth).cuda()
    res = {"card": card(), "frame": [1544, 2064]}

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
