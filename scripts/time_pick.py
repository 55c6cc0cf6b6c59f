"""Wall time of compute_candidate_grasp (catgrasp_b200/pick.py) and of each of its stages (its ``timings``: scene
stages once, per-object stages summed over the objects) on the 16-object full-resolution render_depth pile (the
reference K, 1544 x 2064), with synthetic weights: the renderer's id map stands in for the segmentation.  Each stage time ends in a device synchronise.

    python scripts/time_pick.py [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from catgrasp_b200 import pick, synthetic   # noqa: E402

K = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)
CFG_RUN = {"nocs_grasp_sampler_score_larger_than": 0.95, "nocs_grasp_sampler_max_n_grasp": 10000,
           "cone_grasp_smapler_n_sphere_dir": 30, "cone_grasp_smapler_approach_step": 0.002}


class IdSegmenter:
    def __init__(self, labels):
        self.labels = labels

    def predict(self, data):
        return self.labels.clone()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("GPU:", smi)
    depth, ids = synthetic.render_depth(K, 1544, 2064, n_objects=16, seed=1)
    bg = ids < 0
    dev = torch.device("cuda", 0)
    from catgrasp_b200.predicter import GraspPredicter, NunocsPredicter
    tmp = tempfile.mkdtemp()
    gp = GraspPredicter("nut", artifact_dir=synthetic.write_artifacts(f"{tmp}/cls", "cls", 2048, seed=3), device=0)
    npd = NunocsPredicter("nut", artifact_dir=synthetic.write_artifacts(
        f"{tmp}/seg", "seg", 2048, with_normalizer=False, state_dict=synthetic.make_lattice_seg_state_dict(seed=5)),
        device=0)
    seg = IdSegmenter(torch.from_numpy(ids[~bg].astype(np.int64)).to(dev))
    g = synthetic.make_gripper_proxy()
    box = [0.0, 0.045, -0.010, 0.010]
    gripper = {"vertices": g["open"]["V"], "faces": g["open"]["F"], "enclosed_vertices": g["enclosed"]["V"],
               "enclosed_faces": g["enclosed"]["F"], "hand_depth": 0.012, "init_bite": 0.002,
               "grasp_in_gripper": np.linalg.inv(g["gripper_in_grasp"]), "finger_boxes": np.array([box, box]),
               "grip_dirs": np.array([[0, -1, 0], [0, 1, 0]]), "finger_mesh_in_grasp": g["gripper_in_grasp"]}
    cam = np.eye(4)
    cam[:3, :3] = np.diag([1.0, -1.0, -1.0])
    cam[:3, 3] = [0.6, 0.0, 0.85]
    eeg = np.eye(4)
    eeg[:3, :3] = np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], float).T
    eeg[:3, 3] = [-0.17, 0, 0]
    up = np.deg2rad([170, 120, 170, 120, 170, 120, 175])
    env = {"cam_in_world": cam, "bin_in_world": np.eye(4), "ee_in_grasp": eeg, "upper": up, "lower": -up}
    rng = np.random.RandomState(31)
    pts, nrm = synthetic.sample_hex_nut(3000, rng)
    lo, s = pts.min(0), (pts.max(0) - pts.min(0)).max()
    poses = synthetic.make_candidates(pts, nrm, 200, seed=32)
    poses[:, :3, 3] = (poses[:, :3, 3] - lo) / s
    canonical = {"canonical_grasps": poses, "canonical_scores": rng.uniform(0.9, 1, 200),
                 "canonical_cloud": (pts - lo) / s, "canonical_normals": nrm,
                 "canonical_affordance": np.clip(0.5 + 0.5 * np.sin(40 * pts[:, 0]), 0, 1)}
    d_depth, d_bg = torch.from_numpy(depth).to(dev), torch.from_numpy(bg).to(dev)

    for rep in range(a.reps):
        np.random.seed(0)
        timings = {}
        t0 = time.perf_counter()
        n_obj, n_grasp = 0, 0
        for r in pick.compute_candidate_grasp(d_depth, K, d_bg, seg, npd, gp, gripper, env, canonical, [np.eye(4)],
                                              CFG_RUN, timings=timings):
            n_obj += 1
            n_grasp += len(r["grasp_poses"])
        torch.cuda.synchronize()
        t_all = (time.perf_counter() - t0) * 1e3
        print(f"rep {rep}: {int(bg.size - bg.sum())} no-background points, {n_obj} objects yielded, {n_grasp} grasps")
        for name, t in timings.items():
            print(f"  {name:40s} {t:10.2f} ms")
        print(f"  {'sum of the stages':40s} {sum(timings.values()):10.2f} ms")
        print(f"  {'compute_candidate_grasp, whole call':40s} {t_all:10.2f} ms")


if __name__ == "__main__":
    main()
