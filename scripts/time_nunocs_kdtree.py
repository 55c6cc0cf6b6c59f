"""Time of the 9-DoF RANSAC's kd-tree evaluation (use_kdtree_for_eval, aligning.py:68-79), forms run alternately:
  the fused launch alone at N = 2048 and 8192, 2 x 10 000 hypotheses, kd-tree evaluation (cg_ransac9d_kdtree_pose_dev)
  against the residual evaluation (cg_ransac9d_pose_dev) on the same draws, CUDA events around each call (the kd
  call synchronises the stream three times, so its time includes those round trips);
  one object's NunocsPredicter.predict (time_nunocs.py's object, n_pts 2048) in host and device mode with the kd-tree
  evaluation on and off, wall clock.

    python scripts/time_nunocs_kdtree.py [--reps 5]
"""
import _harness
import argparse
import copy
import tempfile

import numpy as np
import torch

from catgrasp_b200 import cloud, synthetic
from catgrasp_b200.aligning import ransac9d_pose
from catgrasp_b200.predicter import NunocsPredicter

K = _harness.REFERENCE_K


def scene(N, seed):
    """A noisy scaled rotation with 20 % outliers, as the predicted NOCS cloud against the observed one; the outliers
    stay close enough that good hypotheses pass predict's max_dimensions gate."""
    rng = np.random.RandomState(seed)
    src = rng.uniform(-0.3, 0.3, (N, 3))
    R = synthetic.random_rotation(rng) * 0.03
    tgt = src @ R.T + [0.0, 0.0, 0.7] + rng.normal(0, 0.0008, (N, 3))
    out = rng.choice(N, N // 5, replace=False)
    tgt[out] += rng.uniform(-0.004, 0.004, (len(out), 3))
    return src, tgt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("card:", _harness.card())
    dev = torch.device("cuda", 0)
    H, thr = 10000, NunocsPredicter.THRESHOLDS
    gates = dict(max_scale=[0.05] * 3, min_scale=[0.005, 0.005, 0.001], max_dimensions=NunocsPredicter.MAX_DIMENSIONS)
    for N in (2048, 8192):
        src, tgt = (torch.from_numpy(x).to(dev) for x in scene(N, N))
        rng = np.random.RandomState(1)
        hyp = torch.from_numpy(np.array([rng.choice(N, 4, replace=False) for _ in range(2 * H)], np.int32)).to(dev)
        forms = {"residual": lambda: ransac9d_pose(src, tgt, hyp, thr, **gates),
                 "kd-tree": lambda: ransac9d_pose(src, tgt, hyp, thr, kdtree_eval_resolution=0.003, **gates)}
        times = {k: [] for k in forms}
        for f in forms.values():
            _harness.synced_ms(f, 1, 1)
        for _ in range(a.reps):
            for k, f in forms.items():
                times[k] += _harness.synced_ms(f, 1, 0)
        r = forms["kd-tree"]()
        print(f"N = {N}, 2 x {H}: kd-tree winners {r['winner'].tolist()} counts {r['count'].tolist()} of {2 * N}")
        for k in forms:
            print(f"  fused launch, {k:8s} {_harness.summary(times[k])}")

    depth, ids = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=16, seed=1)
    xyz = cloud.depth2xyzmap(depth, K)
    lab = ids[ids >= 0]
    pts = xyz[ids >= 0].reshape(-1, 3)
    ob = pts[lab == np.bincount(lab).argmax()]
    data = {"cloud_xyz": ob, "cloud_normal": cloud.estimate_normals(ob, 0.002, 30)}
    tmp = tempfile.mkdtemp()
    npd = NunocsPredicter("nut", artifact_dir=synthetic.write_artifacts(
        f"{tmp}/seg", "seg", 2048, with_normalizer=False, state_dict=synthetic.make_lattice_seg_state_dict(seed=5)),
        device=0)
    print(f"object: {len(ob)} points, n_pts {npd.cfg['n_pts']}, H = {npd.ransac_max_iter} per threshold")
    forms = [(m, kd) for m in ("host", "device") for kd in (False, True)]
    times = {f: [] for f in forms}

    def run(mode, kd):
        npd.subsample, npd.use_kdtree_for_eval = mode, kd
        np.random.seed(0)
        return npd.predict(copy.deepcopy(data))

    for f in forms:
        run(*f)
    for _ in range(a.reps):
        for f in forms:
            times[f] += _harness.wall_ms(lambda: run(*f), 1, 0)
    for f in forms:
        run(*f)
        ratio = getattr(npd, "best_ratio", None)
        print(f"predict {f[0]:6s} kd-tree {'on ' if f[1] else 'off'} {_harness.summary(times[f])}  best_ratio {ratio}")


if __name__ == "__main__":
    main()
