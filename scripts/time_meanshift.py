"""Time the segmentation's clustering on the GPU: pointgroup_labels (down-sampling, snap, MeanShift, propagation) and
MeanShift alone, with CUDA events after warm-up, on shifted piles of about 2k, 10k and 40k down-sampled points; then
sklearn's MeanShift on the host cores for comparison.  Prints the card and its power limit in the same run.

    python scripts/time_meanshift.py [--reps 5] [--no-sklearn]
"""
import _harness
import argparse
import os
import time

import numpy as np
import torch

from catgrasp_b200 import segment, synthetic


def scene(n_points, n_objects, seed, pull=0.6, noise=0.001):
    """A pile's points and fixed offsets pulling them `pull` of the way to their object's centre."""
    s = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    xyz = s["cloud_xyz"].astype(np.float32)
    centre = s["object_poses"][:, :3, 3][s["object_id"]]
    off = (pull * (centre - s["cloud_xyz"]) + np.random.RandomState(seed).normal(0, noise, xyz.shape)).astype(np.float32)
    return xyz, off


def cuda_ms(fn, reps):
    ts = _harness.synced_ms(fn, reps, 1)
    return np.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-sklearn", action="store_true")
    args = ap.parse_args()
    print("card:", _harness.card(), "| host cores:", os.cpu_count())
    bw = segment.MEANSHIFT_BANDWIDTH["nut"]
    for n_points, n_objects, seed in ((8000, 16, 1), (40000, 40, 2), (160000, 160, 3)):
        xyz, off = scene(n_points, n_objects, seed)
        labels, shifted = segment.pointgroup_labels(xyz, off, xyz, bw)
        xs = torch.from_numpy(shifted).cuda()
        ms = segment.MeanShift(bandwidth=bw)
        ms.fit(xs)
        t_all = cuda_ms(lambda: segment.pointgroup_labels(xyz, off, xyz, bw), args.reps)
        t_ms = cuda_ms(lambda: ms.fit(xs), args.reps)
        line = (f"points {n_points:7d} -> shifted {len(shifted):6d}: clusters {len(ms.cluster_centers_):4d} "
                f"n_iter {ms.n_iter_:3d} | pointgroup_labels {t_all[0]:8.2f} ms | MeanShift {t_ms[0]:8.2f} ms "
                f"(min {t_ms[1]:.2f}, max {t_ms[2]:.2f})")
        if not args.no_sklearn:
            from sklearn.cluster import MeanShift
            t = time.perf_counter()
            MeanShift(bandwidth=bw, cluster_all=True, n_jobs=-1).fit(shifted)
            line += f" | sklearn {1e3 * (time.perf_counter() - t):9.1f} ms"
        print(line, flush=True)


if __name__ == "__main__":
    main()
