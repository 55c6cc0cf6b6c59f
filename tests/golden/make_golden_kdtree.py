"""Golden vectors for the kd-tree evaluation of the 9-DoF RANSAC, produced by EXECUTING THE REFERENCE's own
aligning.py (``estimate9DTransform(use_kdtree_for_eval=True)``, aligning.py:68-79, with the real cv2 and scipy).

Run in the authoring container only (needs the reference tree; the GPU box does not have it):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_kdtree.py

The reference's imports are stubbed as in make_golden_hostpath.py.  open3d is absent, so for the calls this path makes
(``Utils.toOpen3dCloud`` -> ``PointCloud.voxel_down_sample``) it is replaced by a stand-in whose voxel_down_sample is
oracle/cloud_ref.voxel_down_sample: open3d's origin and cell rule, each voxel the mean of its points in ascending
index.  Parity with open3d itself stays unpinned.  ``estimate9DTransform_worker`` is wrapped (it still runs
unmodified) to record each hypothesis's ratio and transform.

Cases 0-3: the source / target pair of host_ransac9d.npz, PassThreshold 0.003 and 0.005 x kdtree_eval_resolution
0.003 (predict's) and 2^-8, each with 1000 draws under its own seed and predict's gates (the nut's scales,
max_dimensions = [1.2] * 3).  Case 4 is exact: a dyadic lattice (8^3 points 2^-3 apart) under T = 2^-3 I + t, with
every other target point moved by exactly PassThreshold = 2^-8 along x, kdtree_eval_resolution 2^-8 (one point per
voxel) and max_scale 0.2, so every moved point's nearest voxel mean is exactly PassThreshold away.
Written: host_ransac9d_kdtree.npz with, per case c, ``c<k>_source``, ``c<k>_target``, ``c<k>_seed``, ``c<k>_thr``,
``c<k>_res``, ``c<k>_max_scale``, ``c<k>_iters`` (iterations whose hypothesis passed the gates), ``c<k>_ratios``,
``c<k>_T`` (their transforms), ``c<k>_transform`` / ``c<k>_inliers`` (what estimate9DTransform returned) and
``c<k>_next_rand``.
"""
import os
import sys
import types

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden_hostpath as hp            # noqa: E402  stubs the absent imports, imports the reference
from oracle import cloud_ref                 # noqa: E402

CASES = [(0.003, 0.003), (0.003, 2.0 ** -8), (0.005, 0.003), (0.005, 2.0 ** -8)]
MAX_ITER = 1000
MIN_S, MAX_S, MAX_D = [0.005, 0.005, 0.001], [0.05, 0.05, 0.05], np.array([1.2, 1.2, 1.2])


class _PointCloud:
    def __init__(self):
        self.points = np.zeros((0, 3))

    def voxel_down_sample(self, voxel_size):
        out = _PointCloud()
        out.points = cloud_ref.voxel_down_sample(np.asarray(self.points, np.float64), voxel_size)[0]
        return out


def _open3d():
    m = types.ModuleType("open3d")
    m.geometry = types.SimpleNamespace(PointCloud=_PointCloud)
    m.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, np.float64))
    return m


def main():
    sys.modules["open3d"] = _open3d()            # Utils.toOpen3dCloud imports open3d when it is called
    ref = hp.ref_aligning
    worker = ref.estimate9DTransform_worker
    seen = []

    def recording_worker(*a, **k):
        out = worker(*a, **k)
        seen.append(out)
        return out

    ref.estimate9DTransform_worker = recording_worker
    g = np.load(os.path.join(HERE, "host_ransac9d.npz"))
    lat = np.stack(np.meshgrid(*[np.arange(8) * 0.125] * 3, indexing="ij"), -1).reshape(-1, 3)
    moved = lat * 0.125 + np.array([0.5, 0.25, 0.75])
    moved[::2, 0] += 2.0 ** -8
    cases = [(g["source"], g["target"], thr, res, MAX_S) for thr, res in CASES]
    cases.append((lat, moved, 2.0 ** -8, 2.0 ** -8, [0.2] * 3))
    out = {}
    for c, (src, tgt, thr, res, max_s) in enumerate(cases):
        seed = 40 + c
        np.random.seed(seed)
        seen.clear()
        tf, inl = ref.estimate9DTransform(source=src, target=tgt, PassThreshold=thr, max_iter=MAX_ITER,
                                          use_kdtree_for_eval=True, kdtree_eval_resolution=res,
                                          max_scale=max_s, min_scale=MIN_S, max_dimensions=MAX_D)
        iters = [i for i, o in enumerate(seen) if o[0] is not None]
        out.update({f"c{c}_source": src, f"c{c}_target": tgt, f"c{c}_seed": seed, f"c{c}_thr": thr, f"c{c}_res": res,
                    f"c{c}_max_scale": np.asarray(max_s, np.float64),
                    f"c{c}_iters": np.array(iters, np.int32),
                    f"c{c}_ratios": np.array([seen[i][0] for i in iters]),
                    f"c{c}_T": np.array([seen[i][1] for i in iters]).reshape(-1, 4, 4),
                    f"c{c}_transform": tf, f"c{c}_inliers": np.asarray(inl, np.int32),
                    f"c{c}_next_rand": np.random.rand(2)})
        print(f"case {c}: thr {thr} res {res}: {len(iters)} valid of {MAX_ITER}, best ratio "
              f"{max(seen[i][0] for i in iters):.4f}, {len(inl)} inliers")
    ref.estimate9DTransform_worker = worker
    np.savez_compressed(os.path.join(HERE, "host_ransac9d_kdtree.npz"), **out)


if __name__ == "__main__":
    main()
