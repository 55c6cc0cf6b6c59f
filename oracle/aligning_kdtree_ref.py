"""CPU ORACLE (test infrastructure only): the kd-tree evaluation of the NUNOCS 9-DoF RANSAC.

Restates aligning.py:68-79 (``estimate9DTransform_worker`` with ``use_kdtree_for_eval=True``) and the selection of
aligning.py:83-119 around it: numpy + cKDTree on voxel means from oracle/cloud_ref.voxel_down_sample, the rule
open3d's ``voxel_down_sample`` stands in for.  The hypotheses, their gates and the numpy RNG consumption are
oracle/aligning_ref.py's (``_hypothesis``, one ``np.random.choice(len(source), 4, replace=False)`` per iteration,
all drawn up front), so only the scoring differs.
PINNED: tests/test_kdtree_eval_ref.py compares it with outputs of the reference's own aligning.py run with
``use_kdtree_for_eval=True`` (tests/golden/make_golden_kdtree.py -> host_ransac9d_kdtree.npz).
"""
import numpy as np

from . import aligning_ref, cloud_ref


def transform_points(T, source, order="matmul"):
    """src_t = T [source, 1]: numpy's matmul as aligning.py:62 computes it ("matmul"), or the kd-tree kernel's order
    ((T00 x + T01 y) + T02 z) + T03 with each operation rounded on its own ("kernel")."""
    source = np.asarray(source, np.float64)
    if order == "matmul":
        return (T @ aligning_ref._to_homo(source).T).T[:, :3]
    assert order == "kernel", order
    return np.stack([((T[a, 0] * source[:, 0] + T[a, 1] * source[:, 1]) + T[a, 2] * source[:, 2]) + T[a, 3]
                     for a in range(3)], 1)


def kdtree_eval(T, source, target, PassThreshold, kdtree_eval_resolution, order="matmul"):
    """aligning.py:68-79 for one hypothesis: (count of dists1 <= thr plus dists2 <= thr, inliers = where(dists1 <=
    thr)).  The ratio is count / (2 len(source))."""
    from scipy.spatial import cKDTree
    target = np.asarray(target, np.float64)
    src_t = transform_points(T, source, order)
    dists1 = cKDTree(cloud_ref.voxel_down_sample(target, kdtree_eval_resolution)[0]).query(src_t)[0]
    dists2 = cKDTree(cloud_ref.voxel_down_sample(src_t, kdtree_eval_resolution)[0]).query(target)[0]
    count = int(np.sum(dists1 <= PassThreshold)) + int(np.sum(dists2 <= PassThreshold))
    return count, np.where(dists1 <= PassThreshold)[0]


def estimate9DTransform(source, target, PassThreshold, kdtree_eval_resolution, max_iter=1000,
                        max_scale=np.array([99, 99, 99]), min_scale=np.array([0, 0, 0]), max_dimensions=None,
                        order="matmul", ratios_out=None):
    """aligning.py:83-119 with use_kdtree_for_eval=True.  Returns (best_transform (4,4), inliers) or (None, None).
    ``order`` picks how the source is transformed (transform_points); ``ratios_out``, a list, receives
    (iteration, ratio, T) of every hypothesis that passes the gates."""
    source = np.asarray(source, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    max_scale = np.asarray(max_scale, dtype=np.float64)
    min_scale = np.asarray(min_scale, dtype=np.float64)
    srcs, dsts = [], []
    for _ in range(max_iter):                                   # aligning.py:91-97
        ids = np.random.choice(len(source), size=4, replace=False)
        srcs.append(source[ids])
        dsts.append(target[ids])
    transforms, its = [], []
    for i in range(len(srcs)):                                  # aligning.py:99-104
        T = aligning_ref._hypothesis(srcs[i], dsts[i], target, PassThreshold, max_scale, min_scale, max_dimensions)
        if T is not None:
            transforms.append(T)
            its.append(i)
    if len(transforms) == 0:
        return None, None
    evals = [kdtree_eval(T, source, target, PassThreshold, kdtree_eval_resolution, order) for T in transforms]
    ratios = np.array([c / (2 * len(source)) for c, _ in evals])
    if ratios_out is not None:
        ratios_out.extend(zip(its, ratios, transforms))
    best_id = ratios.argmax()                                   # aligning.py:115
    return transforms[best_id], evals[best_id][1]
