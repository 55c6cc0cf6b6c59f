"""9-DoF RANSAC between the predicted NUNOCS cloud and the observed cloud (aligning.py:83-119), with all
hypotheses scored on the GPU (csrc/cg_ransac.cu; SURVEY.md 8f F1).

The host keeps exactly the reference's RNG consumption -- one ``np.random.choice(len(source), 4, replace=False)`` per
iteration, all drawn up front (aligning.py:91-97) -- and the reference's selection rule (first maximum of the inlier
ratio over the hypotheses that survive the gates, aligning.py:105-117).

``ransac9d_pose`` is the device-side form used by NunocsPredicter.predict: both thresholds scored, selected and
checked in one launch on CUDA tensors (cg_ransac9d_pose_dev), with the subsets given by the caller.

Both take the reference's kd-tree evaluation (aligning.py:68-79): each hypothesis is scored by the two-way
nearest-neighbour test between the transformed source and the target, each thinned to voxel means of size
``kdtree_eval_resolution``, out of 2N (cg_ransac9d_kdtree_host / cg_ransac9d_kdtree_pose_dev).
"""
import math

import numpy as np

from . import _lib


def _resolution(r):
    """The kd-tree evaluation's voxel size as a float; ValueError when it is missing, not positive or not finite."""
    try:
        v = float(r)
    except (TypeError, ValueError):
        raise ValueError(f"kdtree_eval_resolution must be a positive finite number, got {r!r}") from None
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError(f"kdtree_eval_resolution must be a positive finite number, got {r!r}")
    return v


def _gates(min_scale, max_scale, max_dimensions):
    """The scale gates and the optional extent gate as the entry points take them: (3,) float64 arrays, None for no
    max_dimensions."""
    def vec3(a):
        return np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(3))
    return vec3(min_scale), vec3(max_scale), None if max_dimensions is None else vec3(max_dimensions)


def _ransac9d(ctx, mode, args, r, outputs):
    """Calls cg_ransac9d_<mode> on ``args`` and ``outputs``, or with a kd-tree resolution ``r``
    cg_ransac9d_kdtree_<mode>, which takes r between them."""
    if r is None:
        ctx.call(f"cg_ransac9d_{mode}", ctx.h, *args, *outputs)
    else:
        ctx.call(f"cg_ransac9d_kdtree_{mode}", ctx.h, *args, r, *outputs)


def transform_points(T, pts):
    """src_t = T [pts, 1] in the kd-tree kernel's operation order, ((T00 x + T01 y) + T02 z) + T03 per row, each
    operation rounded on its own."""
    p = np.asarray(pts, np.float64)
    return np.stack([((T[a, 0] * p[:, 0] + T[a, 1] * p[:, 1]) + T[a, 2] * p[:, 2]) + T[a, 3] for a in range(3)], 1)


def kdtree_inliers(T, source, target, PassThreshold, kdtree_eval_resolution):
    """aligning.py:79 for the hypothesis T: the source points whose transform lies within PassThreshold of a voxel
    mean of the target (voxel size kdtree_eval_resolution), with the kernel's src_t and distances."""
    from .cloud import CloudIndex, _query_cell
    import torch
    src_t = transform_points(T, source)
    down = CloudIndex(np.ascontiguousarray(target, np.float64), kdtree_eval_resolution).voxel_means()[0]
    mask = CloudIndex(down, _query_cell(down, PassThreshold), device=down.device.index).within(
        torch.from_numpy(np.ascontiguousarray(src_t)).to(down.device), PassThreshold, compare_sqrt=True)
    return np.nonzero(mask.cpu().numpy())[0]


def estimate9DTransform(source, target, PassThreshold, max_iter=1000, use_kdtree_for_eval=False,
                        kdtree_eval_resolution=None, max_scale=np.array([99, 99, 99]),
                        min_scale=np.array([0, 0, 0]), max_dimensions=None):
    """Returns (best_transform (4,4) float64, inliers) or (None, None), like aligning.py:83-119.  With
    use_kdtree_for_eval the ratio is the kd-tree evaluation's and the inliers are the winner's source points within
    PassThreshold of the target's voxel means (aligning.py:68-79); at most CG_RANSAC_KD_MAX_N = 65536 points."""
    r = _resolution(kdtree_eval_resolution) if use_kdtree_for_eval else None
    source = np.ascontiguousarray(source, dtype=np.float64)
    target = np.ascontiguousarray(target, dtype=np.float64)
    N = source.shape[0]
    ids = np.empty((max_iter, 4), dtype=np.int32)
    for i in range(max_iter):                                   # aligning.py:91-97
        ids[i] = np.random.choice(len(source), size=4, replace=False)
    ratio = np.empty(max_iter, np.float64)
    T = np.empty((max_iter, 4, 4), np.float64)
    valid = np.empty(max_iter, np.uint8)
    _ransac9d(_lib.Context.get(), "host", (source, target, N, ids, max_iter, float(PassThreshold),
                                          *_gates(min_scale, max_scale, max_dimensions)), r, (ratio, T, valid))
    keep = np.nonzero(valid)[0]
    if keep.size == 0:
        return None, None
    best = keep[np.argmax(ratio[keep])]                         # first maximum among the survivors (aligning.py:115)
    best_transform = T[best].copy()
    if r is not None:
        return best_transform, kdtree_inliers(best_transform, source, target, PassThreshold, r)
    errs = np.linalg.norm((best_transform @ np.c_[source, np.ones(N)].T).T[:, :3] - target, axis=-1)
    inliers = np.where(errs <= PassThreshold)[0]
    return best_transform, inliers


REC_PER_THR = 19     # include/catgrasp_b200.h, cg_ransac9d_pose_dev's record: 19 doubles per threshold, then 18


def read_record(rec, n_thr):
    """cg_ransac9d_pose_dev's record of n_thr thresholds, as views of ``rec`` (a CUDA tensor or its host copy):
    per threshold 'winner' (n_thr,), 'count' (n_thr,), 'T' (n_thr,4,4) and 'count_ratio' (n_thr,); overall 'chosen',
    'pose' (4,4) and 'best_ratio'.  Every value is float64; the integers are stored exactly."""
    per, tail = rec[:n_thr * REC_PER_THR].reshape(n_thr, REC_PER_THR), rec[n_thr * REC_PER_THR:]
    return {"winner": per[:, 0], "count": per[:, 1], "T": per[:, 2:18].reshape(n_thr, 4, 4), "count_ratio": per[:, 18],
            "chosen": tail[0], "pose": tail[1:17].reshape(4, 4), "best_ratio": tail[17]}


def ransac9d_pose(source, target, ids, thresholds, max_scale=np.array([99, 99, 99]), min_scale=np.array([0, 0, 0]),
                  max_dimensions=None, ratio_threshold=0.003, kdtree_eval_resolution=None):
    """The NUNOCS pose search on the device, for CUDA tensors ``source`` / ``target`` (N,3) float64 and ``ids``
    (T*H,4) int32 (rows t*H .. t*H+H-1 are threshold t's subsets), T = len(thresholds) in {1, 2}.  One launch, no
    synchronisation.  Returns a dict of CUDA tensors (views of the launch's record):
      per threshold: 'winner' (T,) the first maximum among valid hypotheses or -1, 'count' (T,) its inlier count,
      'T' (T,4,4) its transform (bit for bit estimate9DTransform's on the same subsets), 'count_ratio' (T,) its
      count of residuals <= ratio_threshold;
      overall: 'chosen' () the threshold predict would pick or -1, 'pose' (4,4), 'best_ratio' ().
    With ``kdtree_eval_resolution`` the hypotheses are scored by the kd-tree evaluation (each 'count' out of 2N; the
    launch then synchronises, see cg_ransac9d_kdtree_pose_dev)."""
    import torch
    r = None if kdtree_eval_resolution is None else _resolution(kdtree_eval_resolution)
    ctx, source, target = _lib.inputs(source, target, dtype=torch.float64)
    _, ids = _lib.inputs(ids, dtype=torch.int32, ctx=ctx)
    thr = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float64).reshape(-1))
    T = thr.size
    assert T in (1, 2) and ids.shape[0] % T == 0 and ids.shape[1] == 4, (thr, tuple(ids.shape))
    H = ids.shape[0] // T
    rec = torch.empty((T * REC_PER_THR + 18,), dtype=torch.float64, device=source.device)
    _ransac9d(ctx, "pose_dev", (source, target, source.shape[0], ids, H, thr, T,
                                *_gates(min_scale, max_scale, max_dimensions), float(ratio_threshold)), r, (rec,))
    out = read_record(rec, T)
    for k in ("winner", "count", "count_ratio", "chosen"):
        out[k] = out[k].to(torch.int64)
    return {**out, "record": rec}


def ransac9d_pose_many(source, target, ids, thresholds, max_scale=np.array([99, 99, 99]),
                       min_scale=np.array([0, 0, 0]), max_dimensions=None, ratio_threshold=0.003):
    """ransac9d_pose (residual evaluation) for B objects at once: ``source`` / ``target`` (B,N,3) float64 and ``ids``
    (B,T*H,4) int32 CUDA tensors.  Returns the (B, T*19 + 18) float64 CUDA tensor of records, row b being
    ransac9d_pose's 'record' for source[b], target[b], ids[b] bit for bit (cg_ransac9d_pose_many_dev); read a row
    with read_record.  No synchronisation."""
    import torch
    ctx, source, target = _lib.inputs(source, target, dtype=torch.float64)
    _, ids = _lib.inputs(ids, dtype=torch.int32, ctx=ctx)
    thr = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float64).reshape(-1))
    T = thr.size
    B, N = source.shape[0], source.shape[1]
    assert T in (1, 2) and source.shape == (B, N, 3) and target.shape == (B, N, 3), (thr, tuple(source.shape))
    assert ids.dim() == 3 and ids.shape[0] == B and ids.shape[1] % T == 0 and ids.shape[2] == 4, tuple(ids.shape)
    H = ids.shape[1] // T
    rec = torch.empty((B, T * REC_PER_THR + 18), dtype=torch.float64, device=source.device)
    ctx.call("cg_ransac9d_pose_many_dev", ctx.h, source, target, B, N, ids, H, thr, T,
             *_gates(min_scale, max_scale, max_dimensions), float(ratio_threshold), rec)
    return rec
