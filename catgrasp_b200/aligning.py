"""9-DoF RANSAC between the predicted NUNOCS cloud and the observed cloud (aligning.py:83-119), with all
hypotheses scored on the GPU (csrc/cg_ransac.cu; SURVEY.md 8f F1).

The host keeps exactly the reference's RNG consumption -- one ``np.random.choice(len(source), 4, replace=False)`` per
iteration, all drawn up front (aligning.py:91-97) -- and the reference's selection rule (first maximum of the inlier
ratio over the hypotheses that survive the gates, aligning.py:105-117).

``ransac9d_pose`` is the device-side form used by NunocsPredicter.predict: both thresholds scored, selected and
checked in one launch on CUDA tensors (cg_ransac9d_pose_dev), with the subsets given by the caller.
"""
import numpy as np

from . import _lib


def estimate9DTransform(source, target, PassThreshold, max_iter=1000, use_kdtree_for_eval=False,
                        kdtree_eval_resolution=None, max_scale=np.array([99, 99, 99]),
                        min_scale=np.array([0, 0, 0]), max_dimensions=None):
    """Returns (best_transform (4,4) float64, inliers) or (None, None), like aligning.py:83-119."""
    if use_kdtree_for_eval:
        raise NotImplementedError("kd-tree evaluation (aligning.py:68-79) is never enabled by the predicter")
    source = np.ascontiguousarray(source, dtype=np.float64)
    target = np.ascontiguousarray(target, dtype=np.float64)
    N = source.shape[0]
    ids = np.empty((max_iter, 4), dtype=np.int32)
    for i in range(max_iter):                                   # aligning.py:91-97
        ids[i] = np.random.choice(len(source), size=4, replace=False)
    ctx = _lib.Context.get()
    mins = np.ascontiguousarray(np.asarray(min_scale, dtype=np.float64).reshape(3))
    maxs = np.ascontiguousarray(np.asarray(max_scale, dtype=np.float64).reshape(3))
    mdim = None if max_dimensions is None else np.ascontiguousarray(np.asarray(max_dimensions, dtype=np.float64).reshape(3))
    ratio = np.empty(max_iter, np.float64)
    T = np.empty((max_iter, 4, 4), np.float64)
    valid = np.empty(max_iter, np.uint8)
    ctx.call("cg_ransac9d_host", ctx.h, source, target, N, ids, max_iter, float(PassThreshold), mins, maxs, mdim, ratio,
             T, valid)
    keep = np.nonzero(valid)[0]
    if keep.size == 0:
        return None, None
    best = keep[np.argmax(ratio[keep])]                         # first maximum among the survivors (aligning.py:115)
    best_transform = T[best].copy()
    errs = np.linalg.norm((best_transform @ np.c_[source, np.ones(N)].T).T[:, :3] - target, axis=-1)
    inliers = np.where(errs <= PassThreshold)[0]
    return best_transform, inliers


REC_PER_THR = 19     # include/catgrasp_b200.h, cg_ransac9d_pose_dev's record


def ransac9d_pose(source, target, ids, thresholds, max_scale=np.array([99, 99, 99]), min_scale=np.array([0, 0, 0]),
                  max_dimensions=None, ratio_threshold=0.003):
    """The NUNOCS pose search on the device, for CUDA tensors ``source`` / ``target`` (N,3) float64 and ``ids``
    (T*H,4) int32 (rows t*H .. t*H+H-1 are threshold t's subsets), T = len(thresholds) in {1, 2}.  One launch, no
    synchronisation.  Returns a dict of CUDA tensors (views of the launch's record):
      per threshold: 'winner' (T,) the first maximum among valid hypotheses or -1, 'count' (T,) its inlier count,
      'T' (T,4,4) its transform (bit for bit estimate9DTransform's on the same subsets), 'count_ratio' (T,) its
      count of residuals <= ratio_threshold;
      overall: 'chosen' () the threshold predict would pick or -1, 'pose' (4,4), 'best_ratio' ()."""
    import torch
    from . import _lib
    ctx, source, target = _lib.inputs(source, target, dtype=torch.float64)
    _, ids = _lib.inputs(ids, dtype=torch.int32, ctx=ctx)
    thr = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float64).reshape(-1))
    T = thr.size
    assert T in (1, 2) and ids.shape[0] % T == 0 and ids.shape[1] == 4, (thr, tuple(ids.shape))
    H = ids.shape[0] // T
    mins = np.ascontiguousarray(np.asarray(min_scale, dtype=np.float64).reshape(3))
    maxs = np.ascontiguousarray(np.asarray(max_scale, dtype=np.float64).reshape(3))
    mdim = None if max_dimensions is None else np.ascontiguousarray(np.asarray(max_dimensions, dtype=np.float64).reshape(3))
    rec = torch.empty((T * REC_PER_THR + 18,), dtype=torch.float64, device=source.device)
    ctx.call("cg_ransac9d_pose_dev", ctx.h, source, target, source.shape[0], ids, H, thr, T, mins, maxs, mdim,
             float(ratio_threshold), rec)
    per = rec[:T * REC_PER_THR].view(T, REC_PER_THR)
    tail = rec[T * REC_PER_THR:]
    return {"winner": per[:, 0].to(torch.int64), "count": per[:, 1].to(torch.int64), "T": per[:, 2:18].view(T, 4, 4),
            "count_ratio": per[:, 18].to(torch.int64), "chosen": tail[0].to(torch.int64), "pose": tail[1:17].view(4, 4),
            "best_ratio": tail[17], "record": rec}
