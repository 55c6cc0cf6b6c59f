"""numpy restatement of the per-pick control stages that catgrasp_b200/csrc/cg_pick.cu runs on the device: the segment
table (run_grasp_simulation.py:217-240, :253-259, :273) and the ranking of one object's grasps (:311-328).

Both follow the reference's own expressions: np.unique over the labels, the inlier test in the cloud's dtype, the
count-ordered dict reversed, a boolean mask per segment; p_G from numpy's own sum, and Python's stable sorted.
"""
import numpy as np


def segment_table(labels, cloud_xyz):
    """Returns a dict: ``labels`` (the input with outliers set to -1), ``inlier_ids`` (ascending: one colour draw
    each, :237), ``order`` (kept labels, count descending with ties in descending label order), ``indices`` (per kept
    label, its ascending point indices), ``count``, ``min``, ``max`` and ``inlier`` per label in [0, labels.max()]."""
    scene_seg = np.array(labels, copy=True)
    xyz = np.asarray(cloud_xyz)
    L = int(scene_seg.max()) + 1 if scene_seg.size else 0
    count = np.zeros(L, np.int64)
    lo = np.zeros((L, 3))
    hi = np.zeros((L, 3))
    inlier = np.zeros(L, bool)
    inlier_ids = []
    for seg_id in np.unique(labels):
        seg_mask = labels == seg_id
        n_pt = np.sum(seg_mask)
        is_inlier = True
        if n_pt < 500:
            is_inlier = False
        seg_pts = xyz[seg_mask]
        if seg_id >= 0:
            count[seg_id] = n_pt
            lo[seg_id], hi[seg_id] = seg_pts.min(axis=0), seg_pts.max(axis=0)
        if is_inlier:
            max_xyz = seg_pts.max(axis=0)
            min_xyz = seg_pts.min(axis=0)
            with np.errstate(divide="ignore"):
                density = n_pt / np.prod((max_xyz - min_xyz) / 0.001)
            if density < 0.01:
                is_inlier = False
        if is_inlier:
            inlier_ids.append(int(seg_id))
            inlier[seg_id] = True
        else:
            scene_seg[seg_mask] = -1
    ob_n_pix = {}
    for seg_id in np.unique(scene_seg):
        if seg_id < 0:
            continue
        ob_n_pix[seg_id] = (scene_seg == seg_id).sum()
    ob_n_pix = {k: v for k, v in reversed(sorted(ob_n_pix.items(), key=lambda item: item[1]))}
    order = [int(k) for k in ob_n_pix]
    indices = [np.nonzero(scene_seg == k)[0] for k in order]
    return {"labels": scene_seg, "inlier_ids": inlier_ids, "order": order, "indices": indices, "count": count,
            "min": lo, "max": hi, "inlier": inlier}


def rank_grasps(probs, p_T_given_G, n_classes):
    """(p_G (G,), p_T_G (G,), perm (G,)): p_G = (pred * arange(C)).sum() / (n_classes - 1) with numpy's sum per row,
    p_T_G = p_T_given_G * p_G, perm = sorted(range(G), key=-p_T_G)."""
    probs = np.asarray(probs, np.float32)
    G = probs.shape[0]
    p_G = np.zeros(G)
    p_T_G = np.zeros(G)
    for i in range(G):
        pred = probs[i]
        p_G[i] = (pred * np.arange(len(pred))).sum() / (n_classes - 1)
        p_T_G[i] = float(p_T_given_G[i]) * p_G[i]
    perm = np.array(sorted(range(G), key=lambda i: -p_T_G[i]), dtype=np.int64)
    return p_G, p_T_G, perm
