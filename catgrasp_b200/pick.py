"""The per-pick call: the reference's ``compute_candidate_grasp`` (run_grasp_simulation.py:188-329, with
``compute_candidate_grasp_one_ob`` :112-183 and ``compute_grasp_affordance`` :73-107) from a depth frame to each
object's ranked grasps, built from the package's per-stage calls.

The glue that was host code in the reference runs on the device (csrc/cg_pick.cu): the segment table of the
segmentation's labels (inlier test, largest-first order, each object's points) and the ranking of an object's scored
grasps.  Scene-sized arrays stay on the device.  Per-object arrays reach the host only for the stages that are
host-side (NUNOCS, the cone sampler's frames, the affordance's kd-tree query, grasp-Q's subset draw).  The host
synchronises only where a control-flow decision or a size is needed; DESIGN.md lists each one.

The global numpy generator is consumed exactly as the reference consumes it: one ``np.random.randint(0, 255, size=3)``
per inlier segment (the segment colours of :237, whose values nothing reads), then per object the draws of NUNOCS,
the cone sampler and grasp-Q, in the reference's order.

Several frames (a cell with several bins or cameras) go through ``compute_candidate_grasp_many``: the scene stages of
all frames run once, on one flat buffer and many-set indices, and each frame's objects are then visited lazily by a
generator of its own.  ``compute_candidate_grasp`` is its one-frame case.
"""
import copy
import time

import numpy as np
import torch

from . import _lib


def segment_table(labels, cloud_xyz, n_labels):
    """run_grasp_simulation.py:217-240, :253-259 and :273 on the device, without synchronising.

    ``labels`` (M,) int32 / int64 and ``cloud_xyz`` (M,3) float32 / float64 are CUDA tensors; labels lie in
    [0, n_labels) (the segmenter's cluster count).  Returns a dict of CUDA tensors: ``labels`` (outliers set to -1),
    ``count`` (L,) int32, ``min`` / ``max`` (L,3) float64, ``inlier`` (L,) uint8, ``order`` (L,) int32 (the kept
    labels, count descending with ties in descending label order, then -1), ``n_kept`` (1,) int32, ``offsets``
    (L+1,) int32 and ``index`` (M,) int32 (the k-th kept segment's point indices, ascending, at
    index[offsets[k]:offsets[k+1]])."""
    if not (isinstance(labels, torch.Tensor) and labels.is_cuda and isinstance(cloud_xyz, torch.Tensor)):
        raise ValueError("segment_table: labels and cloud_xyz must be CUDA tensors")
    if labels.dtype not in (torch.int32, torch.int64) or cloud_xyz.dtype not in (torch.float32, torch.float64):
        raise ValueError("segment_table: labels must be int32 / int64 and cloud_xyz float32 / float64")
    M = labels.shape[0]
    if labels.ndim != 1 or tuple(cloud_xyz.shape) != (M, 3):
        raise ValueError(f"segment_table: labels (M,) and cloud_xyz (M,3), got {tuple(labels.shape)} and "
                         f"{tuple(cloud_xyz.shape)}")
    L = int(n_labels)
    ctx, lab, x = _lib.inputs(labels, cloud_xyz, dtype=(labels.dtype, cloud_xyz.dtype))
    dev = lab.device
    i32 = dict(dtype=torch.int32, device=dev)
    out = {"labels": torch.empty_like(lab), "count": torch.empty(L, **i32),
           "min": torch.empty((L, 3), dtype=torch.float64, device=dev),
           "max": torch.empty((L, 3), dtype=torch.float64, device=dev),
           "inlier": torch.empty(L, dtype=torch.uint8, device=dev), "order": torch.empty(L, **i32),
           "n_kept": torch.empty(1, **i32), "offsets": torch.empty(L + 1, **i32), "index": torch.empty(M, **i32)}
    ctx.call("cg_segment_table_dev", ctx.h, lab, int(lab.dtype == torch.int64), x, int(x.dtype == torch.float64), M, L,
             out["labels"], out["count"], out["min"], out["max"], out["inlier"], out["order"], out["n_kept"],
             out["offsets"], out["index"])
    return out


def segment_table_many(labels, cloud_xyz, point_offsets, n_labels):
    """segment_table of B frames laid end to end, in one pass without synchronising.

    ``labels`` (M,) and ``cloud_xyz`` (M,3) CUDA tensors as segment_table takes them; frame b's points are the rows
    [point_offsets[b], point_offsets[b + 1]) (B + 1 ascending ints from 0 to M; a frame may have no point), with
    frame-local labels in [0, n_labels[b]) (each >= 1).  Returns segment_table's dict with each entry the frames'
    tables laid end to end, frame-local labels and point indices unchanged: ``labels`` and ``index`` (M,) in blocks of
    M_b, ``count`` / ``min`` / ``max`` / ``inlier`` / ``order`` in blocks of L_b = n_labels[b], ``n_kept`` (B,) and
    ``offsets`` (sum L_b + B,) in blocks of L_b + 1.  Frame b's blocks equal segment_table on frame b alone, bit for
    bit."""
    if not (isinstance(labels, torch.Tensor) and isinstance(cloud_xyz, torch.Tensor)):
        raise ValueError("segment_table_many: labels and cloud_xyz must be CUDA tensors")
    if labels.dtype not in (torch.int32, torch.int64) or cloud_xyz.dtype not in (torch.float32, torch.float64):
        raise ValueError("segment_table_many: labels must be int32 / int64 and cloud_xyz float32 / float64")
    M = labels.shape[0]
    if labels.ndim != 1 or tuple(cloud_xyz.shape) != (M, 3):
        raise ValueError(f"segment_table_many: labels (M,) and cloud_xyz (M,3), got {tuple(labels.shape)} and "
                         f"{tuple(cloud_xyz.shape)}")
    nl = np.asarray(n_labels, np.int64).reshape(-1)
    poff = np.asarray(point_offsets, np.int64).reshape(-1)
    B = len(nl)
    if B == 0 or (nl < 1).any():
        raise ValueError(f"segment_table_many: need one label count >= 1 per frame, got {nl.tolist()}")
    if len(poff) != B + 1 or poff[0] != 0 or poff[-1] != M or (np.diff(poff) < 0).any():
        raise ValueError(f"segment_table_many: need {B + 1} ascending point offsets from 0 to {M}, got {poff.tolist()}")
    if not labels.is_cuda:
        raise ValueError("segment_table_many: labels and cloud_xyz must be CUDA tensors")
    loff = np.concatenate([[0], np.cumsum(nl)])
    L = int(loff[-1])
    ctx, lab, x = _lib.inputs(labels, cloud_xyz, dtype=(labels.dtype, cloud_xyz.dtype))
    dev = lab.device
    i32 = dict(dtype=torch.int32, device=dev)
    out = {"labels": torch.empty_like(lab), "count": torch.empty(L, **i32),
           "min": torch.empty((L, 3), dtype=torch.float64, device=dev),
           "max": torch.empty((L, 3), dtype=torch.float64, device=dev),
           "inlier": torch.empty(L, dtype=torch.uint8, device=dev), "order": torch.empty(L, **i32),
           "n_kept": torch.empty(B, **i32), "offsets": torch.empty(L + B, **i32), "index": torch.empty(M, **i32)}
    ctx.call("cg_segment_table_many_dev", ctx.h, lab, int(lab.dtype == torch.int64), x, int(x.dtype == torch.float64),
             B, poff.astype(np.int32), loff.astype(np.int32), out["labels"], out["count"], out["min"], out["max"],
             out["inlier"], out["order"], out["n_kept"], out["offsets"], out["index"])
    return out


def rank_grasps(probs, p_T_given_G, n_classes):
    """run_grasp_simulation.py:311-328 on the device, without synchronising: ``probs`` (G,C) float32 and
    ``p_T_given_G`` (G,) float64 CUDA tensors, ``n_classes`` = len(cfg_grasp['classes']).  Returns (p_G (G,) float64,
    p_T_G (G,) float64, perm (G,) int64): p_G = (pred * arange(C)).sum() / (n_classes - 1) bit for bit with numpy,
    p_T_G = p_T_given_G * p_G, perm = Python's stable sorted(range(G), key=-p_T_G)."""
    if probs.ndim != 2 or p_T_given_G.shape != (probs.shape[0],):
        raise ValueError(f"rank_grasps: probs (G,C) and p_T_given_G (G,), got {tuple(probs.shape)} and "
                         f"{tuple(p_T_given_G.shape)}")
    G, C = probs.shape
    ctx, pr, pt = _lib.inputs(probs, p_T_given_G, dtype=(torch.float32, torch.float64))
    p_G = torch.empty(G, dtype=torch.float64, device=pr.device)
    p_T_G = torch.empty_like(p_G)
    perm = torch.empty(G, dtype=torch.int32, device=pr.device)
    ctx.call("cg_rank_grasps_dev", ctx.h, pr, G, C, int(n_classes) - 1, pt, p_G, p_T_G, perm)
    return p_G, p_T_G, perm.to(torch.int64)


def preselect_canonical(grasps, scores, score_larger_than=0, max_n_grasp=None):
    """NocsTransferGraspSampler.__init__ (grasp_sampler.py:330-349, without center_ob_between_gripper, which the
    reference's sampler leaves False): keep the canonical grasps with score >= score_larger_than when that is > 0,
    then the first max_n_grasp of them by descending score (a stable sort).  Returns the (N,4,4) poses."""
    grasps = np.asarray(grasps, np.float64).reshape(-1, 4, 4)
    scores = np.asarray(scores, np.float64).reshape(-1)
    keep = np.arange(len(grasps))
    if score_larger_than > 0:
        keep = keep[scores[keep] >= score_larger_than]
    if max_n_grasp is not None:
        keep = keep[np.argsort(-scores[keep], kind="stable")][:max_n_grasp]
    return grasps[keep]


def _filter(poses, symmetry_tfs, nocs_pose, gripper_in_grasp, open_pts, background_pts, gripper, env):
    """my_cpp.filterGraspPose as the samplers call it (filter_approach_dir_face_camera, filter_ik and
    adjust_collision_pose all True, canonical_to_nocs = I, octo resolution 0.0005): the surviving poses as a (Q,4,4)
    float32 CUDA tensor in (pose, symmetry) order.  A host IK hook (my_cpp.set_ik_solver) goes through
    filterGraspPose itself."""
    from . import my_cpp
    eye = np.eye(4)
    if my_cpp._IK_SOLVER is not None:
        got = my_cpp.filterGraspPose(
            poses.cpu().numpy() if isinstance(poses, torch.Tensor) else poses, list(symmetry_tfs), nocs_pose, eye,
            env["cam_in_world"], env["ee_in_grasp"], gripper_in_grasp, True, True, True, env["upper"], env["lower"],
            gripper["vertices"], gripper["faces"], gripper["enclosed_vertices"], gripper["enclosed_faces"],
            open_pts.cpu().numpy(), background_pts.cpu().numpy(), 0.0005, False)
        return torch.from_numpy(np.array(got, np.float32).reshape(-1, 4, 4)).to(open_pts.device)
    if len(poses) == 0 or len(symmetry_tfs) == 0:
        return torch.zeros((0, 4, 4), dtype=torch.float32, device=open_pts.device)
    sdf_open = my_cpp._sdf_for(gripper["vertices"], gripper["faces"])
    sdf_encl = my_cpp._sdf_for(gripper["enclosed_vertices"], gripper["enclosed_faces"])
    margin = my_cpp.voxel_margin(0.0005) if my_cpp.COLLISION_PREDICATE == "voxel" else 0.0
    poses = poses if isinstance(poses, torch.Tensor) else torch.from_numpy(np.asarray(poses, np.float64))
    status, _, out = my_cpp.filter_grasp_pose_raw(
        poses.to(open_pts.device), symmetry_tfs, nocs_pose, eye, gripper_in_grasp, True, True, sdf_open, open_pts,
        sdf_encl, background_pts, sdf_margin=margin,
        ik=(env["cam_in_world"], env["ee_in_grasp"], env["upper"], env["lower"]))
    return out[status == _lib.CG_ST_ACCEPT]


def _lap(timings, name, t0):
    """With a ``timings`` dict: synchronise the device, add the wall time since ``t0`` to timings[name] (ms) and return
    the new start.  Without one: nothing."""
    if timings is None:
        return None
    torch.cuda.synchronize()
    t = time.perf_counter()
    timings[name] = timings.get(name, 0.0) + (t - t0) * 1e3
    return t


def compute_candidate_grasp(depth, K, bg_mask, seg_predicter, nocs_predicter, grasp_predicter, gripper, env, canonical,
                            symmetry_tfs, cfg_run, n_classes=None, device=None, timings=None):
    """run_grasp_simulation.py:188-329: a generator over the objects of one depth frame, largest first, yielding each
    object that has grasps left as a dict

      seg_id, ob_pts (the object's points, CUDA tensor), data (the dict predict_batch saw), nocs_pose, and in ranked
      order grasp_poses (G,4,4) float32, pred_label (G,), pred (G,C), p_T_given_G, p_G, p_T_G (G,) float64.

    Arguments (what the reference reads from its globals and ``env``):
      depth (H,W), K (3,3); bg_mask (H,W), nonzero where a pixel is background (:193-195: depth < 0.1 or a pixel
      of an environment body; the caller computes it);
      seg_predicter / nocs_predicter / grasp_predicter: objects with the predictors' ``predict`` / ``predict_batch``;
      a segmenter gets {'cloud_xyz', 'cloud_normal'} CUDA tensors and returns one label per point in [0, L);
      gripper: dict of 'vertices', 'faces', 'enclosed_vertices', 'enclosed_faces' (the open and enclosed meshes),
      'hand_depth', 'init_bite', 'grasp_in_gripper' (get_grasp_pose_in_gripper_base()), 'finger_boxes',
      'grip_dirs' and 'finger_mesh_in_grasp' (see affordance.py);
      env: dict of 'cam_in_world', 'bin_in_world', 'ee_in_grasp' (inv(grasp_in_ee)), 'upper', 'lower';
      canonical: dict of 'canonical_grasps' (N,4,4), 'canonical_scores' (N,), 'canonical_cloud',
      'canonical_normals', 'canonical_affordance';
      symmetry_tfs (S,4,4); cfg_run: the sampler settings of config_run.yml;
      n_classes: len(cfg_grasp['classes']), default grasp_predicter.cfg['classes'];
      timings: an optional dict that accumulates each stage's wall time in ms, every stage ending in a device
      synchronise (the added synchronisations change no result); time spent by the caller between yields is not
      counted.

    It is ``compute_candidate_grasp_many`` on this one frame; see there for the synchronisations and the segmenter.
    """
    yield from compute_candidate_grasp_many([depth], [K], [bg_mask], [env], seg_predicter, nocs_predicter,
                                            grasp_predicter, gripper, canonical, symmetry_tfs, cfg_run,
                                            n_classes=n_classes, device=device, timings=timings)[0]


def compute_candidate_grasp_many(depths, Ks, bg_masks, envs, seg_predicter, nocs_predicter, grasp_predicter, gripper,
                                 canonical, symmetry_tfs, cfg_run, n_classes=None, device=None, timings=None):
    """compute_candidate_grasp for B frames: a list of B generators, generator b yielding what compute_candidate_grasp
    yields for (depths[b], Ks[b], bg_masks[b], envs[b]).  Frames may differ in size, intrinsics and depth dtype.

    The scene stages of all frames run once, at the first ``next()`` of any generator: back-projection into one flat
    buffer (one cg_depth2xyz_dev launch per frame) and the two masks, the normals (one many-set index), the
    segmentation, the label ranges, one segment table over all frames (segment_table_many), the visit orders and the
    1 mm scenes (one many-set index, its voxel means set-major).  Their synchronisations do not grow with B: the
    masks' per-frame counts and the two compactions, the normals' cell size and index build, the segmenter's own, one
    read of every frame's label range, one of all kept counts, one of all visit orders, offsets and segment bounds,
    and the 1 mm index build.  ``timings`` counts them once, under compute_candidate_grasp's stage names.  An error in
    them (a negative label, a CgError for a batch whose cell keys need more than 63 bits) is raised by every generator
    on its first ``next()``.

    The segmenter gets the non-empty frames through ``seg_predicter.predict_many`` (one list), or one ``predict`` per
    frame when it has no predict_many; its ``xyz_shifted`` is then the last non-empty frame's.

    Generator b draws its frame's colour ``randint``s at its own first ``next()``, then visits its objects exactly as
    compute_candidate_grasp does.  So, for a segmenter that draws no numpy random numbers (PointGroupPredictor draws
    none), consuming the generators one after another in any order leaves numpy's generator, and every yield, as a
    loop of compute_candidate_grasp calls in that order leaves them.  A frame with no non-background pixel yields
    nothing and draws nothing.  ValueError, before any device work, for an empty frame list, lists of different
    lengths, a depth that is not 2-D, a mask of another shape or a K without 9 entries."""
    depths, Ks, bg_masks, envs = list(depths), list(Ks), list(bg_masks), list(envs)
    B = len(depths)
    if B == 0:
        raise ValueError("compute_candidate_grasp_many: no frames")
    if not len(Ks) == len(bg_masks) == len(envs) == B:
        raise ValueError(f"compute_candidate_grasp_many: {B} depths, {len(Ks)} Ks, {len(bg_masks)} masks and "
                         f"{len(envs)} envs")
    for b in range(B):
        shape, mshape = tuple(np.shape(depths[b])), tuple(np.shape(bg_masks[b]))
        if len(shape) != 2 or mshape != shape or np.size(Ks[b]) != 9:
            raise ValueError(f"compute_candidate_grasp_many: frame {b} needs a 2-D depth, a mask of its shape and a "
                             f"3x3 K, got {shape}, {mshape} and {np.size(Ks[b])} entries")
    state = {}

    def scene():
        if "error" in state:
            raise state["error"]
        if "scene" not in state:
            try:
                state["scene"] = _scene_stages(depths, Ks, bg_masks, seg_predicter, grasp_predicter, gripper,
                                               canonical, cfg_run, n_classes, device, timings)
            except Exception as e:
                state["error"] = e
                raise
        return state["scene"]

    return [_frame_objects(b, scene, envs[b], nocs_predicter, grasp_predicter, gripper, canonical, symmetry_tfs,
                           cfg_run, timings) for b in range(B)]


def _scene_stages(depths, Ks, bg_masks, seg_predicter, grasp_predicter, gripper, canonical, cfg_run, n_classes, device,
                  timings):
    """The scene stages of compute_candidate_grasp_many, all frames at once: (common, frames), common the per-pick
    constants and frames[b] None for a frame with no non-background pixel, else a dict of its scene-stage results."""
    from . import cloud
    dev = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
    if n_classes is None:
        n_classes = len(grasp_predicter.cfg["classes"])
    canonical_poses = preselect_canonical(canonical["canonical_grasps"], canonical["canonical_scores"],
                                          cfg_run["nocs_grasp_sampler_score_larger_than"],
                                          cfg_run["nocs_grasp_sampler_max_n_grasp"])
    V = np.asarray(gripper["vertices"])
    common = {"dev": dev, "n_classes": n_classes, "canonical_poses": canonical_poses,
              "gripper_in_grasp": np.linalg.inv(np.asarray(gripper["grasp_in_gripper"], np.float64)),
              "gripper_diameter": np.linalg.norm(V.max(axis=0) - V.min(axis=0))}
    Ks = [np.asarray(K, np.float64).reshape(3, 3) for K in Ks]
    B = len(depths)
    t0 = None if timings is None else time.perf_counter()

    # :197-207 back-projection of every frame into its slice of one buffer, the scene and the no-background points
    ds = [d if isinstance(d, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(d)) for d in depths]
    pix = np.cumsum([0] + [d.shape[0] * d.shape[1] for d in ds])
    xyz = torch.empty((int(pix[-1]), 3), dtype=torch.float32, device=dev)
    for b, d in enumerate(ds):
        cloud.depth2xyzmap(d.to(dev), Ks[b], out=xyz[pix[b]:pix[b + 1]])
    in_scene = xyz[:, 2] >= 0.1
    fg = torch.cat([(m if isinstance(m, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(m))).to(dev)
                    .reshape(-1) == 0 for m in bg_masks])
    ends = torch.from_numpy(pix[1:] - 1).to(dev)
    counts = torch.stack([in_scene, fg]).to(torch.int64).cumsum(1)[:, ends].cpu().numpy()   # sync: frame sizes
    scene_off = np.concatenate([[0], counts[0]])
    pts_off = np.concatenate([[0], counts[1]])
    scene_all = xyz[in_scene]
    pts = xyz[fg]
    t0 = _lap(timings, "back-projection and masks", t0)
    live = [b for b in range(B) if pts_off[b + 1] > pts_off[b]]
    frames = [None] * B
    if not live:
        return common, frames
    # :208-213 normals, segmentation
    nrm = cloud.estimate_normals_many(pts, pts_off, 0.002, 30)
    t0 = _lap(timings, "normals", t0)
    datas = [{"cloud_xyz": pts[pts_off[b]:pts_off[b + 1]], "cloud_normal": nrm[pts_off[b]:pts_off[b + 1]]}
             for b in live]
    if hasattr(seg_predicter, "predict_many"):
        labels = list(seg_predicter.predict_many(datas))
    else:
        labels = [seg_predicter.predict(d) for d in datas]
    for j, lab in enumerate(labels):
        lab = (lab if isinstance(lab, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(lab))).to(dev)
        labels[j] = lab if lab.dtype in (torch.int32, torch.int64) else lab.to(torch.int64)
    t0 = _lap(timings, "segmentation", t0)
    ranges = torch.stack([torch.stack([lab.min(), lab.max()]).to(torch.int64) for lab in labels]).tolist()   # sync
    if any(lo < 0 for lo, _ in ranges):
        raise ValueError("compute_candidate_grasp: the segmenter returned a negative label")
    if len({lab.dtype for lab in labels}) > 1:
        labels = [lab.to(torch.int64) for lab in labels]
    n_labels = [hi + 1 for _, hi in ranges]
    loff = np.concatenate([[0], np.cumsum(n_labels)])
    table = segment_table_many(torch.cat(labels), pts, pts_off[[0] + [b + 1 for b in live]], n_labels)
    n_kept = table["n_kept"].tolist()                                                  # sync: the kept counts
    # sync: every kept frame's visit order, offsets and segment bounds, in one float64 read (the ints are exact)
    parts = []
    for j, nk in enumerate(n_kept):
        if nk:
            lo = int(loff[j])
            o = table["order"][lo:lo + nk]
            rows = o.to(torch.int64) + lo
            parts += [o.to(torch.float64), table["offsets"][lo + j:lo + j + nk + 1].to(torch.float64),
                      table["min"][rows].reshape(-1), table["max"][rows].reshape(-1)]
    head = torch.cat(parts).cpu().numpy() if parts else None
    t0 = _lap(timings, "segment table", t0)
    # :245-251 the 1 mm scenes of the frames with a kept segment, one many-set index
    kept = [b for j, b in enumerate(live) if n_kept[j]]
    with_pts = [b for b in kept if scene_off[b + 1] > scene_off[b]]
    scenes = {b: torch.zeros((0, 3), dtype=torch.float64, device=dev) for b in kept}
    if with_pts:
        ix = cloud.CloudIndex(torch.cat([scene_all[scene_off[b]:scene_off[b + 1]] for b in with_pts]), 0.001,
                              dev.index, set_offsets=np.cumsum([0] + [scene_off[b + 1] - scene_off[b] for b in with_pts]))
        means, _ = ix.voxel_means()
        for s, b in enumerate(with_pts):
            scenes[b] = means[ix.cell_offsets[s]:ix.cell_offsets[s + 1]]
        del ix
    _lap(timings, "1 mm scene", t0)

    at = 0
    for j, b in enumerate(live):
        nk = n_kept[j]
        f = {"n_kept": nk}
        if nk:
            order = head[at:at + nk].astype(np.int64)
            offsets = head[at + nk:at + 2 * nk + 1].astype(np.int64)
            lo_xyz = head[at + 2 * nk + 1:at + 5 * nk + 1].reshape(nk, 3)
            hi_xyz = head[at + 5 * nk + 1:at + 8 * nk + 1].reshape(nk, 3)
            at += 8 * nk + 1
            p0, p1 = int(pts_off[b]), int(pts_off[b + 1])
            f.update(K=Ks[b], pts=pts[p0:p1], nrm=nrm[p0:p1], index=table["index"][p0:p1], order=order,
                     offsets=offsets, lo_xyz=lo_xyz, hi_xyz=hi_xyz, scene_pts=scenes[b])
        frames[b] = f
    return common, frames


def _frame_objects(b, scene, env, nocs_predicter, grasp_predicter, gripper, canonical, symmetry_tfs, cfg_run, timings):
    """Generator b of compute_candidate_grasp_many: the shared scene stages (run by the first generator to start),
    frame b's colour draws, then its objects, largest first."""
    from . import cloud
    from .affordance import compute_grasp_affordance
    from .grasp_sampler import cone_grasp_poses
    common, frames = scene()
    f = frames[b]
    if f is None:
        return
    for _ in range(f["n_kept"]):                                                      # :237, one draw per inlier
        np.random.randint(0, 255, size=(3))
    if f["n_kept"] == 0:                                                              # :261-263
        return
    dev, n_classes, canonical_poses = common["dev"], common["n_classes"], common["canonical_poses"]
    gripper_in_grasp, gripper_diameter = common["gripper_in_grasp"], common["gripper_diameter"]
    K, pts, nrm, scene_pts = f["K"], f["pts"], f["nrm"], f["scene_pts"]
    order, offsets, lo_xyz, hi_xyz = f["order"], f["offsets"], f["lo_xyz"], f["hi_xyz"]
    np_dtype = np.float32 if pts.dtype == torch.float32 else np.float64

    for k, seg_id in enumerate(order.tolist()):                                        # :266
        t0 = None if timings is None else time.perf_counter()
        idx = f["index"][int(offsets[k]):int(offsets[k + 1])].to(torch.int64)
        ob_pts, ob_normals = pts[idx], nrm[idx]                                        # :273-275
        prep = cloud.prepare_object(ob_pts, ob_normals, scene_pts, gripper_diameter, octo_resolution=0.001, K=K)
        t0 = _lap(timings, "prepare_object", t0)
        if prep is None:                                                               # :116-118
            continue
        data = {key: v.cpu().numpy() for key, v in prep["data"].items()}
        background_pts = prep["background_pts"]
        nocs_cloud, nocs_pose = nocs_predicter.predict(copy.deepcopy(data))            # :146
        t0 = _lap(timings, "NUNOCS", t0)
        if nocs_pose is None:
            continue
        R, t = nocs_pose[:3, :3], nocs_pose[:3, 3]
        data["nocs_transformed"] = np.asarray(nocs_cloud, np.float64) @ R.T + t          # :154-157
        observed_center = (hi_xyz[k].astype(np_dtype) + lo_xyz[k].astype(np_dtype)) / 2     # :152, cloud dtype
        nocs_in_world = np.asarray(env["cam_in_world"]) @ nocs_pose
        if (np.linalg.norm(observed_center - nocs_pose[:3, 3]) >= 0.05
                or nocs_in_world[2, 3] < np.asarray(env["bin_in_world"])[2, 3]):      # :165-168
            continue
        # :176 CombinedGraspSampler: the cone sampler's survivors, then the canonical transfer's
        _, cone32 = cone_grasp_poses(prep["points_for_sample"].cpu().numpy(), prep["normals_for_sample"].cpu().numpy(),
                                     gripper["hand_depth"], gripper["init_bite"], max_num_samples=np.inf,
                                     n_sphere_dir=cfg_run["cone_grasp_smapler_n_sphere_dir"],
                                     approach_step=cfg_run["cone_grasp_smapler_approach_step"],
                                     center_ob_between_gripper=True, device=dev.index)
        cone = _filter(cone32, [np.eye(4)], np.eye(4), gripper_in_grasp, ob_pts, background_pts, gripper, env)
        transfer = _filter(canonical_poses, symmetry_tfs, nocs_pose, gripper_in_grasp, ob_pts, background_pts,
                           gripper, env)
        grasp_poses = torch.cat([cone, transfer]).cpu().numpy()
        t0 = _lap(timings, "samplers and filters", t0)
        # :180-181 affordance (:73-107), dropping the grasps without a contact patch
        can_cloud = np.asarray(canonical["canonical_cloud"], np.float64) @ R.T + t
        can_nrm = np.asarray(canonical["canonical_normals"], np.float64) @ R.T
        can_pts_down, can_nrm_down = cloud.voxel_down_sample(can_cloud, 0.002, normals=can_nrm)
        p_T_given_G, _ = compute_grasp_affordance(grasp_poses, gripper["finger_mesh_in_grasp"], can_pts_down,
                                                  can_nrm_down, can_cloud, canonical["canonical_affordance"],
                                                  gripper["finger_boxes"], gripper["grip_dirs"], device=dev.index)
        keep = np.isfinite(p_T_given_G)
        grasp_poses, p_T_given_G = grasp_poses[keep], p_T_given_G[keep]
        t0 = _lap(timings, "affordance", t0)
        if len(grasp_poses) == 0:                                                      # :277-278
            continue
        # :310-328 grasp-Q, p_G, p_T_G and the ranking
        ret = grasp_predicter.predict_batch(data, list(grasp_poses))
        pred = np.stack([r[2] for r in ret])
        pred_label = np.array([r[0] for r in ret])
        t0 = _lap(timings, "grasp-Q", t0)
        p_G, p_T_G, perm = rank_grasps(torch.from_numpy(pred).to(dev), torch.from_numpy(p_T_given_G).to(dev),
                                       n_classes)
        p_G, p_T_G, perm = p_G.cpu().numpy(), p_T_G.cpu().numpy(), perm.cpu().numpy()
        _lap(timings, "ranking", t0)
        yield {"seg_id": int(seg_id), "ob_pts": ob_pts, "data": data, "nocs_pose": nocs_pose,
               "grasp_poses": grasp_poses[perm], "pred_label": pred_label[perm], "pred": pred[perm],
               "p_T_given_G": p_T_given_G[perm], "p_G": p_G[perm], "p_T_G": p_T_G[perm]}
