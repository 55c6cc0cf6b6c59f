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
    """
    from . import cloud
    from .affordance import compute_grasp_affordance
    from .grasp_sampler import cone_grasp_poses
    dev = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
    if n_classes is None:
        n_classes = len(grasp_predicter.cfg["classes"])
    canonical_poses = preselect_canonical(canonical["canonical_grasps"], canonical["canonical_scores"],
                                          cfg_run["nocs_grasp_sampler_score_larger_than"],
                                          cfg_run["nocs_grasp_sampler_max_n_grasp"])
    gripper_in_grasp = np.linalg.inv(np.asarray(gripper["grasp_in_gripper"], np.float64))
    V = np.asarray(gripper["vertices"])
    gripper_diameter = np.linalg.norm(V.max(axis=0) - V.min(axis=0))
    K = np.asarray(K, np.float64).reshape(3, 3)
    t0 = None if timings is None else time.perf_counter()

    # :197-207 back-projection, the scene and the no-background points
    d = depth if isinstance(depth, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(depth))
    xyz_map = cloud.depth2xyzmap(d.to(dev), K)
    scene_pts = xyz_map[xyz_map[:, :, 2] >= 0.1].reshape(-1, 3)
    bg = bg_mask if isinstance(bg_mask, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(bg_mask))
    pts = xyz_map[bg.to(dev) == 0].reshape(-1, 3)
    t0 = _lap(timings, "back-projection and masks", t0)
    if pts.shape[0] == 0:
        return
    # :208-213 normals, segmentation
    nrm = cloud.estimate_normals(pts, 0.002, 30)
    t0 = _lap(timings, "normals", t0)
    labels = seg_predicter.predict({"cloud_xyz": pts, "cloud_normal": nrm})
    labels = labels if isinstance(labels, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(labels))
    labels = labels.to(dev)
    if labels.dtype not in (torch.int32, torch.int64):
        labels = labels.to(torch.int64)
    t0 = _lap(timings, "segmentation", t0)
    lo, hi = torch.stack([labels.min(), labels.max()]).to(torch.int64).tolist()      # sync: the table's size
    if lo < 0:
        raise ValueError("compute_candidate_grasp: the segmenter returned a negative label")
    table = segment_table(labels, pts, hi + 1)
    n_kept = int(table["n_kept"].item())                                              # sync: the kept count
    for _ in range(n_kept):                                                           # :237, one draw per inlier
        np.random.randint(0, 255, size=(3))
    if n_kept == 0:                                                                   # :261-263
        return
    head = torch.cat([table["order"][:n_kept], table["offsets"][:n_kept + 1]]).cpu().numpy()   # sync: the visit order
    order, offsets = head[:n_kept], head[n_kept:]
    lo_xyz = table["min"][torch.from_numpy(order.astype(np.int64)).to(dev)].cpu().numpy()
    hi_xyz = table["max"][torch.from_numpy(order.astype(np.int64)).to(dev)].cpu().numpy()
    t0 = _lap(timings, "segment table", t0)
    # :245-251 the 1 mm scene
    scene_pts = cloud.voxel_down_sample(scene_pts, 0.001)
    _lap(timings, "1 mm scene", t0)
    np_dtype = np.float32 if pts.dtype == torch.float32 else np.float64

    for k, seg_id in enumerate(order.tolist()):                                        # :266
        t0 = None if timings is None else time.perf_counter()
        idx = table["index"][int(offsets[k]):int(offsets[k + 1])].to(torch.int64)
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
