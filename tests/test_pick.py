"""compute_candidate_grasp against a straight-line composition of the package's public per-stage calls, written here in
the reference's order (run_grasp_simulation.py:188-329): the objects and their order, each object's grasp poses,
p_T_given_G, pred, p_G, p_T_G and the ranking bit for bit, and numpy's generator state after every yield.

The scene is a rendered pile at 0.1 mm per pixel, shaped so that named objects take each branch of the per-object
loop, and the test asserts the whole map of object to branch:
- "small": the segmenter stand-in returns the renderer's id map plus one extra segment carved out of object 0, a
  compact patch of 520 pixels on one face that covers fewer than 100 voxels of 0.5 mm;
- "nocs": object SUNK is pushed 0.2 m deeper, below the bin floor, so its NUNOCS pose fails the bin check;
- "no_grasp": the floor around object WELL is raised 1 cm above its top, so the object sits in a well whose rim
  every gripper pose collides with and both samplers come back empty;
- "accepted": the objects that keep grasps, compared bit for bit."""
import copy

import numpy as np
import pytest
import torch

from catgrasp_b200 import synthetic

pytestmark = pytest.mark.gpu

N_OBJ = 12
SUNK, WELL = 1, 2
# object -> branch on this fixture; "small" is the carved patch (label N_OBJ)
EXPECTED = {0: "no_grasp", 1: "nocs", 2: "no_grasp", 3: "no_grasp", 4: "no_grasp", 5: "no_grasp", 6: "no_grasp",
            7: "no_grasp", 8: "accepted", 9: "no_grasp", 10: "no_grasp", 11: "no_grasp", 12: "small"}
H = W = 1000
K = np.array([[6773.3, 0, 500.0], [0, 6772.5, 500.0], [0, 0, 1]])
IK_UPPER = np.deg2rad([170, 120, 170, 120, 170, 120, 175])
N_CLASSES = 11
CFG_RUN = {"nocs_grasp_sampler_score_larger_than": 0.5, "nocs_grasp_sampler_max_n_grasp": 40,
           "cone_grasp_smapler_n_sphere_dir": 8, "cone_grasp_smapler_approach_step": 0.002}


class IdSegmenter:
    """A segmenter stand-in: the labels of the no-background points, fixed in advance."""

    def __init__(self, labels):
        self.labels = labels

    def predict(self, data):
        assert data["cloud_xyz"].shape[0] == len(self.labels)
        return self.labels.copy()


def _gripper():
    g = synthetic.make_gripper_proxy()
    box = [0.0, 0.045, -0.010, 0.010]
    return {"vertices": g["open"]["V"], "faces": g["open"]["F"], "enclosed_vertices": g["enclosed"]["V"],
            "enclosed_faces": g["enclosed"]["F"], "hand_depth": 0.012, "init_bite": 0.002,
            "grasp_in_gripper": np.linalg.inv(g["gripper_in_grasp"]), "finger_boxes": np.array([box, box]),
            "grip_dirs": np.array([[0, -1, 0], [0, 1, 0]]), "finger_mesh_in_grasp": g["gripper_in_grasp"]}


def _canonical():
    """A synthetic canonical set in NOCS coordinates: hex-nut samples normalised to the unit cube, grasps on them and a
    smooth affordance."""
    rng = np.random.RandomState(31)
    pts, nrm = synthetic.sample_hex_nut(3000, rng)
    lo = pts.min(0)
    s = (pts.max(0) - lo).max()
    cloud = (pts - lo) / s
    poses = synthetic.make_candidates(pts, nrm, 80, seed=32)
    poses[:, :3, 3] = (poses[:, :3, 3] - lo) / s
    return {"canonical_grasps": poses, "canonical_scores": rng.uniform(0, 1, 80), "canonical_cloud": cloud,
            "canonical_normals": nrm, "canonical_affordance": np.clip(0.5 + 0.5 * np.sin(40 * pts[:, 0]), 0, 1)}


def _scene(shaped):
    from catgrasp_b200 import cloud
    depth, ids = synthetic.render_depth(K, H, W, n_objects=N_OBJ, seed=40)
    bg = ids < 0
    if shaped:
        from scipy.ndimage import distance_transform_edt
        depth = depth.copy()
        depth[ids == SUNK] += np.float32(0.2)
        rim = bg & (distance_transform_edt(ids != WELL) < 150)     # floor within 15 mm of the object
        depth[rim] = depth[ids == WELL].min() - np.float32(0.01)
    xyz_map = cloud.depth2xyzmap(depth, K)
    # the small segment: the 520 pixels of object 0 nearest its flattest pixel (the least depth range over a 7 x 7
    # window), a patch of one face that covers fewer than 100 voxels of 0.5 mm
    vv, uu = np.nonzero(ids == 0)
    pad = np.pad(np.where(ids == 0, depth, np.inf), 3, constant_values=np.inf)
    win = np.stack([pad[3 + dv + vv, 3 + du + uu] for dv in range(-3, 4) for du in range(-3, 4)])
    c = int(np.argmin(np.where(np.isfinite(win).all(0), win.max(0) - win.min(0), np.inf)))
    d2 = (vv - vv[c]) ** 2 + (uu - uu[c]) ** 2
    patch = np.argsort(d2, kind="stable")[:520]
    img = ids.astype(np.int64).copy()
    img[vv[patch], uu[patch]] = N_OBJ
    labels = img[~bg].reshape(-1)
    cam_in_world = np.eye(4)
    cam_in_world[:3, :3] = np.diag([1.0, -1.0, -1.0])          # the camera looks down at the bin
    cam_in_world[:3, 3] = [0.6, 0.0, 0.85]
    ee_in_grasp = np.eye(4)
    ee_in_grasp[:3, :3] = np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], float).T
    ee_in_grasp[:3, 3] = [-0.17, 0, 0]
    bin_in_world = np.eye(4)
    bin_in_world[2, 3] = 0.85 - 0.75                           # the bin floor lies below the pile
    env = {"cam_in_world": cam_in_world, "bin_in_world": bin_in_world, "ee_in_grasp": ee_in_grasp,
           "upper": IK_UPPER, "lower": -IK_UPPER}
    return {"depth": depth, "bg": bg, "labels": labels, "env": env, "gripper": _gripper(),
            "canonical": _canonical()}


@pytest.fixture(scope="module")
def scene():
    return _scene(True)


@pytest.fixture(scope="module")
def plain_scene():
    return _scene(False)


@pytest.fixture(scope="module")
def predicters(tmp_path_factory):
    from catgrasp_b200.predicter import GraspPredicter, NunocsPredicter
    tmp = tmp_path_factory.mktemp("pick-artifacts")
    gd = synthetic.write_artifacts(str(tmp / "cls"), "cls", 256, seed=3, logit_gain=12.0)
    gp = GraspPredicter("nut", artifact_dir=gd, device=0)
    nd = synthetic.write_artifacts(str(tmp / "seg"), "seg", 2048, with_normalizer=False,
                                   state_dict=synthetic.make_lattice_seg_state_dict(seed=5))
    npd = NunocsPredicter("nut", artifact_dir=nd, device=0)
    return gp, npd


def straight_line(sc, seg, nocs_predicter, grasp_predicter):
    """The reference's compute_candidate_grasp, stage by stage with the package's public calls.  Yields
    (seg_id, branch, result) for every object, branch one of 'small', 'nocs', 'no_grasp', 'accepted'."""
    from catgrasp_b200 import cloud, my_cpp
    from catgrasp_b200.affordance import compute_grasp_affordance
    from catgrasp_b200.grasp_sampler import cone_grasp_poses
    from oracle import pick_ref
    g, env, can = sc["gripper"], sc["env"], sc["canonical"]
    xyz_map = cloud.depth2xyzmap(sc["depth"], K)
    scene_pts = xyz_map[xyz_map[:, :, 2] >= 0.1].reshape(-1, 3)
    pts = xyz_map[sc["bg"] == 0].reshape(-1, 3)
    nrm = cloud.estimate_normals(pts, 0.002, 30)
    scene_seg = seg.predict({"cloud_xyz": pts, "cloud_normal": nrm})
    t = pick_ref.segment_table(scene_seg, pts)
    for _ in t["inlier_ids"]:
        np.random.randint(0, 255, size=(3))
    scene_pts = cloud.voxel_down_sample(scene_pts, 0.001)
    V = g["vertices"]
    diameter = np.linalg.norm(V.max(axis=0) - V.min(axis=0))
    gig = np.linalg.inv(g["grasp_in_gripper"])
    # NocsTransferGraspSampler.__init__ (grasp_sampler.py:330-345): the score threshold, then a stable sort by
    # descending score cut to max_n_grasp
    scores = np.asarray(can["canonical_scores"], np.float64)
    sel = list(range(len(scores)))
    if CFG_RUN["nocs_grasp_sampler_score_larger_than"] > 0:
        sel = [i for i in sel if scores[i] >= CFG_RUN["nocs_grasp_sampler_score_larger_than"]]
    sel.sort(key=lambda i: -scores[i])
    canonical_poses = np.asarray(can["canonical_grasps"], np.float64)[sel[:CFG_RUN["nocs_grasp_sampler_max_n_grasp"]]]
    for seg_id in t["order"]:
        ob_pts = pts[t["labels"] == seg_id]
        ob_normals = nrm[t["labels"] == seg_id]
        prep = cloud.prepare_object(ob_pts, ob_normals, scene_pts, diameter, 0.001, K)
        if prep is None:
            yield seg_id, "small", None
            continue
        data = prep["data"]
        nocs_cloud, nocs_pose = nocs_predicter.predict(copy.deepcopy(data))
        if nocs_pose is None:
            yield seg_id, "nocs", None
            continue
        observed_center = (ob_pts.max(axis=0) + ob_pts.min(axis=0)) / 2
        nocs_in_world = env["cam_in_world"] @ nocs_pose
        if np.linalg.norm(observed_center - nocs_pose[:3, 3]) >= 0.05 or nocs_in_world[2, 3] < env["bin_in_world"][2, 3]:
            yield seg_id, "nocs", None
            continue
        _, cone32 = cone_grasp_poses(prep["points_for_sample"], prep["normals_for_sample"], g["hand_depth"],
                                     g["init_bite"], np.inf, CFG_RUN["cone_grasp_smapler_n_sphere_dir"],
                                     CFG_RUN["cone_grasp_smapler_approach_step"], True)
        args = (env["cam_in_world"], env["ee_in_grasp"], gig, True, True, True, env["upper"], env["lower"],
                g["vertices"], g["faces"], g["enclosed_vertices"], g["enclosed_faces"], ob_pts,
                prep["background_pts"], 0.0005, False)
        poses = my_cpp.filterGraspPose(cone32.cpu().numpy(), [np.eye(4)], np.eye(4), np.eye(4), *args)
        poses += my_cpp.filterGraspPose(list(canonical_poses), [np.eye(4)], nocs_pose, np.eye(4), *args)
        poses = np.array(poses, np.float32).reshape(-1, 4, 4)
        if len(poses) == 0:
            yield seg_id, "no_grasp", "filters"
            continue
        R, tt = nocs_pose[:3, :3], nocs_pose[:3, 3]
        can_cloud = can["canonical_cloud"] @ R.T + tt
        down, down_n = cloud.voxel_down_sample(can_cloud, 0.002, normals=can["canonical_normals"] @ R.T)
        p, _ = compute_grasp_affordance(poses, g["finger_mesh_in_grasp"], down, down_n, can_cloud,
                                        can["canonical_affordance"], g["finger_boxes"], g["grip_dirs"])
        keep = np.isfinite(p)
        poses, p = poses[keep], p[keep]
        if len(poses) == 0:
            yield seg_id, "no_grasp", "affordance"
            continue
        ret = grasp_predicter.predict_batch(data, list(poses))
        pred = np.stack([r[2] for r in ret])
        p_G = np.array([(pr * np.arange(len(pr))).sum() / (N_CLASSES - 1) for pr in pred])
        p_T_G = np.array([p[i] * p_G[i] for i in range(len(p))])
        order = sorted(range(len(p)), key=lambda i: -p_T_G[i])
        yield seg_id, "accepted", {"grasp_poses": poses[order], "pred": pred[order], "p_T_given_G": p[order],
                                   "p_G": p_G[order], "p_T_G": p_T_G[order],
                                   "pred_label": np.array([ret[i][0] for i in order])}


class RecordingNunocs:
    """The NUNOCS predicter, recording for every call the numpy generator's state and the object cloud it gets."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def predict(self, data):
        st = np.random.get_state()
        self.calls.append((st[1].tobytes(), int(st[2]), np.asarray(data["cloud_xyz"]).tobytes()))
        return self.inner.predict(data)


def _run_pipeline(sc, seg, npd, gp, **kw):
    from catgrasp_b200.pick import compute_candidate_grasp
    out = []
    for r in compute_candidate_grasp(sc["depth"], K, sc["bg"], seg, npd, gp, sc["gripper"], sc["env"],
                                     sc["canonical"], [np.eye(4)], CFG_RUN, n_classes=N_CLASSES, **kw):
        out.append((r, np.random.get_state()))
    return out


def _compare(got, want):
    assert [r["seg_id"] for r, _ in got] == [w[0] for w in want]
    for (r, st), (_, _, w, wst) in zip(got, want):
        for key in ("grasp_poses", "pred", "p_T_given_G", "p_G", "p_T_G", "pred_label"):
            a, b = np.asarray(r[key]), np.asarray(w[key])
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), key
        assert np.array_equal(st[1], wst[1]) and st[2] == wst[2]


def _straight(sc, seg, npd, gp):
    out = []
    for seg_id, branch, res in straight_line(sc, seg, npd, gp):
        if branch == "accepted":
            out.append((seg_id, branch, res, np.random.get_state()))
    return out


def test_pick_matches_straight_line(scene, predicters):
    gp, npd = predicters
    seg = IdSegmenter(scene["labels"])
    rec_got, rec_want = RecordingNunocs(npd), RecordingNunocs(npd)
    np.random.seed(7)
    got = _run_pipeline(scene, seg, rec_got, gp)
    np.random.seed(7)
    branches, detail, want = {}, {}, []
    for seg_id, branch, res in straight_line(scene, seg, rec_want, gp):
        branches[seg_id] = branch
        if branch == "accepted":
            want.append((seg_id, branch, res, np.random.get_state()))
        elif branch == "no_grasp":
            detail[seg_id] = res
    print("branches:", branches, detail)
    _compare(got, want)
    assert rec_got.calls == rec_want.calls          # the same objects reach NUNOCS, with the same RNG state
    assert branches == EXPECTED
    assert branches[N_OBJ] == "small" and branches[SUNK] == "nocs" and branches[WELL] == "no_grasp"
    assert detail[WELL] == "filters"                 # both samplers came back empty
    assert "accepted" in branches.values()


def test_pick_with_pointgroup(plain_scene, predicters, tmp_path):
    """The wiring through the real segmentation network (synthetic weights) on the pile without the shaped objects:
    CUDA tensors in, the same objects out as the composition on numpy, and the same objects handed to NUNOCS with the
    same generator state."""
    import json
    import os
    import yaml
    from catgrasp_b200.predicter import PointGroupPredictor
    from oracle import pointgroup_ref as PR
    gp, npd = predicters
    PG = np.load(os.path.join(os.path.dirname(__file__), "golden", "pointgroup.npz"))
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": int(PG["m"]), "block_residual": True, "block_reps": int(PG["block_reps"]),
                         "use_coords": True}, "GROUP": {"prepare_epochs": 999999}}
    (tmp_path / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    sd = PR.synthetic_state_dict([(k, tuple(s)) for k, s in json.loads(str(PG["key_shapes"]))], int(PG["seed"]))
    torch.save({"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}},
               str(tmp_path / "best_val.pth.tar"))
    pg = PointGroupPredictor("nut", artifact_dir=str(tmp_path), device=0)
    rec_got, rec_want = RecordingNunocs(npd), RecordingNunocs(npd)
    np.random.seed(8)
    got = _run_pipeline(plain_scene, pg, rec_got, gp)
    np.random.seed(8)
    want = _straight(plain_scene, pg, rec_want, gp)
    print("pointgroup: objects at NUNOCS", len(rec_want.calls), "yielded", len(want))
    assert len(rec_want.calls) >= 1 and rec_got.calls == rec_want.calls
    _compare(got, want)
