"""The per-pick kernels (csrc/cg_pick.cu) against oracle/pick_ref.py, and the device paths of PointGroupPredictor's
front and cloud.prepare_object against their numpy results."""
import os

import numpy as np
import pytest
import torch

from oracle import pick_ref

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pick_control.npz"))


def _table(labels, xyz, L=None):
    from catgrasp_b200 import pick
    lab = torch.from_numpy(labels).cuda()
    x = torch.from_numpy(xyz).cuda()
    t = pick.segment_table(lab, x, int(labels.max()) + 1 if L is None else L)
    return {k: v.cpu().numpy() for k, v in t.items()}


def _check_table(labels, xyz):
    ref = pick_ref.segment_table(labels, xyz)
    got = _table(labels, xyz)
    L = len(ref["count"])
    assert np.array_equal(got["labels"], ref["labels"]) and got["labels"].dtype == labels.dtype
    assert np.array_equal(got["count"], ref["count"])
    assert np.array_equal(got["inlier"].astype(bool), ref["inlier"])
    present = ref["count"] > 0
    assert np.array_equal(got["min"][present], ref["min"][present].astype(np.float64))
    assert np.array_equal(got["max"][present], ref["max"][present].astype(np.float64))
    n = int(got["n_kept"][0])
    assert n == len(ref["order"]) == len(ref["inlier_ids"])
    assert got["order"][:n].tolist() == ref["order"] and (got["order"][n:] == -1).all()
    off = got["offsets"]
    assert off[0] == 0 and len(off) == L + 1 and (off[n:] == off[n]).all()
    for k, idx in enumerate(ref["indices"]):
        assert np.array_equal(got["index"][off[k]:off[k + 1]], idx)
    return ref


@pytest.mark.parametrize("name", ("mixed", "equal", "none"))
@pytest.mark.parametrize("ltype", (np.int32, np.int64))
@pytest.mark.parametrize("xtype", (np.float32, np.float64))
def test_segment_table_golden(name, ltype, xtype):
    labels = G[f"{name}_labels"].astype(ltype)
    xyz = G[f"{name}_cloud_xyz"].astype(xtype)
    ref = _check_table(labels, xyz)
    if xtype == np.float32:
        assert ref["order"] == G[f"{name}_visits"].tolist()


@pytest.mark.parametrize("M, L, seed", [(1, 1, 0), (5000, 7, 1), (200_000, 300, 2), (1 << 21, 40, 3),
                                        (1 << 20, 600, 4), (300_000, 2000, 5)])
@pytest.mark.parametrize("xtype", (np.float32, np.float64))
def test_segment_table_random(M, L, seed, xtype):
    # L <= 512 runs the shared-memory statistics kernel, larger tables the global one
    rng = np.random.RandomState(seed)
    w = rng.uniform(0.2, 3, L)
    labels = rng.choice(L, M, p=w / w.sum()).astype(np.int64)
    labels[:L] = np.arange(L)                                   # dense in [0, L)
    centre = rng.uniform(-0.1, 0.1, (L, 3))[labels]
    size = rng.uniform(0.001, 0.2, (L, 3))[labels]
    xyz = (centre + size * rng.uniform(-0.5, 0.5, (M, 3))).astype(xtype)
    _check_table(labels, xyz)


def test_segment_table_equal_counts():
    L, n = 64, 600
    labels = np.repeat(np.arange(L), n)[np.random.RandomState(9).permutation(L * n)]
    xyz = np.random.RandomState(10).uniform(0, 0.01, (L * n, 3)).astype(np.float32)
    ref = _check_table(labels, xyz)
    assert ref["order"] == list(range(L - 1, -1, -1))


def _softmax_rows(rng, G, C, scale=30.0):
    z = rng.normal(0, scale, (G, C))
    e = np.exp(z - z.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def _check_rank(probs, p_t, n_classes):
    from catgrasp_b200 import pick
    p_G, p_T_G, perm = pick.rank_grasps(torch.from_numpy(probs).cuda(), torch.from_numpy(p_t).cuda(), n_classes)
    rg, rt, rp = pick_ref.rank_grasps(probs, p_t, n_classes)
    assert np.array_equal(p_G.cpu().numpy().view(np.uint64), rg.view(np.uint64))
    assert np.array_equal(p_T_G.cpu().numpy().view(np.uint64), rt.view(np.uint64))
    assert np.array_equal(perm.cpu().numpy(), rp)


@pytest.mark.parametrize("C, n_classes", [(10, 11), (5, 6), (10, 10)])
@pytest.mark.parametrize("G_", [0, 1, 7, 70_000])
def test_rank_wide_rows_ties_and_zeros(C, n_classes, G_):
    rng = np.random.RandomState(G_ + C)
    probs = _softmax_rows(rng, G_, C)
    if G_ >= 7:
        probs[1::7] = probs[0::7][:len(probs[1::7])]                            # repeated rows: equal p_G
    p_t = rng.uniform(0, 1, G_)
    if G_ >= 7:
        p_t[rng.choice(G_, G_ // 3, replace=False)] = 0.5                       # exact ties
        z = rng.choice(G_, max(2, G_ // 5), replace=False)
        p_t[z] = np.where(np.arange(len(z)) % 2, 0.0, -0.0)                     # zeros of both signs
    _check_rank(probs, p_t, n_classes)


def test_rank_golden():
    from catgrasp_b200 import pick
    for name in ("mixed", "equal"):
        for k in range(int(G[f"{name}_n_yield"])):
            p_G, p_T_G, perm = pick.rank_grasps(torch.from_numpy(G[f"{name}_probs_{k}"]).cuda(),
                                                torch.from_numpy(G[f"{name}_p_T_given_G_{k}"]).cuda(),
                                                int(G["n_classes"]))
            perm = perm.cpu().numpy()
            assert np.array_equal(perm, G[f"{name}_order_{k}"])
            assert np.array_equal(p_G.cpu().numpy()[perm].view(np.uint64), G[f"{name}_p_G_{k}"].view(np.uint64))
            assert np.array_equal(p_T_G.cpu().numpy()[perm].view(np.uint64), G[f"{name}_p_T_G_{k}"].view(np.uint64))


def test_entries_do_not_synchronise():
    from catgrasp_b200 import pick
    rng = np.random.RandomState(3)
    lab = torch.from_numpy(rng.randint(0, 20, 100_000)).cuda()
    x = torch.from_numpy(rng.uniform(0, 0.05, (100_000, 3))).cuda()
    probs = torch.from_numpy(_softmax_rows(rng, 5000, 10)).cuda()
    p_t = torch.from_numpy(rng.uniform(0, 1, 5000)).cuda()
    pick.segment_table(lab, x, 20)            # workspaces sized before the checked calls
    pick.rank_grasps(probs, p_t, 11)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t = pick.segment_table(lab, x, 20)
        r = pick.rank_grasps(probs, p_t, 11)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(t["n_kept"][0]) >= 1 and r[2].shape == (5000,)


def test_bad_arguments_raise():
    from catgrasp_b200 import _lib, pick
    with pytest.raises(ValueError):
        pick.segment_table(torch.zeros(5, dtype=torch.int64).cuda(), torch.zeros(4, 3).cuda(), 1)
    with pytest.raises(_lib.CgError):
        pick.rank_grasps(torch.zeros(3, 200).cuda(), torch.zeros(3, dtype=torch.float64).cuda(), 201)


# --------------------------------------------------------------------- PointGroup's front and prepare_object on tensors
PG = np.load(os.path.join(os.path.dirname(__file__), "golden", "pointgroup.npz"))


@pytest.fixture(scope="module")
def artifact_dir(tmp_path_factory):
    import json
    import yaml
    from oracle import pointgroup_ref as PR
    d = tmp_path_factory.mktemp("artifacts-pg-pick")
    m, reps = int(PG["m"]), int(PG["block_reps"])
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": m, "block_residual": True, "block_reps": reps, "use_coords": True},
           "GROUP": {"prepare_epochs": 999999}}
    (d / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    shapes = [(k, tuple(s)) for k, s in json.loads(str(PG["key_shapes"]))]
    sd = PR.synthetic_state_dict(shapes, int(PG["seed"]))
    torch.save({"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}},
               str(d / "best_val.pth.tar"))
    return str(d)


@pytest.mark.parametrize("cls", ("hnm", "nut", "screw"))
def test_device_front_on_tensors(cls, artifact_dir):
    from catgrasp_b200.predicter import PointGroupPredictor
    from oracle import pointgroup_ref as PR
    p = PointGroupPredictor(cls, artifact_dir=artifact_dir, device=0)
    xyz, nrm = PG[f"{cls}_cloud_xyz"], PG[f"{cls}_cloud_normal"]
    xo, locs, feats, shape = p.device_front({"cloud_xyz": torch.from_numpy(xyz).cuda(),
                                             "cloud_normal": torch.from_numpy(nrm).cuda()})
    rxo, rlocs, rfeats, rshape = PR.host_front(xyz, nrm)
    assert np.array_equal(xo.cpu().numpy(), rxo) and np.array_equal(locs.cpu().numpy(), rlocs)
    assert np.array_equal(feats.cpu().numpy().view(np.uint32), rfeats.view(np.uint32))
    assert tuple(shape) == tuple(rshape)
    labels_np = p.predict({"cloud_xyz": xyz.copy(), "cloud_normal": nrm.copy()})
    labels_t = p.predict({"cloud_xyz": torch.from_numpy(xyz).cuda(), "cloud_normal": torch.from_numpy(nrm).cuda()})
    assert isinstance(labels_t, torch.Tensor) and labels_t.is_cuda and isinstance(p.xyz_shifted, torch.Tensor)
    assert np.array_equal(labels_t.cpu().numpy(), labels_np) and np.array_equal(labels_np, PG[f"{cls}_labels_all"])


def _order_sensitive_xs(xmin, count):
    """float32 x > xmin where trunc(fl(fl(x * 500) - fl(xmin * 500))) differs from trunc(fl(fl(x - xmin) * 500))."""
    f, out = np.float32, []
    for k in range(1, 400):
        x = f(xmin + f(k) / f(500))
        for _ in range(40):
            x = np.nextafter(x, f(-1))
        for _ in range(80):
            if int(f(f(x * f(500)) - f(xmin * f(500)))) != int(f(f(x - xmin) * f(500))):
                out.append(x)
                break
            x = np.nextafter(x, f(1))
        if len(out) == count:
            return np.array(out, np.float32)
    raise AssertionError("no order-sensitive coordinates found")


def test_device_front_order_sensitive_x(artifact_dir):
    from catgrasp_b200.predicter import PointGroupPredictor
    from oracle import pointgroup_ref as PR
    xmin = np.float32(0.0123457)
    xs = np.concatenate([[xmin], _order_sensitive_xs(xmin, 6)]).astype(np.float32)
    xyz = np.stack([xs, np.arange(len(xs), dtype=np.float32) * np.float32(0.002),
                    np.full(len(xs), 0.7, np.float32)], 1)
    nrm = np.tile(np.float32([0, 0, 1]), (len(xs), 1))
    p = PointGroupPredictor("nut", artifact_dir=artifact_dir, device=0)
    xo, locs, _, shape = p.device_front({"cloud_xyz": torch.from_numpy(xyz).cuda(),
                                         "cloud_normal": torch.from_numpy(nrm).cuda()})
    rxo, rlocs, _, rshape = PR.host_front(xyz, nrm)
    assert np.array_equal(xo.cpu().numpy(), rxo) and np.array_equal(locs.cpu().numpy(), rlocs)
    assert tuple(shape) == tuple(rshape)


@pytest.mark.parametrize("dtype", (np.float32, np.float64))
def test_prepare_object_on_tensors(dtype):
    from catgrasp_b200 import cloud, synthetic
    K = np.array([[2257.75 / 3, 0, 1032 / 3], [0, 2257.49 / 3, 772 / 3], [0, 0, 1]])
    depth, ids = synthetic.render_depth(K, 1544 // 3, 2064 // 3, n_objects=6, seed=5)
    xyz_map = cloud.depth2xyzmap(depth, K)
    scene = cloud.voxel_down_sample(xyz_map[xyz_map[:, :, 2] >= 0.1].reshape(-1, 3), 0.001)
    ob = int(np.bincount(ids[ids >= 0]).argmax())
    ob_pts = xyz_map[ids == ob].reshape(-1, 3).astype(dtype)
    ob_nrm = cloud.estimate_normals(ob_pts, 0.002, 30)
    want = cloud.prepare_object(ob_pts, ob_nrm, scene, 0.05, 0.001, K)
    got = cloud.prepare_object(torch.from_numpy(ob_pts).cuda(), torch.from_numpy(ob_nrm).cuda(),
                               torch.from_numpy(scene).cuda(), 0.05, 0.001, K)
    assert want is not None and got is not None
    for key in ("background_pts", "points_for_sample", "normals_for_sample"):
        assert isinstance(got[key], torch.Tensor) and np.array_equal(got[key].cpu().numpy(), want[key]), key
    for key in ("cloud_xyz", "cloud_normal"):
        assert np.array_equal(got["data"][key].cpu().numpy(), want["data"][key]), key
    assert got["data"]["cloud_xyz"].dtype == torch.from_numpy(ob_pts).dtype
