"""GPU (-m gpu): the fused NUNOCS pose search (cg_ransac9d_pose_dev, aligning.ransac9d_pose) against the host rule on
cg_ransac9d_host's scores, and NunocsPredicter's two draw modes.

The host rule is aligning.estimate9DTransform's: the first maximum of the inlier ratio among valid hypotheses, and that
hypothesis's T; then predict's choice between thresholds (det test, ratio at 3 mm, strict `>` from 0)."""
import copy
import os

import numpy as np
import pytest
import torch

from test_ransac_kernel import _exact_case, _gate_points, kernel
from test_ransac_ref import MAX_D, MAX_S, MIN_S, THR, golden_ransac_case, lattice_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def fused(src, tgt, ids, thrs=(THR,), max_dims=MAX_D, ratio_thr=0.003, min_s=MIN_S, max_s=MAX_S):
    from catgrasp_b200.aligning import ransac9d_pose
    d = torch.device("cuda", 0)
    r = ransac9d_pose(torch.from_numpy(np.ascontiguousarray(src, np.float64)).to(d),
                      torch.from_numpy(np.ascontiguousarray(tgt, np.float64)).to(d),
                      torch.from_numpy(np.ascontiguousarray(ids, np.int32).reshape(-1, 4)).to(d), thrs,
                      max_scale=max_s, min_scale=min_s, max_dimensions=max_dims, ratio_threshold=ratio_thr)
    return {k: v.cpu().numpy() for k, v in r.items()}


def host_rule(src, tgt, ids, thr=THR, max_dims=MAX_D, min_s=MIN_S, max_s=MAX_S):
    ratio, T, valid = kernel(src, tgt, ids, thr=thr, max_dims=max_dims, min_s=min_s, max_s=max_s)
    keep = np.nonzero(valid)[0]
    if keep.size == 0:
        return -1, 0, None
    w = keep[np.argmax(ratio[keep])]
    return int(w), int(round(ratio[w] * len(src))), T[w]


def same_as_host(src, tgt, ids, thr=THR, max_dims=MAX_D, **kw):
    r = fused(src, tgt, ids, (thr,), max_dims, **kw)
    w, c, T = host_rule(src, tgt, ids, thr, max_dims, **kw)
    assert r["winner"][0] == w, (r["winner"][0], w)
    if w >= 0:
        assert r["count"][0] == c and r["T"][0].tobytes() == T.tobytes()
    else:
        assert r["count"][0] == 0 and not r["T"][0].any() and r["chosen"] == -1 and not r["pose"].any()
    return r


def test_golden_draws(cuda, golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    r = same_as_host(g["source"], g["target"], ids)
    assert r["winner"][0] >= 0
    same_as_host(g["source"], g["target"], ids[:500], max_dims=None)
    same_as_host(g["source"], g["target"], ids[:1])                          # H = 1


def test_lattice_ties_and_rotation(cuda, golden_dir):
    """Tied ratio 1.0 on the lattice golden; then the same draws rotated so that the first holder is not at 0."""
    g, src, tgt, ids = lattice_case(golden_dir, 3000)
    r = same_as_host(src, tgt, ids)
    w = int(r["winner"][0])
    assert r["count"][0] == len(src)
    ratio, _, valid = kernel(src, tgt, ids)
    lower = np.nonzero((valid == 0) | (ratio < 1.0))[0][:10]
    rot = np.r_[ids[lower], ids[w:]]                  # ten non-holders first, then the first holder and later ties
    r2 = same_as_host(src, tgt, rot)
    assert len(lower) == 10 and r2["winner"][0] == 10


def test_mirrored_fit_with_higher_raw_count(cuda):
    A, t, _, _ = _gate_points()
    rng = np.random.RandomState(12)
    q = np.c_[rng.randint(-32, 33, (1000, 2)) / 64.0, np.zeros(1000)]
    e = np.array([[0.25, 0.25, 0.5], [-0.25, 0.25, 0.5], [0.25, -0.25, 0.5], [0.25, 0.25, -0.5]])
    s4 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    src = np.r_[s4, q, e]
    tgt = np.r_[s4 @ A.T + t, q @ A.T + t, e @ (A @ np.diag([1.0, 1.0, -1.0])).T + t]
    r = same_as_host(src, tgt, [np.arange(1004, 1008), np.arange(4), np.arange(4)], max_dims=None)
    assert r["winner"][0] == 1 and r["count"][0] == 1004


def test_all_invalid(cuda, golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    r = same_as_host(g["source"], g["target"], ids[:300], max_s=np.array([1e-6] * 3))
    assert r["winner"][0] == -1 and r["best_ratio"] == 0.0


@pytest.mark.parametrize("N", [4, 129, 8192, 2 ** 20 + 3])
def test_point_counts(cuda, N):
    rng = np.random.RandomState(N)
    src, tgt = _exact_case(N, rng)
    H = 60 if N < 2 ** 20 else 6
    ids = np.array([rng.choice(N, 4, replace=False) for _ in range(H)], np.int32)
    ids[0] = [N - 1, N - 2, N - 3, N - 4]
    for mdims in (MAX_D, None):
        same_as_host(src, tgt, ids, max_dims=mdims)


def test_two_thresholds_equal_two_launches(cuda, golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    a, b = ids[:1500], ids[1500:3000]
    both = fused(g["source"], g["target"], np.r_[a, b], (0.003, 0.005))
    for t, (sub, thr) in enumerate(((a, 0.003), (b, 0.005))):
        one = fused(g["source"], g["target"], sub, (thr,))
        for k in ("winner", "count", "T", "count_ratio"):
            assert one[k][0].tobytes() == both[k][t].tobytes(), (t, k)


def _dyadic_scene():
    """An exact diagonal dyadic affine A | t (the polar step is exact, T = A bit for bit) through points 0..3 and 1000
    dyadic points, 100 of them at a residual of exactly 1/64 along x and 100 at 1/64 + 2^-30; four mirrored points
    (1004..1007, a det < 0 fit); four points (1008..1011) through a second valid affine A2 | t2 that nothing else fits."""
    A, t = np.diag([1 / 64, 1 / 32, 1 / 128]), np.array([0.125, -0.25, 0.5])
    A2, t2 = np.diag([1 / 32, 1 / 64, 1 / 128]), np.array([0.625, 0.25, -0.5])
    rng = np.random.RandomState(8)
    s4 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    q = rng.randint(-32, 33, (1000, 3)) / 64.0
    e = np.array([[0.25, 0.25, 0.5], [-0.25, 0.25, 0.5], [0.25, -0.25, 0.5], [0.25, 0.25, -0.5]])
    s4b = s4 + 2.0
    src = np.r_[s4, q, e, s4b]
    tgt = np.r_[s4 @ A.T + t, q @ A.T + t, e @ (A @ np.diag([1.0, 1.0, -1.0])).T + t, s4b @ A2.T + t2]
    tgt[4:104, 0] += 1 / 64
    tgt[104:204, 0] += 1 / 64 + 2.0 ** -30
    good, mirror, other = np.arange(4), np.arange(1004, 1008), np.arange(1008, 1012)
    return A, t, src, tgt, good, mirror, other


def test_ratio_count_and_threshold_choice(cuda):
    A, t, src, tgt, good, mirror, other = _dyadic_scene()
    N = len(src)
    T = np.r_[np.c_[A, t], [[0, 0, 0, 1]]]
    err = np.linalg.norm(np.c_[src, np.ones(N)] @ T[:3].T - tgt, axis=1)          # exact on this data
    want = int(np.count_nonzero(err <= 1 / 64))
    assert want == N - 100 - 4      # the mirrored points sit 1/128 from the model (counted), A2's points far off
    r = fused(src, tgt, [good], (1.0,), max_dims=None, ratio_thr=1 / 64)
    assert r["winner"][0] == 0 and r["count_ratio"][0] == want and np.array_equal(r["T"][0], T)
    kw = dict(max_dims=None, ratio_thr=1 / 64)
    # tie: the first threshold wins
    r = fused(src, tgt, [good, good], (0.5, 1.0), **kw)
    assert r["chosen"] == 0 and r["best_ratio"] == want / N and np.array_equal(r["pose"], r["T"][0])
    # the second strictly better
    r = fused(src, tgt, [other, other, good, good], (0.5, 1.0), **kw)
    assert list(r["winner"]) == [0, 0] and r["count_ratio"][0] < r["count_ratio"][1]
    assert r["chosen"] == 1 and r["best_ratio"] == want / N and np.array_equal(r["pose"], T)
    # only the second valid
    r = fused(src, tgt, [mirror, good], (0.5, 1.0), **kw)
    assert list(r["winner"]) == [-1, 0] and r["chosen"] == 1
    # a winner with no point within the ratio threshold is not a pose
    r = fused(src, tgt, [good, good], (0.5, 1.0), max_dims=None, ratio_thr=-1.0)
    assert list(r["winner"]) == [0, 0] and list(r["count_ratio"]) == [0, 0] and r["chosen"] == -1
    assert r["best_ratio"] == 0.0 and not r["pose"].any()


def test_deterministic_and_does_not_synchronise(cuda, golden_dir):
    from catgrasp_b200.aligning import ransac9d_pose
    g, ids = golden_ransac_case(golden_dir)
    d = torch.device("cuda", 0)
    s, tg = torch.from_numpy(g["source"]).to(d), torch.from_numpy(g["target"]).to(d)
    i2 = torch.from_numpy(np.r_[ids, ids[::-1]].astype(np.int32)).to(d)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = ransac9d_pose(s, tg, i2, (0.003, 0.005), max_scale=MAX_S, min_scale=MIN_S, max_dimensions=MAX_D)["record"]
        b = ransac9d_pose(s, tg, i2, (0.003, 0.005), max_scale=MAX_S, min_scale=MIN_S, max_dimensions=MAX_D)["record"]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


# ------------------------------------------------------------------ NunocsPredicter.predict in its two modes
def old_predict(npred, data, ids=None):
    """predict as a straight composition of predict_nocs, estimate9DTransform at both thresholds and predict's
    post-processing (predicter.py:135-203)."""
    from catgrasp_b200.aligning import estimate9DTransform
    from catgrasp_b200.predicter import to_homo
    nocs_cloud, _ = npred.predict_nocs(data, ids=ids)
    ori = npred.data_transformed["cloud_xyz_original"]
    src = (np.eye(4) @ to_homo(nocs_cloud).T).T[:, :3]
    best_ratio, best = 0, None
    for thres in (0.003, 0.005):
        tf, _ = estimate9DTransform(source=src, target=ori, PassThreshold=thres, max_iter=npred.ransac_max_iter,
                                    max_scale=npred.max_scale, min_scale=npred.min_scale,
                                    max_dimensions=np.array([1.2, 1.2, 1.2]))
        if tf is None or np.linalg.det(tf[:3, :3]) < 0:
            continue
        errs = np.linalg.norm((tf @ to_homo(src).T).T[:, :3] - ori, axis=1)
        ratio = np.sum(errs <= 0.003) / len(errs)
        if ratio > best_ratio:
            best_ratio, best = ratio, tf.copy()
    if best is None:
        return None, None, None
    return (np.eye(4) @ to_homo(nocs_cloud).T).T[:, :3], best, best_ratio


def _golden_predicter(g, tmp_path, sd):
    from catgrasp_b200.predicter import NunocsPredicter
    from catgrasp_b200.synthetic import write_artifacts
    ndir = write_artifacts(str(tmp_path / "artifacts-78"), "seg", n_pts=8192, state_dict=sd, normalizer=(g["mean"], g["std"]))
    return NunocsPredicter("nut", artifact_dir=ndir)


def _cases(golden_dir, tmp_path):
    """(name, predicter, object data): both NUNOCS goldens and two seeded piles with lattice weights."""
    from catgrasp_b200.predicter import NunocsPredicter
    from catgrasp_b200.synthetic import make_lattice_seg_state_dict, make_pile, make_state_dict, write_artifacts
    gr = np.load(os.path.join(golden_dir, "host_nunocs_random.npz"))
    gl = np.load(os.path.join(golden_dir, "host_nunocs_lattice.npz"))
    yield "random", _golden_predicter(gr, tmp_path / "r", make_state_dict("seg", 300, seed=int(gr["weight_seed"]))), \
        {"cloud_xyz": gr["cloud_xyz"].astype(np.float64), "cloud_normal": gr["cloud_normal"].astype(np.float64)}
    yield "lattice", _golden_predicter(gl, tmp_path / "l", make_lattice_seg_state_dict(
        seed=int(gl["weight_seed"]), mean=gl["mean"], std=gl["std"])), \
        {"cloud_xyz": gl["cloud_xyz"], "cloud_normal": gl["cloud_normal"].astype(np.float64)}
    nd = write_artifacts(str(tmp_path / "seg"), "seg", 2048, with_normalizer=False,
                         state_dict=make_lattice_seg_state_dict(seed=5))
    npd = NunocsPredicter("nut", artifact_dir=nd, device=0)
    for seed in (21, 22):
        scene = make_pile(6000, n_objects=3, seed=seed)
        obj = scene["object_id"] == 1
        yield f"pile{seed}", npd, {"cloud_xyz": scene["cloud_xyz"][obj], "cloud_normal": scene["cloud_normal"][obj]}


def test_host_mode_equals_composition(cuda, golden_dir, tmp_path):
    for name, npred, data in _cases(golden_dir, tmp_path):
        np.random.seed(0)
        want = old_predict(npred, copy.deepcopy(data))
        want_state = np.random.get_state()
        np.random.seed(0)
        assert npred.subsample == "host"
        nocs, tf = npred.predict(copy.deepcopy(data))
        got_state = np.random.get_state()
        assert np.array_equal(want_state[1], got_state[1]) and want_state[2:] == got_state[2:], name
        if want[1] is None:
            assert nocs is None and tf is None, name
            continue
        print(name, "best_ratio", npred.best_ratio)
        assert nocs.tobytes() == want[0].tobytes() and tf.tobytes() == want[1].tobytes(), name
        assert npred.best_ratio == want[2] and npred.nocs_pose.tobytes() == want[1].tobytes(), name


def test_device_transform_equals_host_transform(cuda, golden_dir, tmp_path):
    for name, npred, data in _cases(golden_dir, tmp_path):
        data = {k: np.asarray(v, np.float64) for k, v in data.items()}
        M = int((data["cloud_xyz"][:, 2] >= 0.1).sum())
        n = int(npred.cfg["n_pts"])
        ids = np.random.RandomState(3).choice(M, n, replace=M < n)
        d = copy.deepcopy(data)
        d["cloud_nocs"] = np.zeros(d["cloud_xyz"].shape)
        d["cloud_rgb"] = np.zeros(d["cloud_xyz"].shape)
        want = npred.transform(d, ids=ids)
        for inp in (data, {k: torch.from_numpy(v).cuda() for k, v in data.items()}):
            got = npred.device_transform(inp, ids=ids)
            for k in ("input", "cloud_xyz_original", "cloud_xyz", "cloud_normal", "keep_ids"):
                g = got[k].cpu().numpy()
                assert g.tobytes() == np.asarray(want[k], g.dtype).tobytes(), (name, k)


def test_device_mode(cuda, golden_dir, tmp_path):
    """One numpy value consumed; on the lattice golden the pose reaches the reference's best_ratio (every point within
    3 mm).  Tolerance: the golden's transform and the device's both put every one of the N points within 3 mm of its
    target, so by the triangle inequality they move each point to within 6 mm of each other; entry by entry, the device
    transform is one more hypothesis reaching ratio 1.0, so it lies within twice the largest distance to the golden's
    transform over 3000 other such hypotheses on the same correspondences."""
    from catgrasp_b200.predicter import to_homo
    gl = np.load(os.path.join(golden_dir, "host_nunocs_lattice.npz"))
    cases = {name: (npred, data) for name, npred, data in _cases(golden_dir, tmp_path)}
    npred, data = cases["lattice"]
    npred.subsample = "device"
    try:
        np.random.seed(0)
        np.random.randint(0, 2 ** 63 - 1, dtype=np.int64)
        want_next = np.random.rand(2)
        np.random.seed(0)
        nocs, tf = npred.predict(copy.deepcopy(data))
        assert np.array_equal(np.random.rand(2), want_next)
        assert tf is not None and npred.best_ratio == float(gl["best_ratio"])
        assert isinstance(tf, np.ndarray) and tf.shape == (4, 4) and nocs.shape == (8192, 3)
        src = np.asarray(nocs, np.float64)
        tgt = npred.data_transformed["cloud_xyz_original"]
        ids = np.random.RandomState(1).randint(0, len(src), (3000, 4)).astype(np.int32)
        ratio, T, valid = kernel(src, tgt, ids)
        full = T[(valid == 1) & (ratio == 1.0)]
        spread = np.abs(full - gl["transform"][None]).max()
        assert len(full) > 100
        assert np.abs(tf - gl["transform"]).max() <= 2 * spread, (np.abs(tf - gl["transform"]).max(), spread)
        moved = np.linalg.norm(np.c_[src, np.ones(len(src))] @ (tf - gl["transform"])[:3].T, axis=1)
        assert moved.max() <= 2 * 0.003, moved.max()
        errs = np.linalg.norm((tf @ to_homo(src).T).T[:, :3] - tgt, axis=1)
        assert np.sum(errs <= 0.003) / len(errs) == npred.best_ratio
        # CUDA input: CUDA results
        np.random.seed(0)
        nocs_c, tf_c = npred.predict({k: torch.from_numpy(np.asarray(v, np.float64)).cuda() for k, v in data.items()})
        assert tf_c.is_cuda and nocs_c.is_cuda and npred.pred_bins.is_cuda
    finally:
        npred.subsample = "host"


def test_pick_in_device_mode(cuda, tmp_path):
    """compute_candidate_grasp with both predicters in device mode: the same objects reach NUNOCS as in host mode."""
    import test_pick as P
    from catgrasp_b200 import synthetic
    from catgrasp_b200.predicter import GraspPredicter, NunocsPredicter
    sc = P._scene(True)
    gd = synthetic.write_artifacts(str(tmp_path / "cls"), "cls", 256, seed=3, logit_gain=12.0)
    gp = GraspPredicter("nut", artifact_dir=gd, device=0)
    nd = synthetic.write_artifacts(str(tmp_path / "seg"), "seg", 2048, with_normalizer=False,
                                   state_dict=synthetic.make_lattice_seg_state_dict(seed=5))
    npd = NunocsPredicter("nut", artifact_dir=nd, device=0)
    seg = P.IdSegmenter(sc["labels"])
    host_rec = P.RecordingNunocs(npd)
    np.random.seed(7)
    P._run_pipeline(sc, seg, host_rec, gp)
    npd.subsample = gp.subsample = "device"
    dev_rec = P.RecordingNunocs(npd)
    np.random.seed(7)
    out = P._run_pipeline(sc, seg, dev_rec, gp)
    assert [c[2] for c in dev_rec.calls] == [c[2] for c in host_rec.calls] and len(dev_rec.calls) >= 2
    print("device-mode pick: objects at NUNOCS", len(dev_rec.calls), "yielded", len(out))
