"""GPU (-m gpu): the kd-tree evaluation of the 9-DoF RANSAC (cg_ransac9d_kdtree_host, cg_ransac9d_kdtree_pose_dev,
estimate9DTransform(use_kdtree_for_eval=True), NunocsPredicter.use_kdtree_for_eval) against
oracle/aligning_kdtree_ref.py.

For every valid hypothesis the kernel's count (ratio * 2N) must equal the oracle's bit for bit, evaluated on the
kernel's own T with the source transformed in the kernel's order; the gates, valid flags and T are the residual
entry's.  Exact dyadic scenes pin the voxel rule and the `<=` at the threshold."""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import aligning_kdtree_ref
from test_ransac_kernel import kernel as plain_kernel

pytestmark = pytest.mark.gpu
MIN_S, MAX_S, MAX_D = np.array([0.005, 0.005, 0.001]), np.array([0.05] * 3), np.array([1.2] * 3)
LOOSE = dict(min_s=np.zeros(3), max_s=np.full(3, 99.0), max_dims=None)
KD_MAX_N = 65536


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "host_ransac9d_kdtree.npz"))


def kd_kernel(src, tgt, ids, thr, res, min_s=MIN_S, max_s=MAX_S, max_dims=MAX_D):
    from catgrasp_b200 import _lib
    src = np.ascontiguousarray(src, np.float64)
    tgt = np.ascontiguousarray(tgt, np.float64)
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1, 4)
    H = len(ids)
    mins = np.ascontiguousarray(min_s, np.float64).reshape(3)
    maxs = np.ascontiguousarray(max_s, np.float64).reshape(3)
    mdim = None if max_dims is None else np.ascontiguousarray(max_dims, np.float64).reshape(3)
    ratio, T, valid = np.empty(H), np.empty((H, 4, 4)), np.empty(H, np.uint8)
    ctx = _lib.Context.get()
    ctx.use_own_stream()
    ctx.check(ctx.lib.cg_ransac9d_kdtree_host(ctx.h, _lib.ptr(src), _lib.ptr(tgt), len(src), _lib.ptr(ids), H,
                                              C.c_double(thr), _lib.ptr(mins), _lib.ptr(maxs), _lib.ptr(mdim),
                                              C.c_double(res), _lib.ptr(ratio), _lib.ptr(T), _lib.ptr(valid)))
    return ratio, T, valid


def check(src, tgt, ids, thr, res, min_s=MIN_S, max_s=MAX_S, max_dims=MAX_D, min_valid=1):
    """Every valid hypothesis's count equals the oracle's on the kernel's T; gates and T are the residual entry's."""
    ratio, T, valid = kd_kernel(src, tgt, ids, thr, res, min_s, max_s, max_dims)
    pr, pT, pv = plain_kernel(src, tgt, ids, thr, min_s, max_s, max_dims)
    assert np.array_equal(valid, pv) and T.tobytes() == pT.tobytes()
    N = len(src)
    assert np.all(ratio[valid == 0] == 0.0)
    counts = np.rint(ratio * (2 * N))
    assert np.array_equal(ratio, counts / (2 * N))
    for h in np.nonzero(valid)[0]:
        want, _ = aligning_kdtree_ref.kdtree_eval(T[h], src, tgt, thr, res, order="kernel")
        assert int(counts[h]) == want, (h, int(counts[h]), want)
    assert int(valid.sum()) >= min_valid
    return ratio, T, valid


def _draws(N, H, seed):
    np.random.seed(seed)
    return np.array([np.random.choice(N, 4, replace=False) for _ in range(H)], np.int32)


def test_golden_draws(cuda, golden):
    for c in range(5):
        src, tgt = golden[f"c{c}_source"], golden[f"c{c}_target"]
        ids = _draws(len(src), 1000, int(golden[f"c{c}_seed"]))
        check(src, tgt, ids, float(golden[f"c{c}_thr"]), float(golden[f"c{c}_res"]), max_s=golden[f"c{c}_max_scale"])


def _pile(N, seed, noise=0.0015):
    """A cloud with outliers under a scaled rotation: most 4-subsets pass loose gates."""
    from catgrasp_b200.synthetic import random_rotation
    rng = np.random.RandomState(seed)
    src = rng.uniform(-0.5, 0.5, (N, 3))
    T = np.eye(4)
    T[:3, :3] = random_rotation(rng) * rng.uniform(0.02, 0.05)
    T[:3, 3] = rng.uniform(-0.1, 0.1, 3) + [0, 0, 0.7]
    tgt = src @ T[:3, :3].T + T[:3, 3] + rng.normal(0, noise, (N, 3))
    out = rng.choice(N, N // 5, replace=False)
    tgt[out] += rng.uniform(-0.02, 0.02, (len(out), 3))
    return src, tgt


@pytest.mark.parametrize("N", [4, 127, 128, 129, 2048, 8192, KD_MAX_N])
def test_point_counts(cuda, N):
    src, tgt = _pile(N, seed=N)
    H = 24 if N >= 8192 else 96
    rng = np.random.RandomState(N + 1)
    ids = np.array([rng.choice(N, 4, replace=False) for _ in range(H)], np.int32)
    for thr, res in ((0.003, 0.003), (0.005, 2.0 ** -8)):
        check(src, tgt, ids, thr, res, **LOOSE)


def test_seeded_piles(cuda):
    from catgrasp_b200.synthetic import make_pile
    for seed in (31, 32):
        scene = make_pile(6000, n_objects=3, seed=seed)
        tgt = scene["cloud_xyz"][scene["object_id"] == 1].astype(np.float64)
        rng = np.random.RandomState(seed)
        src = (tgt - tgt.mean(0)) * 9.0 + rng.normal(0, 0.002, tgt.shape)
        ids = np.array([rng.choice(len(src), 4, replace=False) for _ in range(200)], np.int32)
        check(src, tgt, ids, 0.003, 0.003, min_s=np.zeros(3), max_s=np.full(3, 0.5), max_dims=MAX_D)


# ---------------------------------------------------------------------------------------- exact dyadic geometry
def _dyadic(pts, t=(0.5, 0.25, 0.75)):
    """source = 4 anchor points + pts, target = source + t exactly; the subset of the anchors gives T = [I | t]."""
    src = np.r_[np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64), pts]
    return src, src + np.asarray(t), np.zeros((1, 4), np.int32) + np.arange(4, dtype=np.int32)


def _exact(src, tgt, ids, thr, res):
    ratio, T, valid = check(src, tgt, ids, thr, res, **LOOSE)
    want = np.eye(4)
    want[:3, 3] = tgt[0]
    assert T[0].tobytes() == want.tobytes()
    return int(round(ratio[0] * 2 * len(src)))


def test_distance_exactly_threshold_counts(cuda):
    thr = 2.0 ** -4
    lat = np.stack(np.meshgrid(*[np.arange(4) * 0.5 + 2.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    src, tgt, ids = _dyadic(lat)
    tgt[4::2, 0] += thr                            # every other lattice target exactly thr from its source
    N = len(src)
    assert _exact(src, tgt, ids, thr, 2.0 ** -6) == 2 * N
    assert _exact(src, tgt, ids, thr * (1 - 2.0 ** -20), 2.0 ** -6) == 2 * N - 2 * len(lat[::2])


def test_points_on_voxel_faces(cuda):
    r = 2.0 ** -3
    # origin = min - r/2; a coordinate min + (k + 1/2) r lies exactly on the face between cells k and k + 1
    faces = np.array([[0.0625, 0.0, 0.0], [0.0625 + r, 0.0, 0.0], [0.0625, 0.0625, 0.0625], [0.0, 0.0625 + 2 * r, 0.0]])
    src, tgt, ids = _dyadic(faces)
    for thr in (2.0 ** -4, 2.0 ** -6, 2.0 ** -2):
        _exact(src, tgt, ids, thr, r)


def test_one_voxel_own_voxels_and_duplicates(cuda):
    rng = np.random.RandomState(5)
    pts = np.round(rng.uniform(0, 1, (200, 3)) * 64) / 64
    pts = np.r_[pts, pts[:50], pts[:10]]                                  # duplicate points
    src, tgt, ids = _dyadic(pts)
    N = len(src)
    assert _exact(src, tgt, ids, 2.0 ** -8, 8.0) < 2 * N                   # all points in one voxel
    _exact(src, tgt, ids, 0.0, 2.0 ** -10)                                 # each distinct point in its own voxel
    _exact(src, tgt, ids, 2.0 ** -5, 2.0 ** -6)


def test_out_of_key_cloud_is_reported(cuda):
    from catgrasp_b200._lib import CgError
    src = np.random.RandomState(7).uniform(-0.5, 0.5, (256, 3))
    tgt = src * 0.03 + [0.0, 0.0, 0.7]
    src[100] = [300.0, 0.0, 0.0]                   # its target stays in the cloud: only src_t spans 2^21 voxels
    ids = np.array([[0, 1, 2, 3]], np.int32)
    with pytest.raises(CgError, match="2\\^21"):
        kd_kernel(src, tgt, ids, 0.003, 1e-6, **LOOSE)
    big = np.zeros((KD_MAX_N + 1, 3))
    with pytest.raises(CgError, match="CG_RANSAC_KD_MAX_N"):
        kd_kernel(big, big, ids, 0.003, 0.003, **LOOSE)


# ---------------------------------------------------------------------------------------- the fused pose entry
def kd_pose(src, tgt, ids, thrs, res, max_dims=MAX_D, min_s=MIN_S, max_s=MAX_S, ratio_thr=0.003):
    from catgrasp_b200.aligning import ransac9d_pose
    d = torch.device("cuda", 0)
    r = ransac9d_pose(torch.from_numpy(np.ascontiguousarray(src, np.float64)).to(d),
                      torch.from_numpy(np.ascontiguousarray(tgt, np.float64)).to(d),
                      torch.from_numpy(np.ascontiguousarray(ids, np.int32).reshape(-1, 4)).to(d), thrs,
                      max_scale=max_s, min_scale=min_s, max_dimensions=max_dims, ratio_threshold=ratio_thr,
                      kdtree_eval_resolution=res)
    return {k: v.cpu().numpy() for k, v in r.items()}


def test_two_thresholds_equal_two_launches_and_host_rule(cuda, golden):
    src, tgt = golden["c0_source"], golden["c0_target"]
    res = 0.003
    ids = [_draws(len(src), 1000, 40), _draws(len(src), 1000, 42)]
    both = kd_pose(src, tgt, np.r_[ids[0], ids[1]], (0.003, 0.005), res)
    assert both["record"].tobytes() == kd_pose(src, tgt, np.r_[ids[0], ids[1]], (0.003, 0.005), res)["record"].tobytes()
    best_ratio, chosen, pose = 0.0, -1, np.zeros((4, 4))
    for t, thr in enumerate((0.003, 0.005)):
        one = kd_pose(src, tgt, ids[t], (thr,), res)
        for k in ("winner", "count", "T", "count_ratio"):
            assert one[k][0].tobytes() == both[k][t].tobytes(), (t, k)
        ratio, T, valid = kd_kernel(src, tgt, ids[t], thr, res)
        keep = np.nonzero(valid)[0]
        w = int(keep[np.argmax(ratio[keep])])
        assert both["winner"][t] == w and both["count"][t] == int(round(ratio[w] * 2 * len(src)))
        assert both["T"][t].tobytes() == T[w].tobytes()
        errs = np.linalg.norm(np.c_[src, np.ones(len(src))] @ T[w][:3].T - tgt, axis=1)
        assert both["count_ratio"][t] == np.sum(errs <= 0.003)
        r3 = both["count_ratio"][t] / len(src)
        if not np.linalg.det(T[w][:3, :3]) < 0 and r3 > best_ratio:
            best_ratio, chosen, pose = r3, t, T[w]
    assert both["chosen"] == chosen and both["best_ratio"] == best_ratio and both["pose"].tobytes() == pose.tobytes()


# ---------------------------------------------------------------------------------------- public interface
def test_estimate9DTransform_matches_golden(cuda, golden):
    """The same winning hypothesis as the reference's run, its T within 1e-9 of the reference's (the tolerance
    tests/test_host_golden.py holds the residual mode's kernel T to), and the same inliers.  Cases 0-3 only: case 4
    puts half the distances exactly on the threshold, where the last bit of T -- the kernel's solve against cv2's --
    decides the count; the tests above hold the kernel to the oracle there on the kernel's own T."""
    from catgrasp_b200.aligning import estimate9DTransform
    for c in range(4):
        src, tgt = golden[f"c{c}_source"], golden[f"c{c}_target"]
        thr, res, seed = float(golden[f"c{c}_thr"]), float(golden[f"c{c}_res"]), int(golden[f"c{c}_seed"])
        ratio, T, valid = kd_kernel(src, tgt, _draws(len(src), 1000, seed), thr, res, max_s=golden[f"c{c}_max_scale"])
        keep = np.nonzero(valid)[0]
        gi = golden[f"c{c}_iters"]
        assert keep[np.argmax(ratio[keep])] == gi[np.argmax(golden[f"c{c}_ratios"])], c
        np.random.seed(seed)
        tf, inl = estimate9DTransform(src, tgt, thr, max_iter=1000, use_kdtree_for_eval=True,
                                      kdtree_eval_resolution=res, max_scale=golden[f"c{c}_max_scale"],
                                      min_scale=MIN_S, max_dimensions=MAX_D)
        assert np.array_equal(np.random.rand(2), golden[f"c{c}_next_rand"])
        np.testing.assert_allclose(tf, golden[f"c{c}_transform"], rtol=0, atol=1e-9)
        assert np.array_equal(inl, golden[f"c{c}_inliers"]), c


def kd_composition(npred, data, res):
    """predict with the kd-tree evaluation as the straight composition of predict_nocs, estimate9DTransform(
    use_kdtree_for_eval=True) at both thresholds and predict's post-processing (predicter.py:135-191)."""
    from catgrasp_b200.aligning import estimate9DTransform
    from catgrasp_b200.predicter import to_homo
    nocs_cloud, _ = npred.predict_nocs(data)
    ori = npred.data_transformed["cloud_xyz_original"]
    src = (np.eye(4) @ to_homo(nocs_cloud).T).T[:, :3]
    best_ratio, best = 0, None
    for thres in (0.003, 0.005):
        tf, _ = estimate9DTransform(source=src, target=ori, PassThreshold=thres, max_iter=npred.ransac_max_iter,
                                    use_kdtree_for_eval=True, kdtree_eval_resolution=res, max_scale=npred.max_scale,
                                    min_scale=npred.min_scale, max_dimensions=np.array([1.2, 1.2, 1.2]))
        if tf is None or np.linalg.det(tf[:3, :3]) < 0:
            continue
        errs = np.linalg.norm((tf @ to_homo(src).T).T[:, :3] - ori, axis=1)
        ratio = np.sum(errs <= 0.003) / len(errs)
        if ratio > best_ratio:
            best_ratio, best = ratio, tf.copy()
    return best, best_ratio


def test_predicter_kd_mode(cuda, golden_dir, tmp_path):
    from test_ransac_pose import _cases
    for name, npred, data in _cases(golden_dir, tmp_path):
        if name == "random":
            continue
        npred.use_kdtree_for_eval = True
        try:
            np.random.seed(0)
            want, want_ratio = kd_composition(npred, copy.deepcopy(data), npred.kdtree_eval_resolution)
            want_state = np.random.get_state()
            np.random.seed(0)
            nocs, tf = npred.predict(copy.deepcopy(data))
            got_state = np.random.get_state()
            assert np.array_equal(want_state[1], got_state[1]) and want_state[2:] == got_state[2:], name
            assert want is not None and tf.tobytes() == want.tobytes() and npred.best_ratio == want_ratio, name
            print(name, "kd best_ratio", want_ratio)
            npred.subsample = "device"
            np.random.seed(0)
            np.random.randint(0, 2 ** 63 - 1, dtype=np.int64)
            want_next = np.random.rand(2)
            np.random.seed(0)
            npred.predict(copy.deepcopy(data))
            assert np.array_equal(np.random.rand(2), want_next), name
        finally:
            npred.use_kdtree_for_eval = False
            npred.subsample = "host"
