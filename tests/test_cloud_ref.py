"""CPU tests of oracle/cloud_ref.py, the float64 restatement that the point-cloud kernels are checked against:
bit-identical to the reference's own functions (tests/golden/cloud_prep.npz), equal to live scipy on random, dyadic
and tied clouds with points at exactly the radius, and analytically right on a plane and a sphere."""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import cloud_ref

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "cloud_prep.npz")))


def test_backprojection_bit_identical_to_reference(golden):
    got = cloud_ref.depth2xyzmap(golden["depth"], golden["K"])
    assert got.dtype == np.float32
    assert (got.view(np.uint32) == golden["xyz_map"].view(np.uint32)).all()
    exact = golden["depth"] == np.float32(0.1)
    assert exact.any() and (got[exact][:, 2] == np.float32(0.1)).all()       # 0.1 itself is kept


def test_snap_crop_and_minus_bit_identical_to_reference(golden):
    xyz = golden["xyz_map"]
    scene = xyz[xyz[:, :, 2] >= 0.1].reshape(-1, 3)
    ob = xyz[golden["ids"] == golden["ob_id"]].reshape(-1, 3)
    down, _ = cloud_ref.voxel_down_sample(ob, 0.0005)
    assert (down.view(np.uint64) == golden["ob_pts_down"].view(np.uint64)).all()
    _, snap = cloud_ref.nearest(ob, down, np.inf)
    assert (snap == golden["snap_idx"]).all()
    crop = np.nonzero(cloud_ref.within(ob, scene, float(golden["gripper_diameter"]) / 2, compare_sqrt=True))[0]
    assert (crop == golden["crop_keep_ids"]).all()
    pts, keep = cloud_ref.cloudA_minus_cloudB(scene[crop], ob, 0.005)
    assert (keep == golden["minus_ids"]).all()
    assert (pts.view(np.uint32) == golden["minus_pts"].view(np.uint32)).all()


def test_orientation_bit_identical_to_reference(golden):
    xyz = golden["xyz_map"]
    pts = xyz[xyz[:, :, 2] >= 0.1].reshape(-1, 3)[golden["orient_ids"]].astype(np.float64)
    got = cloud_ref.orient(pts, golden["normals_in"])
    assert (got.view(np.uint64) == golden["oriented"].view(np.uint64)).all()
    got = cloud_ref.orient(pts, golden["normals_in"], golden["view_port"])
    assert (got.view(np.uint64) == golden["oriented_vp"].view(np.uint64)).all()


def _clouds():
    rng = np.random.RandomState(5)
    yield "random", rng.uniform(-0.02, 0.02, size=(1500, 3)) + [0.1, -0.05, 0.7]
    yield "dyadic", rng.randint(-24, 24, size=(1500, 3)).astype(np.float64) / 1024.0     # exact coordinates, many ties
    g = np.stack(np.meshgrid(np.arange(12), np.arange(12), np.arange(3), indexing="ij"), -1).reshape(-1, 3)
    yield "lattice", (g * 0.25).astype(np.float64)                                         # exact lattice ties


@pytest.mark.parametrize("case", ["random", "dyadic", "lattice"])
def test_nearest_and_radius_match_scipy(case):
    pts = dict(_clouds())[case]
    rng = np.random.RandomState(6)
    ref, q = pts[: len(pts) // 2], pts[len(pts) // 2:]
    if case == "lattice":                                     # half-way between lattice points: exact ties
        ref, q = pts, pts[::7] + [0.125, 0.0, 0.125]
    q = np.concatenate([q, ref[:50] + 0.0])                   # queries that coincide with reference points
    tree = cKDTree(ref)
    d_sp, i_sp = tree.query(q)
    d, i = cloud_ref.nearest(ref, q, np.inf)
    assert (d.view(np.uint64) == d_sp.view(np.uint64)).all()
    # the oracle picks the smallest index among the points at the minimum distance; scipy picks one of them, the same
    # one wherever there is no tie
    d2 = cloud_ref._d2(q, ref)
    tied = d2 == d2.min(axis=1, keepdims=True)
    ntie = tied.sum(1)
    assert (i == tied.argmax(1)).all()
    assert tied[np.arange(len(q)), i_sp].all()
    assert (i[ntie == 1] == i_sp[ntie == 1]).all()
    if case != "random":
        assert (ntie > 1).any()
    # a bound of exactly the found distance keeps it (inclusive), one ulp less drops it
    md = d_sp[7]
    d2, i2 = cloud_ref.nearest(ref, q[7:8], md)
    assert i2[0] == i[7]
    d3, i3 = cloud_ref.nearest(ref, q[7:8], np.nextafter(md, 0))
    assert i3[0] == -1 and np.isinf(d3[0])
    # radius membership at radii that are exact pairwise distances
    dd = np.sqrt(((q[:30, None, :] - ref[None, :, :]) ** 2).sum(-1)).reshape(-1)
    for r in [float(rng.choice(dd[dd > 0])), float(np.sort(dd)[40]), 0.003, 0.25]:
        balls = tree.query_ball_point(q, r)
        want = np.array([len(b) > 0 for b in balls])
        assert (cloud_ref.within(ref, q, r, compare_sqrt=False) == want).all()
        dist_all = tree.query(q)[0]
        assert (cloud_ref.within(ref, q, r, compare_sqrt=True) == (dist_all <= r)).all()


def test_radius_and_sqrt_forms_differ_at_the_boundary():
    """d2 <= r*r and sqrt(d2) <= r disagree for some r: the crop and cloudA_minus_cloudB must each use their own."""
    rng = np.random.RandomState(8)
    found = False
    for _ in range(2000):
        a, b = rng.uniform(0, 1, 3), rng.uniform(0, 1, 3)
        d2 = ((a[0] - b[0]) ** 2 + (a[1] - b[1]) ** 2) + (a[2] - b[2]) ** 2
        r = np.sqrt(d2)
        for rr in (r, np.nextafter(r, 0), np.nextafter(r, 2)):
            sq = cloud_ref.within(b[None], a[None], rr, True)[0]
            ba = cloud_ref.within(b[None], a[None], rr, False)[0]
            found |= sq != ba
    assert found


def test_neighbour_lists_match_scipy_ball_and_order():
    pts = dict(_clouds())["lattice"]
    nbr, cnt = cloud_ref.neighbours(pts, 0.5, 9)
    tree = cKDTree(pts)
    for i in range(0, len(pts), 37):
        ball = np.array(sorted(tree.query_ball_point(pts[i], 0.5)))
        d2 = ((pts[ball] - pts[i]) ** 2).sum(1)
        want = ball[np.lexsort((ball, d2))][:9]
        assert cnt[i] == len(want) and (nbr[i, :cnt[i]] == want).all()
        assert nbr[i, 0] == i


def test_voxel_means_are_sequential_sums():
    rng = np.random.RandomState(9)
    pts = rng.uniform(-0.01, 0.01, size=(3000, 3))
    nrm = rng.normal(size=pts.shape)
    means, nsum, vox = cloud_ref.voxel_down_sample(pts, 0.004, normals=nrm)
    for v in [0, 5, len(means) - 1]:
        m = np.nonzero(vox == v)[0]
        s = np.zeros(3)
        n = np.zeros(3)
        for k in m:
            s = s + pts[k]
            n = n + nrm[k]
        assert (means[v] == s / len(m)).all()
        assert np.allclose(nsum[v], n / np.linalg.norm(n), rtol=0, atol=1e-15)
    cells = cloud_ref.voxel_cells(pts, 0.004)
    order = np.lexsort((cells[:, 2], cells[:, 1], cells[:, 0]))
    assert (np.diff(vox[order]) >= 0).all()          # ascending (ix, iy, iz)


def test_normals_plane_and_sphere_are_analytic():
    rng = np.random.RandomState(10)
    xy = rng.uniform(-0.02, 0.02, size=(2500, 2))
    z0 = 0.6
    tilt = np.array([0.3, -0.2])
    plane = np.column_stack([xy, z0 + xy @ tilt])
    n_true = np.array([-tilt[0], -tilt[1], 1.0])
    n_true /= np.linalg.norm(n_true)
    n, bound, _, cnt = cloud_ref.estimate_normals(plane, 0.004, 30)
    assert (cnt >= 3).all() and (bound < cloud_ref.NORMAL_DECIDED).all()
    n_true = -n_true if n_true @ (-plane[0]) < 0 else n_true        # facing the camera at the origin
    assert np.abs(n - n_true).max() < 1e-9

    d = rng.normal(size=(4000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    c = np.array([0.0, 0.0, 0.5])
    sphere = c + 0.05 * d
    n, bound, _, _ = cloud_ref.estimate_normals(sphere, 0.006, 30)
    cosang = np.abs((n * d).sum(1))
    assert np.median(cosang) > 0.999 and cosang.min() > 0.99
    view = -sphere / np.linalg.norm(sphere, axis=1, keepdims=True)
    assert ((n * view).sum(1) >= 0).all()


def test_too_few_neighbours_give_z():
    pts = np.array([[0.0, 0.0, 0.5], [0.0, 0.0, 0.6], [0.001, 0.0, 0.6]])
    n, bound, _, cnt = cloud_ref.estimate_normals(pts, 0.002, 30)
    assert cnt.tolist() == [1, 2, 2]
    # (0,0,1) / (1 + 1e-10), flipped towards the camera at the origin
    assert (n[:, 2] == -(1.0 / (1.0 + 1e-10))).all() and (n[:, :2] == 0).all()
