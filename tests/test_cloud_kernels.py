"""GPU tests of the point-cloud kernels (csrc/cg_cloud.cu via catgrasp_b200/cloud.py) against oracle/cloud_ref.py.

Bit-identical: back-projection on the full 2064 x 1544 frame; voxel membership, means and normals; nearest indices
and distances; radius masks.  Normals: neighbour sets equal to the oracle's, normals within the oracle's eigengap
bound on every decided point.  prepare_object equals the oracle composition on every object of a rendered pile.

Seeded mutations of cg_cloud.cu and the test aimed at each (the mutants are not built by this file):
- ``<`` for ``<=`` at the radius (radius_mask_kernel / normals_kernel): test_radius_masks_bit_identical (radii that
  are exact pairwise distances) and test_normals_neighbour_sets_and_bound (lattice points at exactly r);
- a skipped neighbour cell (axis_range without its slack, or a column dropped): test_nearest_bit_identical and
  test_radius_masks_bit_identical (queries on cell faces, radius = cell);
- ties to the larger index (key_less / nearest_kernel): test_nearest_bit_identical (lattice ties) and
  test_normals_neighbour_sets_and_bound (ties at the max_nn-th neighbour);
- voxel origin without ``- voxel/2``: test_voxel_bit_identical (points on voxel faces);
- the crop compared in squares: test_radius_masks_bit_identical (sqrt form at boundary radii) and
  test_prepare_object_matches_oracle;
- orientation flipped on ``<=``: test_normals_neighbour_sets_and_bound (isolated points at camera z = 0 have
  normal (0,0,1), dot == 0 with the view ray, and must keep their sign).
"""
import numpy as np
import pytest
import torch

from catgrasp_b200 import cloud, synthetic
from oracle import cloud_ref

pytestmark = pytest.mark.gpu

K_FULL = np.array([2257.7500557850776, 0, 1032, 0, 2257.4882391629421, 772, 0, 0, 1], np.float64).reshape(3, 3)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_backprojection_full_frame_bit_identical(dtype):
    depth, _ = synthetic.render_depth(K_FULL, 1544, 2064, n_objects=8, seed=1)
    depth = depth.astype(dtype)
    rng = np.random.RandomState(2)
    flat = depth.reshape(-1)
    pick = rng.choice(flat.size, 3000, replace=False)
    flat[pick[:1000]] = 0
    flat[pick[1000:2000]] = dtype(0.1)
    flat[pick[2000:]] = np.nextafter(dtype(0.1), dtype(0))
    got = cloud.depth2xyzmap(depth, K_FULL)
    want = cloud_ref.depth2xyzmap(depth, K_FULL)
    assert got.shape == (1544, 2064, 3) and got.dtype == np.float32
    assert (_bits(got) == _bits(want)).all()
    assert (got.reshape(-1, 3)[pick[1000:2000], 2] == np.float32(0.1)).all()
    assert (got.reshape(-1, 3)[pick[2000:]] == 0).all()


def _voxel_cases():
    rng = np.random.RandomState(3)
    v = 0.001
    yield "random", rng.uniform(-0.05, 0.05, size=(20000, 3)) + [0.0, 0.0, 0.6], v
    # points on voxel faces: coordinates at multiples of the voxel (relative to a min that sits on the lattice too)
    g = rng.randint(0, 40, size=(20000, 3)).astype(np.float64) * 0.5 - 7.0
    yield "faces", g * 2.0 ** -10, 2.0 ** -10                              # dyadic: half the points lie on faces
    yield "one_voxel", rng.uniform(0, 0.2 * v, size=(5000, 3)), v
    yield "one_point", np.array([[0.1, -0.2, 0.3]]), v
    yield "negative", rng.uniform(-0.3, -0.1, size=(30000, 3)), 0.002
    yield "big", rng.uniform(-0.2, 0.2, size=((1 << 20) + 3, 3)) * [1, 1, 0.25], 0.002      # > 2^16 voxels


@pytest.mark.parametrize("case", ["random", "faces", "one_voxel", "one_point", "negative", "big"])
def test_voxel_bit_identical(case):
    pts, voxel = dict((c, (p, v)) for c, p, v in _voxel_cases())[case]
    nrm = np.random.RandomState(4).normal(size=pts.shape)
    nrm[: len(nrm) // 7] = 0.0
    means, nsum, _ = cloud_ref.voxel_down_sample(pts, voxel, normals=nrm)
    got_p, got_n = cloud.voxel_down_sample(pts, voxel, normals=nrm)
    assert got_p.shape == means.shape
    assert (_bits(got_p) == _bits(means)).all()
    assert (_bits(got_n) == _bits(nsum)).all()
    if case == "big":
        assert len(means) > (1 << 16)
    got_only = cloud.voxel_down_sample(pts, voxel)
    assert (_bits(got_only) == _bits(means)).all()
    # torch in, torch out
    t = cloud.voxel_down_sample(torch.from_numpy(pts).cuda(), voxel)
    assert t.is_cuda and (_bits(t.cpu().numpy()) == _bits(means)).all()


def _query_cases():
    rng = np.random.RandomState(5)
    yield "random", rng.uniform(-0.02, 0.02, (20000, 3)) + [0, 0, 0.6], rng.uniform(-0.021, 0.021, (20000, 3)) + [0, 0, 0.6]
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), np.arange(4), indexing="ij"), -1).reshape(-1, 3) / 1024.0
    q = g[::3] + np.array([0.5, 0.0, 0.5]) / 1024.0                                         # exact ties between lattice points
    yield "lattice", g, np.concatenate([q, g[::5]])


@pytest.mark.parametrize("case", ["random", "lattice"])
def test_nearest_bit_identical(case):
    ref, q = dict((c, (a, b)) for c, a, b in _query_cases())[case]
    for max_dist in [0.0005, 0.002, 1.0 / 1024.0, np.sqrt(0.5) / 1024.0]:
        d, i = cloud.nearest(ref, q, max_dist)
        dw, iw = cloud_ref.nearest(ref, q, max_dist)
        assert (i == iw).all(), max_dist
        assert (_bits(d) == _bits(dw)).all()
    if case == "lattice":
        d2 = cloud_ref._d2(q[:200], ref)
        assert ((d2 == d2.min(1, keepdims=True)).sum(1) > 1).any()
        # a bound of exactly the tied distance keeps the smaller index
        d, i = cloud.nearest(ref, q[:200], np.sqrt(0.5) / 1024.0)
        assert (i >= 0).all()


@pytest.mark.parametrize("case", ["random", "lattice"])
def test_radius_masks_bit_identical(case):
    ref, q = dict((c, (a, b)) for c, a, b in _query_cases())[case]
    dd = np.sqrt(cloud_ref._d2(q[:40], ref)).reshape(-1)
    radii = [float(np.sort(dd)[100]), float(np.sort(dd)[2000]), 0.001, 1.0 / 1024.0]
    for r in radii:
        idx = cloud.CloudIndex(ref, r)
        for sq in (False, True):
            got = idx.within(q, r, compare_sqrt=sq).cpu().numpy().astype(bool)
            want = cloud_ref.within(ref, q, r, compare_sqrt=sq)
            assert (got == want).all(), (r, sq)
    pa, keep = cloud.cloudA_minus_cloudB(q, ref, radii[0])
    pw, kw = cloud_ref.cloudA_minus_cloudB(q, ref, radii[0])
    assert (keep == kw).all() and (_bits(pa) == _bits(pw)).all()
    far = ref + 10.0                                                       # distant B: nothing removed
    pa, keep = cloud.cloudA_minus_cloudB(q, far, 0.005)
    assert (keep == np.arange(len(q))).all()
    pa, keep = cloud.cloudA_minus_cloudB(q, np.zeros((0, 3)), 0.005)       # empty B
    assert (keep == np.arange(len(q))).all()


def _normal_cases():
    K = K_FULL.copy()
    K[:2] /= 8
    depth, _ = synthetic.render_depth(K, 1544 // 8, 2064 // 8, n_objects=8, seed=6, bin_size=0.25)
    xyz = cloud_ref.depth2xyzmap(depth, K).reshape(-1, 3).astype(np.float64)
    xyz = xyz[np.abs(xyz[:, 0]) < 0.12][:14000]
    yield "scene", xyz, 0.012, 30
    # fronto-parallel dyadic lattice: exact ties everywhere, more than 256 points in a ball
    g = np.stack(np.meshgrid(np.arange(60), np.arange(60), indexing="ij"), -1).reshape(-1, 2) / 1024.0
    yield "lattice", np.column_stack([g, np.full(len(g), 0.5)]), 12.0 / 1024.0, 30
    yield "lattice_exact_r", np.column_stack([g[:900], np.full(900, 0.5)]), 2.0 / 1024.0, 7
    # a plane through the camera: normals perpendicular to the view ray (dot == 0 must not flip)
    # plus isolated points at z = 0, whose (0,0,1) normals have dot == 0 with the view ray and must stay unflipped
    iso = np.column_stack([0.2 + 0.01 * np.arange(20), np.zeros(20), np.zeros(20)])
    yield "through_camera", np.concatenate([np.column_stack([g[:1200] - 0.03, np.zeros(1200)]), iso]), 3.0 / 1024.0, 20


@pytest.mark.parametrize("case", ["scene", "lattice", "lattice_exact_r", "through_camera"])
def test_normals_neighbour_sets_and_bound(case):
    pts, r, max_nn = dict((c, (p, rr, m)) for c, p, rr, m in _normal_cases())[case]
    n_ref, bound, nbr_ref, cnt_ref = cloud_ref.estimate_normals(pts, r, max_nn)
    idx = cloud.CloudIndex(pts, r)
    n, nbr, cnt = idx.normals(r, max_nn, neighbours=True)
    n, nbr, cnt = n.cpu().numpy(), nbr.cpu().numpy().astype(np.int64), cnt.cpu().numpy()
    assert (cnt == cnt_ref).all()
    assert (nbr == nbr_ref).all()
    decided = bound <= cloud_ref.NORMAL_DECIDED
    # orientation is decided when the oracle's dot with the view direction is clear of the bound
    view = -pts / np.linalg.norm(pts, axis=1, keepdims=True)
    dots = (view * n_ref).sum(1)
    fixed = bound == 0
    err = np.abs(n - n_ref).max(1)
    assert (err[fixed] == 0).all()
    clear = decided & ~fixed & (np.abs(dots) > 4 * np.maximum(bound, 1e-15))
    assert (err[clear] <= 4 * bound[clear] + 1e-15).all(), err[clear].max()
    # up to sign where the orientation itself is undecided
    amb = decided & ~fixed & ~clear
    e2 = np.minimum(np.abs(n - n_ref).max(1), np.abs(n + n_ref).max(1))
    assert (e2[amb] <= 4 * bound[amb] + 1e-15).all()
    print(f"{case}: {len(pts)} points, decided {decided.sum()}, undecided {(~decided).sum()}, "
          f"orientation-ambiguous {amb.sum()}")
    if case == "through_camera":
        assert (n[-20:] == [0.0, 0.0, 1.0 / (1.0 + 1e-10)]).all()
    # the wrapper = estimation + orientation
    assert (_bits(cloud.estimate_normals(pts, r, max_nn)) == _bits(n)).all()


def test_prepare_object_matches_oracle():
    from catgrasp_b200.my_cpp import makeOccupancyGridFromCloudScan
    K = K_FULL.copy()
    K[:2] /= 3
    depth, ids = synthetic.render_depth(K, 1544 // 3, 2064 // 3, n_objects=8, seed=7)
    xyz = cloud.depth2xyzmap(depth, K)
    scene_full = xyz[xyz[:, :, 2] >= 0.1].reshape(-1, 3)
    scene = cloud.voxel_down_sample(scene_full, 0.001)
    done = 0
    for ob_id in np.unique(ids[ids >= 0]):
        ob = xyz[ids == ob_id].reshape(-1, 3)
        ob_n = cloud.estimate_normals(ob, 0.003, 30)
        got = cloud.prepare_object(ob, ob_n, scene, 0.06)
        want = cloud_ref.prepare_object(ob, ob_n, scene, 0.06)
        if want is None:
            assert got is None
            continue
        data, occ_in, pfs, nfs = want
        assert (_bits(got["data"]["cloud_xyz"]) == _bits(data["cloud_xyz"])).all()
        assert (_bits(got["data"]["cloud_normal"]) == _bits(data["cloud_normal"])).all()
        occ = makeOccupancyGridFromCloudScan(occ_in, K, 0.001) if len(occ_in) else np.zeros((0, 3), np.float32)
        assert (_bits(got["background_pts"]) == _bits(occ)).all()
        assert (_bits(got["points_for_sample"]) == _bits(pfs)).all()
        assert (_bits(got["normals_for_sample"]) == _bits(nfs)).all()
        done += 1
    assert done >= 4
