"""GPU (-m gpu): cg_grasp_affordance_dev (csrc/cg_affordance.cu) against oracle/affordance_ref.py, grasp by grasp.

Exact cases: dyadic points and cam_in_finger transforms that are signed axis permutations with dyadic translations,
so the kernel's fma chains and numpy's products are both exact and every inclusive edge can be hit on purpose: points
on xmin / xmax / zmin / zmax, points at |y - y_ext| == tol, many points tied at the extreme y across threads and
warps (np.argmin's first index decides which normal is tested), normals with ny = 0 (not facing away) and zero
normals (NaN, kept like the reference).  Random cases: random rigid transforms on the golden nut."""
import itertools

import numpy as np
import pytest
import torch

from oracle import affordance_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def kernel(cif, pts, nrm, aff, boxes, dirs, tol):
    import ctypes as C
    from catgrasp_b200 import _lib
    G = len(cif)
    dev = torch.device("cuda", 0)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)      # noqa: E731
    d_T, d_p, d_n, d_a = up(np.r_[np.asarray(cif).reshape(G, 16), np.zeros((int(G == 0), 16))]), up(pts), up(nrm), up(aff)
    out_p = torch.full((max(G, 1),), -7.0, dtype=torch.float64, device=dev)
    out_c = torch.full((max(G, 1), 4), -7, dtype=torch.int32, device=dev)
    boxes = np.ascontiguousarray(boxes, np.float64).reshape(-1, 4)
    F = len(boxes)
    ctx = _lib.Context.get(0)
    ctx.use_torch_stream()
    ctx.check(ctx.lib.cg_grasp_affordance_dev(ctx.h, _lib.ptr(d_T), G, _lib.ptr(d_p), _lib.ptr(d_n), _lib.ptr(d_a),
                                              len(pts), _lib.ptr(boxes), (C.c_int * F)(*dirs), F, C.c_double(tol),
                                              _lib.ptr(out_p), _lib.ptr(out_c)))
    torch.cuda.synchronize()
    return out_p.cpu().numpy()[:G], out_c.cpu().numpy()[:G, :F]


def oracle(cif, pts, nrm, aff, boxes, dirs, tol):
    poses = np.linalg.inv(cif)                  # the oracle takes grasp poses; fmig = I
    assert np.array_equal(np.linalg.inv(poses), cif)
    return affordance_ref.grasp_affordance_pointwise_nn(poses, np.eye(4), pts, nrm, aff, boxes, dirs, tol, exact=True)


def compare(cif, pts, nrm, aff, boxes, dirs, tol, tol_p=1e-12):
    p, c = kernel(cif, pts, nrm, aff, boxes, dirs, tol)
    po, co = oracle(cif, pts, nrm, aff, boxes, dirs, tol)
    np.testing.assert_array_equal(c, co)
    np.testing.assert_array_equal(np.isnan(p), np.isnan(po))
    ok = ~np.isnan(p)
    assert np.abs(p[ok] - po[ok]).max(initial=0) <= tol_p
    return p, c


def signed_permutations(rng, n):
    """n cam_in_finger transforms: signed axis permutations (det +1) with translations on a 1/64 grid."""
    out = []
    perms = list(itertools.permutations(range(3)))
    while len(out) < n:
        T = np.zeros((4, 4))
        T[3, 3] = 1
        p = perms[rng.randint(6)]
        s = rng.choice([-1.0, 1.0], 3)
        for i in range(3):
            T[i, p[i]] = s[i]
        if np.linalg.det(T[:3, :3]) < 0:
            continue
        T[:3, 3] = rng.randint(-4, 5, 3) / 64.0
        out.append(T)
    return np.array(out)


def dyadic_cloud(rng, P, zero_normals=True):
    """P points on a 1/64 grid in [-0.5, 0.5]^3 (many on every box edge, ties at every y), normals on a 1/4 grid
    (ny = 0 and zero normals included), affordances on a 1/1024 grid."""
    pts = rng.randint(-32, 33, (P, 3)) / 64.0
    nrm = rng.randint(-2, 3, (P, 3)) / 4.0
    if not zero_normals:
        nrm[~nrm.any(axis=1)] = [0.0, 0.0, 1.0]
    aff = rng.randint(0, 1025, P) / 1024.0
    return pts, nrm, aff


BOXES = np.array([[-0.25, 0.25, -0.125, 0.125], [-0.5, 0.0, 0.0, 0.5], [0.0, 0.125, -0.5, 0.5], [-0.0625, 0.0625, -0.0625, 0.0625]])


@pytest.mark.parametrize("P", [1, 127, 128, 129, 4099, 100003])
@pytest.mark.parametrize("F", [1, 2, 3, 4])
def test_exact_dyadic(cuda, P, F):
    rng = np.random.RandomState(P * 10 + F)
    pts, nrm, aff = dyadic_cloud(rng, P, zero_normals=(F % 2 == 0))
    dirs = [1, -1, -1, 1][:F]
    cif = signed_permutations(rng, 24 if P < 100000 else 6)
    compare(cif, pts, nrm, aff, BOXES[:F], dirs, 1.0 / 32)
    compare(cif, pts, nrm, aff, BOXES[:F], dirs, 0.0)


def test_edges_and_ties_constructed(cuda):
    """One grasp (identity), one finger closing along +y, box [-1/4, 1/4] x [-1/8, 1/8]; points built per rule."""
    box = BOXES[:1]
    P = 512
    pts = np.zeros((P, 3))
    pts[:, 0] = 0.75                                           # outside in x: ignored
    nrm = np.tile([0.0, -1.0, 0.0], (P, 1))                    # facing the finger (not away)
    aff = np.arange(P) / 1024.0
    # on the four edges, at the extreme y (= -1/8): inside
    pts[10] = [-0.25, -0.125, 0.0]
    pts[230] = [0.25, -0.125, 0.0]
    pts[300] = [0.0, -0.125, -0.125]
    pts[450] = [0.0, -0.125, 0.125]
    pts[460] = [0.0, -0.125 + 1 / 32, 0.0]                     # d == tol exactly: in the patch
    pts[470] = [0.0, -0.125 + 1 / 32 + 1 / 1024, 0.0]          # just beyond tol
    pts[480] = [0.25 + 1 / 1024, -0.5, 0.0]                    # just outside x, lower y: not the extreme
    cif = np.eye(4)[None]
    p, c = compare(cif, pts, nrm, aff, box, [1], 1 / 32)
    assert c[0, 0] == 5 and p[0] == (10 + 230 + 300 + 450 + 460) / 1024 / 5
    # the first extreme point decides the facing test: index 10 faces away -> finger dropped, whatever the others say
    n2 = nrm.copy()
    n2[10] = [0.0, 1.0, 0.0]
    p, c = compare(cif, pts, n2, aff, box, [1], 1 / 32)
    assert c[0, 0] == 0 and np.isnan(p[0])
    # ... and when the first extreme point sits at index >= 128, in the last warp of the block stride (230 % 128 = 102)
    pts2 = pts.copy()
    pts2[10] = [0.0, 0.0, 0.0]
    n3 = nrm.copy()
    n3[230] = [0.0, 1.0, 0.0]
    p, c = compare(cif, pts2, n3, aff, box, [1], 1 / 32)
    assert c[0, 0] == 0
    n3[230] = [1.0, 0.0, 0.0]                                  # ny == 0: not facing away, kept
    p, c = compare(cif, pts2, n3, aff, box, [1], 1 / 32)
    assert c[0, 0] == 4
    n3[230] = [0.0, 0.0, 0.0]                                  # zero normal: NaN test result, kept like the reference
    p, c = compare(cif, pts2, n3, aff, box, [1], 1 / 32)
    assert c[0, 0] == 4
    # a finger with no points, next to one with points; all fingers dropped -> NaN
    p, c = compare(cif, pts, nrm, aff, np.r_[box, [[2.0, 3.0, 2.0, 3.0]]], [1, -1], 1 / 32)
    assert c[0, 1] == 0 and c[0, 0] == 5
    p, c = compare(cif, pts, nrm, aff, [[2.0, 3.0, 2.0, 3.0]], [1], 1 / 32)
    assert np.isnan(p[0]) and c[0, 0] == 0


def test_negative_or_nan_tolerance_drops_fingers(cuda):
    """surface_tol < 0 or NaN: no point is in any patch, every finger is dropped without reading a normal."""
    rng = np.random.RandomState(1)
    pts, nrm, aff = dyadic_cloud(rng, 1000)
    cif = signed_permutations(rng, 8)
    for tol in (-1e-3, float("nan")):
        p, c = compare(cif, pts, nrm, aff, BOXES[:2], [1, -1], tol)
        assert np.isnan(p).all() and not c.any()


def test_grasp_counts(cuda):
    """G = 0 launches nothing; G = 70 000 (35 transforms repeated) scores every copy alike."""
    rng = np.random.RandomState(2)
    pts, nrm, aff = dyadic_cloud(rng, 129)
    p, c = kernel(np.zeros((0, 4, 4)), pts, nrm, aff, BOXES[:2], [1, -1], 1 / 32)
    assert p.shape == (0,)
    base = signed_permutations(rng, 35)
    p0, c0 = compare(base, pts, nrm, aff, BOXES[:2], [1, -1], 1 / 32)
    p, c = kernel(np.tile(base, (2000, 1, 1)), pts, nrm, aff, BOXES[:2], [1, -1], 1 / 32)
    assert np.array_equal(c, np.tile(c0, (2000, 1)))
    assert np.array_equal(p, np.tile(p0, 2000), equal_nan=True)


def test_random_rigid_on_golden_nut(cuda):
    import test_affordance_golden as ta
    from scipy.spatial import cKDTree
    from catgrasp_b200.synthetic import random_rotation
    full, affordance, down, down_n, boxes, fmig, poses = ta.affordance_case()
    _, nn = cKDTree(full).query(down)
    rng = np.random.RandomState(11)
    cif = []
    for g in poses[:40]:
        T = np.linalg.inv(fmig) @ np.linalg.inv(g)
        D = np.eye(4)
        D[:3, :3] = random_rotation(rng) if len(cif) % 2 else np.eye(3)
        D[:3, 3] = rng.normal(0, 0.003, 3)
        cif.append(D @ T)
    cif = np.array(cif)
    p, c = kernel(cif, down, down_n, affordance[nn], boxes, [1, -1], 0.005)
    po, co, _, und = affordance_ref.grasp_affordance_pointwise_nn(np.linalg.inv(cif), np.eye(4), down, down_n,
                                                                  affordance[nn], boxes, [1, -1], 0.005, decisions=True)
    d = ~und                                       # grasps with a decision inside the rounding slack are skipped
    print(f"affordance: {und.sum()} of {len(und)} random grasps undecided")
    assert und.sum() <= len(und) // 10
    np.testing.assert_array_equal(c[d], co[d])
    np.testing.assert_array_equal(np.isnan(p[d]), np.isnan(po[d]))
    ok = d & ~np.isnan(p)
    assert ok.sum() >= 5 and np.abs(p[ok] - po[ok]).max() < 1e-12
