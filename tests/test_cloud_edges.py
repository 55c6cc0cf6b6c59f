"""GPU tests of the point-cloud kernels (csrc/cg_cloud.cu via catgrasp_b200/cloud.py) at the index's edges, against
oracle/cloud_ref.py, bit-identical unless stated.

tests/test_cloud_kernels.py always queries an index whose cell equals the query radius, at small coordinates, without
duplicate points.  This file covers the rest of the index: cells much finer and coarser than the radius (column walks
over many cells), reaches that end within an ulp of a cell face (where only axis_range's RANGE_SLACK keeps the
point's cell in range), radius 0 and points repeated up to 300 times (ties at d2 = 0 across several compactions of the
normals buffer), max_nn at 1, 2, 3, 63 and 64 and the n >= 3 cut-off, clouds 1000 m from the
camera, a cloud 2^21 - 1 cells wide (63-bit keys), NaN and infinite queries, queries exactly r outside the cloud's
bounding box, and back-projection at degenerate shapes and non-finite depths.

Seeded mutations of cg_cloud.cu and the test aimed at each.  Each mutant was built once, when these tests were
written, and failed the test named for it on an H100 (the mutants are not built by this file):
- RANGE_SLACK = 0: test_reach_ending_on_a_cell_face;
- the top cell dropped when a query's reach passes the cloud's box (``hi = fhi > maxc ? maxc - 1 : ...``):
  test_queries_exactly_r_outside_the_box;
- a tie in compact() broken towards the larger index (``ia > ib``): test_duplicates_and_radius_zero (more than 256
  points at d2 = 0) and test_max_nn_edges;
- the n >= 3 cut-off moved to n >= 2: test_max_nn_edges (neighbourhoods of exactly 2 points);
- the column walk bounded by ``cy < C.y1`` instead of ``<=``: test_index_cell_not_equal_to_radius;
- the radix sort over 3 * bits - 1 key bits (the top x bit left unsorted): test_cloud_at_the_2_21_cell_limit;
- an empty query batch launched as a zero-block grid (the ``Q == 0`` early return dropped):
  test_bad_and_empty_queries;
- NaN depths treated as below the 0.1 cut (``z >= 0.1`` for ``!(z < 0.1)``): test_depth2xyz_shapes_and_non_finite_depths.
test_normals_do_not_depend_on_the_cell (a selection that depends on the buffer's fill order),
test_cloud_far_from_the_camera (cell arithmetic that loses precision at 1000 m) and test_tiny_clouds_and_refusals (a
grid-stride loop that skips warps when P < 4) pin contracts without a mutant built for them.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from catgrasp_b200 import _lib, cloud
from oracle import cloud_ref

pytestmark = pytest.mark.gpu


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else t


def _check_queries(idx, ref, q, r):
    """nearest within r and both radius masks at r equal the oracle, bit for bit."""
    d, i = idx.nearest(q, r)
    dw, iw = cloud_ref.nearest(ref, q, r)
    assert (_np(i) == iw).all() and (_bits(_np(d)) == _bits(dw)).all()
    for sq in (False, True):
        got = _np(idx.within(q, r, compare_sqrt=sq)).astype(bool)
        assert (got == cloud_ref.within(ref, q, r, compare_sqrt=sq)).all(), sq
    return iw


def _check_normals(pts, n, nbr, cnt, r, max_nn):
    """Neighbour lists equal the oracle's; normals with fewer than 3 neighbours or a zero covariance are the oriented
    (0,0,1) exactly; the others are within the oracle's eigengap bound where it is decided (up to sign where the
    orientation itself is within the bound)."""
    n_ref, bound, nbr_ref, cnt_ref = cloud_ref.estimate_normals(pts, r, max_nn)
    n, nbr, cnt = _np(n), _np(nbr).astype(np.int64), _np(cnt)
    assert (cnt == cnt_ref).all()
    assert (nbr == nbr_ref).all()
    fixed = bound == 0
    assert (n[fixed] == n_ref[fixed]).all()
    ok = (bound <= cloud_ref.NORMAL_DECIDED) & ~fixed
    e = np.minimum(np.abs(n - n_ref).max(1), np.abs(n + n_ref).max(1))
    assert (e[ok] <= 4 * bound[ok] + 1e-15).all()
    return cnt_ref, fixed


def _scene(seed, n=3000):
    """A random patch plus a dyadic lattice (points on cell faces for power-of-two cells)."""
    rng = np.random.RandomState(seed)
    a = rng.uniform(-0.01, 0.01, (n, 3)) + [0.0, 0.0, 0.6]
    g = np.stack(np.meshgrid(np.arange(12), np.arange(12), np.arange(3), indexing="ij"), -1).reshape(-1, 3) / 1024.0
    return np.concatenate([a, g + [0.0, 0.0, 0.6]])


@pytest.mark.parametrize("div", [7.0, 2.0, 1.0, 1.0 / 3.0])
def test_index_cell_not_equal_to_radius(div):
    """Queries at r from an index of cell r/7, r/2, r and 3r: the walk spans up to 15 x 15 columns of 15 cells, or
    one cell holds several radii."""
    ref = _scene(1)
    r = 4.0 / 1024.0
    rng = np.random.RandomState(2)
    q = np.concatenate([ref[::7] + rng.uniform(-r, r, ref[::7].shape), ref[::11],
                        ref[::13] + [r, 0.0, 0.0], ref[::17] + [0.0, -r, 0.0]])       # r away along an axis
    idx = cloud.CloudIndex(ref, r / div)
    _check_queries(idx, ref, q, r)


def _face_pairs(m, cell, R, n=3000):
    """Points on cell faces, x = o + k * cell for a non-dyadic cell with o = m - cell/2 (the index's origin when m is
    the cloud's minimum), and queries at x -+ R moved by up to 4 ulps.  Returns the points, the queries, and the
    queries that the oracle accepts at R but whose point's cell lies outside the range axis_range computes without
    its slack, floor(((q - o) -+ R) / cell): the rounding of (q - o) -+ R and of the division puts the reach's end one
    cell short.  numpy rounds each operation once, as the kernel does."""
    o = m - cell * 0.5
    x = o + np.arange(1, n) * cell
    cx = np.floor((x - o) / cell)                                         # key_kernel's cell of each point
    qs, need = [], []
    for sign in (-1.0, 1.0):
        q0 = x + sign * R
        for k in range(-4, 5):
            q = q0 + k * np.spacing(q0)
            acc = (q - x) * (q - x) <= R * R
            lo, hi = np.floor(((q - o) - R) / cell), np.floor(((q - o) + R) / cell)
            qs.append(q)
            need.append(acc & ((cx < lo) | (cx > hi)))
    return x, np.concatenate(qs), np.concatenate(need)


@pytest.mark.parametrize("m,cell,R", [(-0.2, 0.003, 0.0071), (-0.2, 0.0017, 0.0017), (0.4123, 0.0007, 0.0031)])
def test_reach_ending_on_a_cell_face(m, cell, R):
    """Queries whose reach ends within an ulp of a cell face holding a point within R: nearest and both radius
    masks equal the oracle, bit for bit, including on the queries that need axis_range's RANGE_SLACK."""
    x, qx, need = _face_pairs(m, cell, R)
    assert need.sum() >= 5
    rng = np.random.RandomState(14)
    pick = np.concatenate([np.nonzero(need)[0], rng.choice(len(qx), 600, replace=False)])
    # each query's own point alone on a line of constant (y, z), 4R from any other line, so that it is the only
    # point within R and a range that misses its cell changes the answer
    j = np.arange(len(pick))
    y, z = 0.5 + (j % 32) * 4 * R, 0.25 + (j // 32) * 4 * R
    ref = np.concatenate([[[m, 0.5 - 4 * R, 0.25 - 4 * R]], np.c_[x[pick % len(x)], y, z]])   # [0]: sets o_x
    q = np.c_[qx[pick], y, z]
    idx = cloud.CloudIndex(ref, cell)
    oc = (C.c_double * 3)()
    idx.ctx.check(idx.ctx.lib.cg_cloud_index_info(idx.h, None, None, None, oc))
    assert oc[0] == m - cell * 0.5                                        # the origin _face_pairs assumed
    hard = q[:need.sum()]
    assert cloud_ref.within(ref, hard, R, compare_sqrt=False).all()
    assert _np(idx.within(hard, R, compare_sqrt=False)).all()
    _check_queries(idx, ref, q, R)


def test_normals_do_not_depend_on_the_cell():
    """Normals at radius r from indices of cell r/3, r and 4r: neighbour lists, counts and normals bit-identical to
    each other (selection and covariance order are the cell's business only through the buffer's fill order)."""
    pts = _scene(3, 2000)
    r = 3.0 / 1024.0
    outs = []
    for cell in (r / 3, r, 4 * r):
        n, nbr, cnt = cloud.CloudIndex(pts, cell).normals(r, 30, neighbours=True)
        outs.append((_np(n), _np(nbr), _np(cnt)))
    for n, nbr, cnt in outs[1:]:
        assert (_bits(n) == _bits(outs[0][0])).all() and (nbr == outs[0][1]).all() and (cnt == outs[0][2]).all()
    _check_normals(pts, *outs[0], r, 30)


def _duplicated(seed):
    """Unique points each repeated 1 to 300 times, shuffled; the point repeated 300 times stands apart."""
    rng = np.random.RandomState(seed)
    u = rng.uniform(-0.02, 0.02, (60, 3)) + [0.0, 0.0, 0.5]
    u[0] = [0.125, 0.125, 0.5]              # isolated: its neighbourhood is its copies, whose sums and means are exact
    reps = rng.randint(1, 301, len(u))
    reps[0] = 300
    reps[1] = 1
    pts = np.repeat(u, reps, axis=0)
    perm = rng.permutation(len(pts))
    return u, pts[perm]


def test_duplicates_and_radius_zero():
    u, pts = _duplicated(4)
    idx = cloud.CloudIndex(pts, 0.004)
    # nearest: the smallest index among the copies
    d, i = idx.nearest(u, 0.0)
    i = _np(i)
    for k in range(len(u)):
        assert i[k] == np.nonzero((pts == u[k]).all(1))[0].min()
    assert (_np(d) == 0).all()
    _check_queries(idx, pts, u, 0.003)
    # radius 0: exactly the queries that coincide with a point
    rng = np.random.RandomState(5)
    q = np.concatenate([u, u + rng.choice([-1, 1], u.shape) * np.spacing(u), u[:10] + [1e-9, 0, 0]])
    for sq in (False, True):
        m = _np(idx.within(q, 0.0, compare_sqrt=sq)).astype(bool)
        assert (m == ((q[:, None, :] == u[None, :, :]).all(2).any(1))).all()
        assert m[:len(u)].all() and not m[len(u):].any()
        assert (m == cloud_ref.within(pts, q, 0.0, compare_sqrt=sq)).all()
    d, i = idx.nearest(q, 0.0)
    assert ((_np(i) >= 0) == m).all()
    # normals: every key at d2 = 0 across several compactions (300 copies > 256 buffer slots)
    for max_nn in (3, 30, 64):
        n, nbr, cnt = cloud.CloudIndex(pts, 0.004).normals(0.004, max_nn, neighbours=True)
        cnt_ref, fixed = _check_normals(pts, n, nbr, cnt, 0.004, max_nn)
        iso = np.nonzero((pts == u[0]).all(1))[0]
        assert (cnt_ref[iso] == max_nn).all() and fixed[iso].all()
        assert (_np(nbr)[iso] == np.sort(iso)[:max_nn]).all()
        z = _np(n)[iso]                                       # (0,0,1), flipped towards the camera at the origin
        assert (z == [0.0, 0.0, -1.0 / (1.0 + 1e-10)]).all()


def _counts_cloud(seed):
    """Points whose neighbourhoods at r hold 1, 2, 3, 4 and up to ~100 points."""
    rng = np.random.RandomState(seed)
    r = 0.002
    iso = []
    for k, m in enumerate([1, 2, 3, 4, 63, 64, 65]):
        c = np.array([0.05 * k, 0.3, 0.5])
        iso.append(c + rng.uniform(-r / 4, r / 4, (m, 3)))   # m points, all within r of each other
    dense = rng.uniform(-0.004, 0.004, (1500, 3)) + [0.0, 0.0, 0.5]
    return np.concatenate(iso + [dense]), r


@pytest.mark.parametrize("max_nn", [1, 2, 3, 63, 64])
def test_max_nn_edges(max_nn):
    pts, r = _counts_cloud(6)
    n, nbr, cnt = cloud.CloudIndex(pts, r).normals(r, max_nn, neighbours=True)
    cnt_ref, fixed = _check_normals(pts, n, nbr, cnt, r, max_nn)
    full = cloud_ref.neighbours(pts, r, 200)[1]
    for c in (1, 2, 3, 4, 63, 64, 65):                         # both sides of 3 and of max_nn are present
        assert (full == c).any()
    assert fixed[cnt_ref < 3].all()
    if max_nn < 3:
        assert fixed.all()
    else:
        assert (~fixed[cnt_ref >= 3]).any()


def test_tiny_clouds_and_refusals():
    """P = 1, 2, 5 (fewer points than one CTA's warps) and the refused arguments."""
    rng = np.random.RandomState(7)
    for P in (1, 2, 5):
        pts = rng.uniform(-0.001, 0.001, (P, 3)) + [0.0, 0.0, 0.4]
        for max_nn in (1, 3, 64):
            n, nbr, cnt = cloud.CloudIndex(pts, 0.003).normals(0.003, max_nn, neighbours=True)
            _check_normals(pts, n, nbr, cnt, 0.003, max_nn)
        idx = cloud.CloudIndex(pts, 0.003)
        _check_queries(idx, pts, rng.uniform(-0.002, 0.002, (9, 3)) + [0.0, 0.0, 0.4], 0.001)
        means, _ = cloud_ref.voxel_down_sample(pts, 0.0005)
        assert (_bits(cloud.voxel_down_sample(pts, 0.0005)) == _bits(means)).all()
    idx = cloud.CloudIndex(rng.uniform(0, 0.01, (50, 3)), 0.003)
    for bad in [dict(radius=0.003, max_nn=0), dict(radius=0.003, max_nn=65), dict(radius=-0.001, max_nn=10),
                dict(radius=float("nan"), max_nn=10), dict(radius=float("inf"), max_nn=10)]:
        with pytest.raises(_lib.CgError):
            idx.normals(**bad)
    for bad_r in (-1e-9, float("nan"), float("inf")):
        with pytest.raises(_lib.CgError):
            idx.within(np.zeros((1, 3)), bad_r, compare_sqrt=False)
        with pytest.raises(_lib.CgError):
            idx.nearest(np.zeros((1, 3)), bad_r)
    with pytest.raises(_lib.CgError):
        cloud.CloudIndex(np.array([[0.0, 0.0, np.nan], [0.0, 0.0, 1.0]]), 0.001)
    n = idx.normals(0.003, 10)                                  # the index still answers
    assert np.isfinite(_np(n)).all()


@pytest.mark.parametrize("shift", [1000.0, -1000.0])
def test_cloud_far_from_the_camera(shift):
    ref = _scene(8, 2000) + [shift, -shift, shift]
    rng = np.random.RandomState(9)
    q = ref[::5] + rng.uniform(-0.004, 0.004, ref[::5].shape)
    r = 3.0 / 1024.0
    _check_queries(cloud.CloudIndex(ref, r), ref, q, r)
    means, _ = cloud_ref.voxel_down_sample(ref, 0.001)
    assert (_bits(cloud.voxel_down_sample(ref, 0.001)) == _bits(means)).all()
    n, nbr, cnt = cloud.CloudIndex(ref, r).normals(r, 30, neighbours=True)
    nbr_ref, cnt_ref = cloud_ref.neighbours(ref, r, 30)
    assert (_np(cnt) == cnt_ref).all() and (_np(nbr) == nbr_ref).all()


def test_cloud_at_the_2_21_cell_limit():
    """x spans exactly 2^21 - 1 cells of 2^-10 (the largest key, 63 bits); half a cell more is refused."""
    c = 2.0 ** -10
    top = (1 << 21) - 1
    rng = np.random.RandomState(10)
    ks = np.concatenate([[0, 1, 2, 3], rng.randint(0, top + 1, 300), top - np.arange(4)])
    yz = rng.randint(0, 4, (len(ks), 2)) * c
    ref = np.concatenate([np.c_[ks * c, yz], np.c_[ks[-4:] * c + 0.25 * c, yz[-4:]]])   # several per top cell
    idx = cloud.CloudIndex(ref, c)
    oc, ncell = (C.c_double * 3)(), C.c_int()
    idx.ctx.check(idx.ctx.lib.cg_cloud_index_info(idx.h, None, C.byref(ncell), None, oc))
    o = np.array(oc[:])
    assert (o == -c / 2).all()
    assert np.floor((ref[:, 0].max() - o[0]) / c) == top
    means, _ = cloud_ref.voxel_down_sample(ref, c)
    assert ncell.value == len(means)
    got, _ = idx.voxel_means()
    assert (_bits(_np(got)) == _bits(means)).all()
    # queries in the top cells, on their faces (x = (k - 1/2) c) and just past the last one
    faces = np.array([top - 0.5, top - 1.5, top + 0.5, top, top - 1, 0.5, -0.5]) * c
    q = np.concatenate([np.c_[faces, np.full(len(faces), c), np.zeros(len(faces))],
                        ref[-12:] + rng.uniform(-c, c, (12, 3)), ref[-8:]])
    for r in (c, 2 * c, 0.5 * c):
        _check_queries(idx, ref, q, r)
    half = np.array([[0.0, 0.0, 0.0], [(top + 0.5) * c, 0.0, 0.0]])
    with pytest.raises(_lib.CgError, match="2\\^21"):
        cloud.CloudIndex(half, c)


def test_queries_exactly_r_outside_the_box():
    """Queries exactly r from a corner point of the cloud, outside its bounding box on a face, an edge and a corner
    (dyadic offsets with integer norms: (5,0,0), (3,4,0), (2,2,1)), and one ulp farther; NaN / inf queries; Q = 0."""
    rng = np.random.RandomState(11)
    u = 2.0 ** -10
    ref = rng.randint(0, 16, (400, 3)) * u + [0.0, 0.0, 0.5]
    ref = np.concatenate([ref, [[16 * u, 16 * u, 0.5 + 16 * u]]])           # the box's top corner is a point
    p = ref[-1]
    for r_units, offs in [(5, [(5, 0, 0), (0, 5, 0), (0, 0, 5)]), (5, [(3, 4, 0), (0, 3, 4), (4, 0, 3)]),
                          (3, [(2, 2, 1), (1, 2, 2), (2, 1, 2)])]:
        r = r_units * u
        q = p + np.array(offs, np.float64) * u
        qf = np.nextafter(q, np.inf)
        for cell in (r, r / 4, 4 * r, u):
            idx = cloud.CloudIndex(ref, cell)
            _check_queries(idx, ref, np.concatenate([q, qf]), r)
            m = _np(idx.within(q, r, compare_sqrt=False)).astype(bool)
            assert m.all()
            assert not _np(idx.within(qf, r, compare_sqrt=False)).any()
            _, i = idx.nearest(q, r)
            assert (_np(i) == len(ref) - 1).all()


def test_bad_and_empty_queries():
    rng = np.random.RandomState(12)
    ref = rng.uniform(-0.01, 0.01, (500, 3)) + [0.0, 0.0, 0.5]
    nan, inf = np.nan, np.inf
    q = np.array([[nan, 0, 0.5], [0, nan, 0.5], [0, 0, nan], [inf, 0, 0.5], [-inf, 0, 0.5], [0, inf, 0.5],
                  [0, 0, -inf], [nan, nan, nan], [inf, inf, inf], [inf, -inf, nan]])
    q = np.concatenate([q, ref[:3]])
    for cell in (0.001, 0.01):
        idx = cloud.CloudIndex(ref, cell)
        for r in (0.0, 0.002, 10.0):
            d, i = idx.nearest(q, r)
            d, i = _np(d), _np(i)
            assert (i[:10] == -1).all() and (d[:10] == np.inf).all()
            assert (i[10:] == [0, 1, 2]).all()
            for sq in (False, True):
                m = _np(idx.within(q, r, compare_sqrt=sq))
                assert (m[:10] == 0).all() and (m[10:] == 1).all()
            _check_queries(idx, ref, q, r)
        d, i = idx.nearest(np.zeros((0, 3)), 0.002)
        assert d.shape == (0,) and i.shape == (0,)
        assert _np(idx.within(np.zeros((0, 3)), 0.002, compare_sqrt=True)).shape == (0,)


K_SMALL = np.array([[610.5, 0.0, 16.25], [0.0, 611.75, 3.5], [0.0, 0.0, 1.0]])


def _depth(shape, dtype, seed):
    rng = np.random.RandomState(seed)
    d = rng.uniform(0.05, 1.5, shape).astype(dtype)
    flat = d.reshape(-1)
    special = np.array([np.nan, np.inf, -np.inf, -0.5, -0.0, 0.0, 0.1, np.nextafter(dtype(0.1), dtype(0))], dtype)
    k = min(len(special), flat.size)
    pos = rng.choice(flat.size, k, replace=False)
    flat[pos] = special[:k] if flat.size > 1 else special[rng.randint(len(special))]
    return d


def _same_xyz(got, want):
    """Bit-identical, except that a NaN only has to be a NaN (payload and sign are not part of the contract)."""
    got, want = _np(got), _np(want)
    gn, wn = np.isnan(got), np.isnan(want)
    assert (gn == wn).all()
    assert (_bits(got)[~gn] == _bits(want)[~wn]).all()


@pytest.mark.parametrize("shape", [(1, 1), (1, 17), (13, 1), (7, 33)])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_depth2xyz_shapes_and_non_finite_depths(shape, dtype):
    for seed in range(3 if shape == (1, 1) else 1):
        depth = _depth(shape, dtype, seed)
        got = cloud.depth2xyzmap(depth, K_SMALL)
        assert got.shape == shape + (3,) and got.dtype == np.float32
        _same_xyz(got, cloud_ref.depth2xyzmap(depth, K_SMALL))
    depth = _depth(shape, dtype, 99)
    want = cloud_ref.depth2xyzmap(depth, K_SMALL)
    if depth.size > 1:
        z = want.reshape(-1, 3)[:, 2]
        assert np.isnan(z).any() and np.isinf(z).any() and (z == 0).any()      # the specials went through
    # a tensor produced on a side stream, consumed on that stream
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        src = torch.from_numpy(depth).cuda(non_blocking=False)
        t = (src * 2) / 2                                                      # exact; written on stream s
        out = cloud.depth2xyzmap(t, K_SMALL)
    s.synchronize()
    assert out.is_cuda
    _same_xyz(out, want)
