"""The mesh -> signed-distance grid builder (csrc/cg_sdf_build.cu, Sdf3D.from_mesh) at its grid, brick, tile and
lattice edges.

The sign is checked against oracle/sdf_parity_exact.py, the exact ray parity of the builder's contract on the
unsnapped mesh, wherever a node is farther than res * 2^-16 from the surface (twice the snap bound the builder
claims); the magnitude against float32(|d|) of oracle/sdf_mesh_ref.c bit for bit.  CPU tests pin the parity oracle to
analytic inside tests, to the winding number on closed non-overlapping meshes and to hand-counted crossings.

GPU cases: extents of k cells and k +- a fraction on both sides of the 1e-4 cell tolerance on each axis, padding 0
and 1, the 2048-node axis limit, single-node axes (closed zero-thickness meshes), every residue of the 4x8x8 brick and
2x4x4 warp sub-brick, face counts around the 32-triangle tile, more than 256 tiles in separated components, one large
triangle pair beside many small tiles, flat meshes (Morton scale 0), meshes 1, 10 and 100 m from the origin, vertices
on the grid lines of a non-dyadic resolution, vertex fans and edges on grid lines, vertices on node x-planes, boxes
that share a face or an edge, and overlapping boxes (positive in the overlap: the parity rule).  Every case builds
twice, bitwise equal, and with its most-crossed triangle removed is refused as not closed."""
import numpy as np
import pytest

from catgrasp_b200.synthetic import _box_mesh, hex_nut_mesh_inside, make_hex_nut_mesh, tessellated_box_mesh
from oracle.sdf_mesh_ref import grid_geometry, node_positions, sdf_mesh_ref
from oracle.sdf_parity_exact import crossings, parity_grid, parity_lines
from test_sdf_build import (PARITY_TOL, GPU_CASES, _cuda, _gpu_case, _hull_mesh, _raw_build, _shell_mesh, check_nodes,
                            report)

R = 2.0 ** -10                  # a dyadic resolution: node coordinates and mesh coordinates coincide exactly


def _join(*meshes):
    Vs, Fs, off = [], [], 0
    for V, F in meshes:
        Vs.append(np.asarray(V, np.float64)); Fs.append(np.asarray(F, np.int64) + off); off += len(V)
    return np.concatenate(Vs), np.concatenate(Fs).astype(np.int32)


def _box(lo, hi):
    return _box_mesh(np.asarray(lo, np.float64), np.asarray(hi, np.float64))


def bipyramid(center, axis, r, h, n, phase=0.0):
    """Closed double pyramid: a ring of n vertices of radius r (or radii (r_b, r_c) along the next two axes) around
    ``axis`` through ``center`` and two apexes at +-h along it; 2n outward faces, n around each apex."""
    a, b, c = axis, (axis + 1) % 3, (axis + 2) % 3
    rb, rc = np.broadcast_to(np.asarray(r, np.float64), (2,))
    th = phase + 2 * np.pi * np.arange(n) / n
    V = np.zeros((n + 2, 3))
    V[:n, b], V[:n, c] = rb * np.cos(th), rc * np.sin(th)
    V[n, a], V[n + 1, a] = h, -h
    V += np.asarray(center, np.float64)
    i = np.arange(n)
    F = np.concatenate([np.stack([i, (i + 1) % n, np.full(n, n)], 1), np.stack([(i + 1) % n, i, np.full(n, n + 1)], 1)])
    return V, F.astype(np.int32)


def zero_thickness(axis, center, size):
    """Two coincident, opposite triangles in the plane through ``center`` normal to ``axis``: closed, no volume."""
    b, c = (axis + 1) % 3, (axis + 2) % 3
    V = np.tile(np.asarray(center, np.float64), (3, 1))
    V[1, b] += size
    V[2, c] += size
    return V, np.array([[0, 1, 2], [0, 2, 1]], np.int32)


def flat_sheet(axis, lo, size, m):
    """An m x m tessellated square in a plane normal to ``axis``, with every triangle also in the opposite winding."""
    b, c = (axis + 1) % 3, (axis + 2) % 3
    t = np.arange(m + 1) / m * size
    gb, gc = np.meshgrid(t, t, indexing="ij")
    V = np.tile(np.asarray(lo, np.float64), ((m + 1) ** 2, 1))
    V[:, b] += gb.reshape(-1)
    V[:, c] += gc.reshape(-1)
    q = (np.arange(m)[:, None] * (m + 1) + np.arange(m)[None, :]).reshape(-1)
    F = np.concatenate([np.stack([q, q + m + 1, q + m + 2], 1), np.stack([q, q + m + 2, q + 1], 1)])
    return V, np.concatenate([F, F[:, ::-1]]).astype(np.int32)


# ------------------------------------------------------------------ the cases
BRICK_SIZES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17]     # every residue of 4 and 8, around one and two bricks
TOL_STEPS = {"m2e-4": -2e-4, "m5e-5": -5e-5, "0": 0.0, "p5e-5": 5e-5, "p2e-4": 2e-4}
TILE_FACES = [4, 31, 32, 33, 64, 65]
FAR = [1, -1, 10, -10, 100, -100]


def _extent_case(axis, k, step, pad):
    """A box whose extent along ``axis`` is k + step cells and 3 cells on the other axes."""
    lo = np.array([0.25, -0.5, 0.125])
    ext = np.full(3, 3.0)
    ext[axis] = k + TOL_STEPS[step]
    V, F = _box(lo, lo + ext * R)
    dims = np.full(3, 4 + 2 * pad)
    dims[axis] = k + 1 + (TOL_STEPS[step] > 1e-4) + 2 * pad
    return V, F, dims


def _tile_mesh(nf):
    """A closed mesh with exactly nf faces around the world origin: a tetrahedron, or a double pyramid padded with one
    zero-area triangle (apex, ring vertex, ring vertex) for an odd count."""
    if nf == 4:
        V = np.array([[-5, -4, -3], [6, -4, -3], [0, 7, -3], [1, 0, 6]], np.float64) * R
        return V, np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]], np.int32)
    V, F = bipyramid([0.1 * R, -0.2 * R, 0.3 * R], 2, 6.3 * R, 5.2 * R, nf // 2, phase=0.1)
    if nf % 2:
        F = np.concatenate([F, [[nf // 2, 0, 0]]]).astype(np.int32)
    assert F.shape[0] == nf
    return V, F


def _anchor():
    """A 2-cell box at the world origin: with it, every coordinate of the form c * R is a node coordinate."""
    return _box([0, 0, 0], [2 * R] * 3)


def edge_case(name):
    """(V, F, res, pad, expected dims or None, winding): winding is False where parity and winding number differ."""
    p = name.split("_")
    if p[0] == "extent":                                        # extent_<axis>_<k>_<step>_pad<p>
        pad = int(p[4][3:])
        V, F, dims = _extent_case(int(p[1]), int(p[2]), p[3], pad)
        return V, F, R, pad, dims, True
    if p[0] == "limit":                                         # limit_<axis>_<cells>_pad<p>: nodes = cells + 1 + 2p
        axis, cells, pad = int(p[1]), int(p[2]), int(p[3][3:])
        hi = np.full(3, 2 * R)
        hi[axis] = cells * R
        dims = np.full(3, 3 + 2 * pad)
        dims[axis] = cells + 1 + 2 * pad
        return (*_box([0, 0, 0], hi), R, pad, dims, True)
    if p[0] == "single":                                        # single_<axis>_pad<p>: a one-node axis at padding 0
        axis, pad = int(p[1]), int(p[2][3:])
        V, F = zero_thickness(axis, [3 * R, -2 * R, 5 * R], 5 * R)
        dims = np.full(3, 6 + 2 * pad)
        dims[axis] = 1 + 2 * pad
        return V, F, R, pad, dims, True
    if p[0] == "brick":                                         # brick_<nx>x<ny>x<nz>, padding 0
        n = np.array([int(v) for v in p[1].split("x")])
        a = int(np.argmax(n))                                   # a 96-face double pyramid spanning exactly n - 1 cells
        half = (n - 1) * R / 2
        V, F = bipyramid(np.array([0.0123, -0.0457, 0.0311]) + half, a, (half[(a + 1) % 3], half[(a + 2) % 3]),
                         half[a], 48)
        return V, F, R, 0, n, True
    if p[0] == "tiles":                                         # tiles_<nf>
        V, F = _tile_mesh(int(p[1]))
        return V, F, R, 2, None, True
    if name == "many_tiles":                                    # 3 x 8748 triangles in three separated components
        V, F = _join(tessellated_box_mesh([0, 0, 0], [0.01, 0.008, 0.006], 27),
                     tessellated_box_mesh([0.04, 0.001, 0.0], [0.05, 0.009, 0.007], 27),
                     tessellated_box_mesh([0.02, 0.012, 0.002], [0.026, 0.02, 0.008], 27))
        return V, F, 0.001, 2, None, True
    if name == "big_pair_small_tiles":                          # a slab with 40 x 40 mm faces beside 54 small tiles
        V, F = _join(_box([-0.02, -0.02, 0.0], [0.02, 0.02, 0.002]),
                     tessellated_box_mesh([-0.004, -0.006, 0.004], [0.006, 0.004, 0.009], 12))
        return V, F, 0.001, 2, None, True
    if p[0] == "flat":                                          # flat_<axis>: Morton scale 0 on that axis
        V, F = flat_sheet(int(p[1]), [0.003, -0.004, 0.002], 0.012, 10)
        return V, F, 0.001, 1, None, True
    if p[0] == "far":                                           # far_<mesh>_<offset>: moved by offset * (1, -1, 1) m
        off = float(p[2]) * np.array([1.0, -1.0, 1.0])
        if p[1] == "hull":
            V, F, _ = _hull_mesh(0)
        else:
            V, F = tessellated_box_mesh([0.001, 0.002, -0.003], [0.009, 0.0075, 0.0021], 3)
        return V + off, F, 0.001, int(p[2] in ("-1", "10", "-100")), None, True
    if p[0] == "lattice1mm":                                    # lattice1mm_pad<p>: vertices on the 1 mm lines
        mm = 0.001
        V, F = _join(_box(np.array([3, -2, 5]) * mm, np.array([9, 4, 9]) * mm),
                     tessellated_box_mesh(np.array([9, -1, 5]) * mm, np.array([15, 5, 11]) * mm, 6))
        return V, F, mm, int(p[1][3:]), None, True
    if p[0] == "fan":                                           # fan_<n>_<axis>: apexes and ring on grid lines
        n, axis = int(p[1]), int(p[2])
        V, F = _join(_anchor(), bipyramid([10 * R, 10 * R, 10 * R], axis, 4 * R, 3 * R, n))
        return V, F, R, 1, None, True
    if name == "shared_face":
        V, F = _join(_box([0, 0, 0], np.array([4, 4, 4]) * R), _box(np.array([4, 0, 0]) * R, np.array([8, 4, 4]) * R))
        return V, F, R, 1, None, True
    if name == "shared_edge":
        V, F = _join(_box([0, 0, 0], np.array([4, 4, 4]) * R), _box(np.array([4, 4, 0]) * R, np.array([8, 8, 4]) * R))
        return V, F, R, 1, None, True
    if name == "overlap":                                       # the overlap is outside by parity, inside by winding
        V, F = _join(_box([0, 0, 0], np.array([6, 4, 4]) * R), _box(np.array([3, 1, 1]) * R, np.array([9, 5, 3]) * R))
        return V, F, R, 1, None, False
    if name == "overlap_1mm":
        V, F = _join(_box([0.0, 0.0, 0.0], [0.006, 0.004, 0.004]),
                     _box([0.0033, 0.0011, 0.0007], [0.009, 0.005, 0.003]),
                     tessellated_box_mesh([0.001, 0.0005, 0.0012], [0.0045, 0.0035, 0.0052], 3))
        return V, F, 0.001, 2, None, False
    raise KeyError(name)


EDGE_CASES = (
    [f"extent_{a}_{k}_{s}_pad{(a + k) % 2}" for a in range(3) for k in (1, 6) for s in TOL_STEPS] +
    [f"limit_{a}_2047_pad0" for a in range(3)] + ["limit_1_2045_pad1"] +
    [f"single_{a}_pad{pad}" for a in range(3) for pad in (0, 1)] +
    [f"brick_{BRICK_SIZES[i]}x{BRICK_SIZES[(i + 5) % 12]}x{BRICK_SIZES[(i + 9) % 12]}" for i in range(12)] +
    [f"tiles_{nf}" for nf in TILE_FACES] + ["many_tiles", "big_pair_small_tiles"] + [f"flat_{a}" for a in range(3)] +
    [f"far_{m}_{d}" for m in ("hull", "tess") for d in FAR] + ["lattice1mm_pad0", "lattice1mm_pad1"] +
    [f"fan_{n}_{a}" for n in range(3, 9) for a in (0, 1)] + ["shared_face", "shared_edge", "overlap", "overlap_1mm"])

# Double pyramids whose ring extremes lie within float32 rounding of a grid line (< res * 2^-17): every line that
# crosses them grazes a vertex, where the snap, not the exact geometry, decides whether it crosses.  A removed face
# need not open such a mesh on the snapped lattice.
GRAZED = {"brick_5x15x2", "brick_6x16x3", "brick_9x2x6"}


def _flat_in_yz(V, F):
    """every face has zero area in (y, z): no line crosses the mesh, so a removed face cannot be seen"""
    a, b, c = (V[F[:, e]][:, 1:] for e in range(3))
    return bool(np.all((b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) == (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0])))


def _all_nodes(dims):
    return np.stack(np.meshgrid(*[np.arange(d) for d in dims], indexing="ij"), -1).reshape(-1, 3)


def _decided_parity(V, F, res, pad):
    """(sd, inside by parity, winding number) at every node of the grid the builder makes"""
    dims, origin, r32 = grid_geometry(V, res, pad)
    sd, wind = sdf_mesh_ref(V, F, node_positions(origin, r32, _all_nodes(dims)))
    inside, open_, _ = parity_grid(V, F, origin, r32, dims)
    assert not open_.any()
    return sd, inside.reshape(-1), wind, float(r32)


# ------------------------------------------------------------------ CPU: the parity oracle
def test_parity_of_boxes_is_the_analytic_inside():
    rng = np.random.RandomState(0)
    for _ in range(6):
        lo = rng.uniform(-0.01, 0.01, 3)
        hi = lo + rng.uniform(0.002, 0.012, 3)
        V, F = _box(lo, hi)
        res = float(rng.choice([0.001, 0.0007, R]))
        dims, origin, r32 = grid_geometry(V, res, 2)
        P = node_positions(origin, r32, _all_nodes(dims))
        inside = parity_grid(V, F, origin, r32, dims)[0].reshape(-1)
        ana = ((P > lo) & (P < hi)).all(1)
        clear = (np.abs(P - lo).min(1) > 1e-12) & (np.abs(P - hi).min(1) > 1e-12)
        assert ana[clear].sum() > 0 and np.array_equal(inside[clear], ana[clear])


def test_parity_of_nested_shells_has_the_cavity_outside():
    V, F = _shell_mesh()
    V2, F2 = _join((V, F), (V * 0.5 + 0.003, F))            # a second, smaller shell inside the cavity
    for V, F, n_shells in ((V, F, 1), (V2, F2, 2)):
        dims, origin, r32 = grid_geometry(V, 0.0005, 2)
        P = node_positions(origin, r32, _all_nodes(dims))
        inside = parity_grid(V, F, origin, r32, dims)[0].reshape(-1)
        ana = np.zeros(P.shape[0], bool)
        clear = np.ones(P.shape[0], bool)
        for s in range(n_shells):
            Vs = V[16 * s:16 * s + 16]
            for lo, hi in ((Vs[:8].min(0), Vs[:8].max(0)), (Vs[8:].min(0), Vs[8:].max(0))):
                ana ^= ((P > lo) & (P < hi)).all(1)
                clear &= (np.abs(P - lo).min(1) > 1e-12) & (np.abs(P - hi).min(1) > 1e-12)
        assert ana[clear].sum() > 100 and (~ana[clear]).sum() > 100
        assert np.array_equal(inside[clear], ana[clear])


def test_parity_of_hex_nut_is_the_analytic_inside():
    V, F = make_hex_nut_mesh()
    sd, inside, _, res = _decided_parity(V, F, 0.0005, 3)
    dims, origin, r32 = grid_geometry(V, 0.0005, 3)
    ana = hex_nut_mesh_inside(node_positions(origin, r32, _all_nodes(dims)))
    clear = np.abs(sd) > 1e-9
    assert ana[clear].sum() > 2000 and np.array_equal(inside[clear], ana[clear])


@pytest.mark.parametrize("name", [c for c in GPU_CASES if c != "proxy_tess200k"] +
                         [c for c in EDGE_CASES if not c.startswith(("limit", "many"))])
def test_parity_equals_winding_number_on_closed_meshes(name):
    """Where the two rules coincide (closed, non-overlapping meshes), the exact parity is the winding-number sign at
    every node farther than res * 2^-16 from the surface; on overlapping boxes they differ exactly in the overlap."""
    if name in GPU_CASES:
        V, F, res, pad, _ = _gpu_case(name)
        winding = True
    else:
        V, F, res, pad, _, winding = edge_case(name)
    sd, inside, wind, r = _decided_parity(V, F, res, pad)
    far = np.abs(sd) > r * PARITY_TOL
    assert np.all(np.abs(wind[far] - np.round(wind[far])) < 1e-6)
    if winding:
        assert np.array_equal(inside[far], (sd < 0)[far])
        assert np.all(np.round(np.abs(wind[far])) <= 1)
    else:
        twice = far & (np.round(wind) == 2)
        assert twice.sum() > 0 and not inside[twice].any()
        assert np.array_equal(inside[far & ~twice], (sd < 0)[far & ~twice])


def test_parity_counts_a_vertex_fan_once():
    """Lines through the apex and the ring centre of a double pyramid meet 2n triangles at one vertex each: by hand,
    one crossing at each apex.  A line through a ring vertex's projected edges: one crossing on each side."""
    for n in range(3, 9):
        V, F = bipyramid([0.0, 0.0, 0.0], 0, 1.0, 0.5, n)
        got = crossings(V, F, 0.0, 0.0)
        assert [x for x, _ in got] == [-0.5, 0.5]
        assert F[got[0][1], 2] == n + 1 and F[got[1][1], 2] == n       # the bottom apex's fan, then the top's
        y, z = 0.5 * V[0, 1], 0.5 * V[0, 2]                            # on the projection of both apex -> ring 0 edges
        got = crossings(V, F, y, z)
        assert len(got) == 2 and got[0][0] == -got[1][0] and got[1][0] > 0
    # the axis in the ring's plane: a fan of side faces whose projections overlap, seen edge-on at the ring vertices
    V, F = bipyramid([0.0, 0.0, 0.0], 1, 1.0, 0.5, 4)                   # ring in the xz-plane, apexes on y
    V = np.round(V, 12)                                                # ring at z = 1, 0, -1, 0 and x = 0, 1, 0, -1
    for y, z, n_cross in ((0.0, 0.0, 2), (0.5, 0.0, 0), (-0.5, 0.0, 2), (0.0, 1.0, 0), (0.0, -1.0, 0),
                          (0.25, 0.25, 2), (0.25, -0.25, 2), (-0.25, 0.25, 2), (0.5, 1.0, 0)):
        got = crossings(V, F, y, z)
        assert len(got) == n_cross, (y, z, got)


def test_parity_counts_a_shared_edge_once():
    V, F = _box([0.0, 0.0, 0.0], [1.0, 1.0, 1.0])
    # the line through both caps' diagonals: one crossing per cap
    assert [x for x, _ in crossings(V, F, 0.5, 0.5)] == [0, 1]
    # lines along the box's x edges: the line moved by (eps, eps^2) is inside only at the (y0, z0) edge
    assert [x for x, _ in crossings(V, F, 0.0, 0.0)] == [0, 1]
    for y, z in ((1.0, 0.0), (0.0, 1.0), (1.0, 1.0)):
        assert crossings(V, F, y, z) == []
    # along a face's edge in y: the line lies in the faces z = 0; moved by +eps^2 in z it is inside
    assert [x for x, _ in crossings(V, F, 0.5, 0.0)] == [0, 1]
    assert crossings(V, F, 0.5, 1.0) == []
    # two boxes sharing the face x = 1: the line crosses it twice, once per box
    V2, F2 = _join((V, F), (V + [1.0, 0.0, 0.0], F))
    assert [x for x, _ in crossings(V2, F2, 0.5, 0.25)] == [0, 1, 1, 2]


def test_parity_reports_open_lines():
    V, F = _box(np.zeros(3), np.array([4, 4, 4]) * R)
    dims, origin, r32 = grid_geometry(V, R, 1)
    _, open_, hits = parity_grid(V, F, origin, r32, dims)
    assert not open_.any() and hits.sum() == 4 * 4 * 2         # the 4 x 4 lines with y, z in [0, 4R), once per cap
    f = int(np.argmax(hits))
    _, open_, _ = parity_grid(V, np.delete(F, f, 0), origin, r32, dims)
    assert open_.sum() == hits[f]


# ------------------------------------------------------------------ GPU: the builder at its edges
@pytest.mark.gpu
@pytest.mark.parametrize("name", EDGE_CASES)
def test_builder_at_edges(name, capsys):
    _cuda()
    from catgrasp_b200 import _lib
    from catgrasp_b200.sdf import Sdf3D
    V, F, res, pad, expect, winding = edge_case(name)
    built = Sdf3D.from_mesh(V, F, res, pad)
    dims, origin, res32 = grid_geometry(V, res, pad)
    assert np.array_equal(built.dims_, dims) and np.array_equal(built.origin_, origin)
    assert built.resolution_ == float(res32)
    if expect is not None:
        assert np.array_equal(dims, expect), (dims, expect)
    stats = check_nodes(built, V, F, _all_nodes(dims), winding)
    report(capsys, name, stats)
    assert stats[2] == 0
    again = Sdf3D.from_mesh(V, F, res, pad)
    assert np.array_equal(again.data_.view(np.uint32), built.data_.view(np.uint32))
    if not winding:                                            # overlapping boxes: the overlap is outside
        sd, wind = sdf_mesh_ref(V, F, node_positions(origin, res32, _all_nodes(dims)))
        twice = (np.round(wind) == 2) & (np.abs(sd) > float(res32) * PARITY_TOL)
        assert twice.sum() > 0 and (built.data_.reshape(-1)[twice] > 0).all()
    # the mesh without its most-crossed triangle is open
    hits = parity_lines(V, F, origin, res32, dims)[2]
    if _flat_in_yz(V, F):
        assert hits.max() == 0
        return
    if name in GRAZED:
        return
    f = int(np.argmax(hits))
    assert hits[f] > 0
    rc, h, msg = _raw_build(V, np.delete(F, f, 0), res, pad)
    assert rc == _lib.CG_EINVAL and not h and "not closed" in msg, (rc, msg)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_builder_axis_limit(axis):
    """2048 nodes along an axis are built (their values are checked in test_builder_at_edges), 2049 are refused."""
    _cuda()
    from catgrasp_b200 import _lib
    for cells, pad, ok in ((2047, 0, True), (2045, 1, True), (2048, 0, False), (2046, 1, False), (2047, 1, False)):
        hi = np.full(3, 2 * R)
        hi[axis] = cells * R
        V, F = _box([0, 0, 0], hi)
        assert grid_geometry(V, R, pad)[0][axis] == cells + 1 + 2 * pad
        rc, h, msg = _raw_build(V, F, R, pad)
        if ok:
            assert rc == _lib.CG_OK and h, msg
        else:
            assert rc == _lib.CG_EINVAL and not h and "2048" in msg, (cells, pad, rc, msg)
