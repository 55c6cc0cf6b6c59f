"""Exact ray-parity sign of the mesh -> signed-distance grid builder -- ORACLE, test infrastructure only.

csrc/cg_sdf_build.cu decides the sign of a node by ray parity along +x, on a fixed-point copy of the mesh whose yz
coordinates are snapped to 2^16 steps per cell.  oracle/sdf_mesh_ref.c signs by winding number, which agrees with
parity only on closed, non-overlapping meshes.  This module states the builder's contract (include/catgrasp_b200.h,
cg_sdf_from_mesh) on the unsnapped float64 mesh, in exact integer arithmetic:

* every float64 input is a dyadic rational: the vertex coordinates, and the node coordinates
  ``float64(origin) + float64(i * float64(res))`` rounded as the builder rounds them.  All y and z values are scaled
  by one power of two to Python integers, all x values by another;
* the line of node (j, k) is {(x, y_j, z_k)}.  A triangle whose projection on (y, z) has zero area is never crossed;
* a line through an edge or a vertex is moved by (eps, eps^2) in (y, z), eps -> 0+.  For an edge s -> t of a
  counter-clockwise projected triangle, ``w = orient(s, t, p)`` becomes ``w + du eps^2 - dv eps`` with (du, dv) = t - s,
  so w == 0 counts as inside iff dv < 0, or dv == 0 and du > 0.  Every line then meets a closed mesh an even number
  of times;
* a crossing at ``x_c = (w_a a_x + w_b b_x + w_c c_x) / W`` (w_a = orient(b, c, p), ...) counts for the nodes with
  x_i > x_c, compared exactly as x_i W > w_a a_x + w_b b_x + w_c c_x; a node is inside when an odd number of crossings
  count for it;
* a line with an odd total is open.

Nothing here snaps, rounds or shares the builder's arithmetic.  Pure Python over the (triangle, line) pairs whose
bounding boxes meet: fine for meshes of up to a few hundred thousand small triangles.
"""
from bisect import bisect_left, bisect_right
from fractions import Fraction

import numpy as np

from oracle.sdf_mesh_ref import node_positions


def _to_ints(values):
    """(ints, e): values[n] == ints[n] * 2**-e exactly, for float64 values"""
    fr = [float(v).as_integer_ratio() for v in np.asarray(values, np.float64).reshape(-1)]
    e = max(d.bit_length() - 1 for _, d in fr)
    return [n << (e - (d.bit_length() - 1)) for n, d in fr], e


def _orient(au, av, bu, bv, pu, pv):
    return (bu - au) * (pv - av) - (bv - av) * (pu - au)


def _edge_in(w, du, dv):
    """p on the inner side of edge s -> t (w = orient(s, t, p), (du, dv) = t - s) after the (eps, eps^2) move"""
    if w != 0:
        return w > 0
    return dv < 0 if dv != 0 else du > 0


class _Mesh:
    """yz of every vertex as integers on the scale 2**-eyz, x on the scale 2**-ex, together with extra yz / x values"""

    def __init__(self, vertices, faces, extra_yz=(), extra_x=()):
        V = np.asarray(vertices, np.float64).reshape(-1, 3)
        self.F = np.asarray(faces, np.int64).reshape(-1, 3)
        nv = V.shape[0]
        yz, _ = _to_ints(np.concatenate([V[:, 1], V[:, 2], np.asarray(extra_yz, np.float64)]))
        x, _ = _to_ints(np.concatenate([V[:, 0], np.asarray(extra_x, np.float64)]))
        self.u, self.v, self.extra_yz = yz[:nv], yz[nv:2 * nv], yz[2 * nv:]
        self.x, self.extra_x = x[:nv], x[nv:]

    def triangle(self, f):
        """(W, a, b, c), the vertices (u, v, x) ordered counter-clockwise in (y, z); W = 0: zero projected area"""
        a, b, c = ((self.u[i], self.v[i], self.x[i]) for i in self.F[f])
        W = _orient(a[0], a[1], b[0], b[1], c[0], c[1])
        if W < 0:
            b, c, W = c, b, -W
        return W, a, b, c


def _crossing(W, a, b, c, pu, pv):
    """None if the line (pu, pv) misses the counter-clockwise triangle, else the numerator N of x_c = N / W"""
    wa = _orient(b[0], b[1], c[0], c[1], pu, pv)
    wb = _orient(c[0], c[1], a[0], a[1], pu, pv)
    wc = _orient(a[0], a[1], b[0], b[1], pu, pv)
    if not (_edge_in(wa, c[0] - b[0], c[1] - b[1]) and _edge_in(wb, a[0] - c[0], a[1] - c[1]) and
            _edge_in(wc, b[0] - a[0], b[1] - a[1])):
        return None
    assert wa + wb + wc == W
    return wa * a[2] + wb * b[2] + wc * c[2]


def crossings(vertices, faces, y, z):
    """Sorted [(x_c as a Fraction, face index)] of the line {(x, y, z)} (y, z float64) with the mesh."""
    V = np.asarray(vertices, np.float64).reshape(-1, 3)
    m = _Mesh(V, faces, extra_yz=[y, z])
    ex = _to_ints(V[:, 0])[1]
    out = []
    for f in range(m.F.shape[0]):
        W, a, b, c = m.triangle(f)
        if W == 0:
            continue
        N = _crossing(W, a, b, c, m.extra_yz[0], m.extra_yz[1])
        if N is not None:
            out.append((Fraction(N, W) / 2 ** ex, f))
    return sorted(out)


def parity_lines(vertices, faces, origin, res, dims, lines=None):
    """Ray parity of the nodes of the grid (float32 origin (3,), float32 res, dims (3,)) on the given lines.

    lines: (L, 2) int (j, k), default every line in (j, k) raster order.  Returns inside (L, nx) bool, open (L,) bool
    and hits (nf,) int, the number of the given lines that cross each face."""
    nx, ny, nz = (int(d) for d in dims)
    if lines is None:
        lines = np.stack(np.meshgrid(np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 2)
    lines = np.asarray(lines, np.int64).reshape(-1, 2)
    line_of = {(int(j), int(k)): n for n, (j, k) in enumerate(lines)}
    nodes = [node_positions(origin, res, np.stack([np.arange(n)] * 3, 1))[:, a] for a, n in enumerate((nx, ny, nz))]
    m = _Mesh(vertices, faces, extra_yz=np.concatenate([nodes[1], nodes[2]]), extra_x=nodes[0])
    Y, Z, X = m.extra_yz[:ny], m.extra_yz[ny:], m.extra_x
    assert all(p < q for p, q in zip(X, X[1:])) and all(p < q for p, q in zip(Y, Y[1:])) and \
        all(p < q for p, q in zip(Z, Z[1:]))
    slots = [[] for _ in range(len(lines))]
    hits = np.zeros(m.F.shape[0], np.int64)
    for f in range(m.F.shape[0]):
        W, a, b, c = m.triangle(f)
        if W == 0:
            continue
        us, vs = (a[0], b[0], c[0]), (a[1], b[1], c[1])
        j0, j1 = bisect_left(Y, min(us)), bisect_right(Y, max(us))
        k0, k1 = bisect_left(Z, min(vs)), bisect_right(Z, max(vs))
        for j in range(j0, j1):
            for k in range(k0, k1):
                n = line_of.get((j, k))
                if n is None:
                    continue
                N = _crossing(W, a, b, c, Y[j], Z[k])
                if N is not None:
                    slots[n].append(bisect_right(X, N // W))   # first node with x_i W > N
                    hits[f] += 1
    inside = np.zeros((len(lines), nx), bool)
    open_ = np.zeros(len(lines), bool)
    for n, s in enumerate(slots):
        if s:
            run = np.cumsum(np.bincount(s, minlength=nx + 1))
            inside[n] = (run[:nx] & 1).astype(bool)
            open_[n] = bool(run[nx] & 1)
    return inside, open_, hits


def parity_grid(vertices, faces, origin, res, dims):
    """parity_lines over every line: inside (nx, ny, nz) bool, open (ny, nz) bool, hits (nf,) int"""
    nx, ny, nz = (int(d) for d in dims)
    inside, open_, hits = parity_lines(vertices, faces, origin, res, dims)
    return inside.reshape(ny, nz, nx).transpose(2, 0, 1), open_.reshape(ny, nz), hits
