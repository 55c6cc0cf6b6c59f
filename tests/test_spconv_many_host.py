"""The batched site tables' key layout and row bound (catgrasp_b200.spconv: key_layout, down_rows), restated in numpy
and checked against oracle/spconv_ref.py's one-frame tables concatenated.  CPU only.

A batched level keys site (x, y, z) of frame b as b << 3w | x << 2w | y << w | z.  The restatement below builds the
batched level from those keys alone (np.unique, np.searchsorted, neighbours bounded by the w-bit field) and must give
every frame's one-frame level, p2v and tables, each plus the frame's row base.
"""
import numpy as np
import pytest

from catgrasp_b200 import spconv
from oracle import spconv_ref as R


def _layout(shapes):
    """The width rule, restated: (f, w) or None when the batch does not fit a 63-bit key."""
    if len(shapes) == 1:
        return 0, 21
    f = int(np.ceil(np.log2(len(shapes))))
    w = int(np.ceil(np.log2(max(max(s) for s in shapes))))
    return (f, w) if f + 3 * w <= 63 else None


def _pack(b, c, w):
    c = np.asarray(c, dtype=np.int64).reshape(-1, 3)
    return (np.int64(b) << 3 * w) | (c[:, 0] << 2 * w) | (c[:, 1] << w) | c[:, 2]


def _unpack(k, w):
    m = (1 << w) - 1
    return (k >> 3 * w), np.stack([(k >> 2 * w) & m, (k >> w) & m, k & m], 1).astype(np.int32)


def _neighbours(keys, w):
    frame, vox = _unpack(keys, w)
    nbr = np.full((len(keys), 27), -1, dtype=np.int32)
    for k in range(27):
        q = vox.astype(np.int64) + np.array([k // 9 - 1, k // 3 % 3 - 1, k % 3 - 1])
        ok = ((q >= 0) & (q < 1 << w)).all(1)
        qk = np.where(ok, (frame << 3 * w) | (q[:, 0] << 2 * w) | (q[:, 1] << w) | q[:, 2], 0)
        pos = np.minimum(np.searchsorted(keys, qk), len(keys) - 1)
        hit = ok & (keys[pos] == qk)
        nbr[hit, k] = pos[hit]
    return nbr


def batched_index(frames, shapes):
    """(keys, p2v, nbr, w) of the batched level of the frames' points."""
    f, w = _layout(shapes)
    keys, p2v = np.unique(np.concatenate([_pack(b, c, w) for b, c in enumerate(frames)]), return_inverse=True)
    return keys, p2v.reshape(-1).astype(np.int32), _neighbours(keys, w), w


def batched_down(keys, shapes, w):
    """(parent keys, their nbr, down, up, coarse shapes): each child dropped against its own frame's coarse shape."""
    frame, vox = _unpack(keys, w)
    cs = np.array([spconv.coarse_shape(s) for s in shapes], dtype=np.int64)
    par = vox.astype(np.int64) >> 1
    keep = (par < cs[frame]).all(1)
    pk = _pack(0, par, w) | (frame << 3 * w)
    pkeys = np.unique(pk[keep])
    parent = np.full(len(keys), -1, dtype=np.int64)
    parent[keep] = np.searchsorted(pkeys, pk[keep])
    kc = (vox[:, 0] & 1) * 4 + (vox[:, 1] & 1) * 2 + (vox[:, 2] & 1)
    dn = np.full((len(pkeys), 8), -1, dtype=np.int32)
    up = np.full((len(keys), 8), -1, dtype=np.int32)
    c = np.nonzero(keep)[0]
    dn[parent[c], kc[c]] = c
    up[c, kc[c]] = parent[c]
    return pkeys, _neighbours(pkeys, w), dn, up, [tuple(int(v) for v in s) for s in cs]


def _rebase(t, base):
    return np.where(t >= 0, t + base, -1)


def _coords(shape, n, seed):
    rng = np.random.RandomState(seed)
    return np.stack([rng.randint(0, s, n) for s in shape], 1).astype(np.int32)


def _carry_frames(side):
    """Frames of shape side^3 = 2^w: sites on every top plane, and the next frame's sites at its origin planes."""
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    top = g[(g == side - 1).any(1)]
    origin = g[(g == 0).any(1)]
    return [top, origin, np.concatenate([top, origin])], [(side,) * 3] * 3


def _batches():
    return {
        "mixed": ([_coords((13, 11, 12), 300, 1), _coords((9, 10, 7), 200, 2), _coords((20, 16, 17), 1500, 3),
                   np.array([[2, 3, 4]] * 3, np.int32), _coords((2, 3, 4), 5, 4)],
                  [(13, 11, 12), (9, 10, 7), (20, 16, 17), (5, 5, 5), (2, 3, 4)]),
        "shape_1": ([_coords((1, 6, 7), 30, 5), _coords((8, 9, 10), 200, 6)], [(1, 6, 7), (8, 9, 10)]),
        "identical": ([_coords((6, 6, 6), 80, 7), _coords((6, 6, 6), 80, 7), _coords((7, 5, 6), 50, 8)],
                      [(6, 6, 6), (6, 6, 6), (7, 5, 6)]),
        "carry": _carry_frames(8),
        "one_frame": ([_coords((13, 11, 12), 300, 9)], [(13, 11, 12)]),
    }


@pytest.mark.parametrize("name", list(_batches()))
def test_restated_layout_is_the_frames_tables_concatenated(name):
    """Index and every down step the frames allow: sites, p2v, nbr, down, up, each frame's own plus its row base."""
    frames, shapes = _batches()[name]
    keys, p2v, nbr, w = batched_index(frames, shapes)
    assert spconv.key_layout(shapes) == _layout(shapes)
    assert (np.diff(keys) > 0).all()
    frame, vox = _unpack(keys, w)
    assert (np.diff(frame) >= 0).all()                               # frame by frame, in key order within each
    single = [R.index(c) for c in frames]
    base = np.cumsum([0] + [len(s[0]) for s in single])
    pbase = np.cumsum([0] + [len(c) for c in frames])
    for b, (v, pv, nb) in enumerate(single):
        rows = slice(base[b], base[b + 1])
        assert (frame[rows] == b).all() and np.array_equal(vox[rows], v)
        assert np.array_equal(nbr[rows], _rebase(nb, base[b]))
        assert np.array_equal(p2v[pbase[b]:pbase[b + 1]], pv + base[b])
    fine = [s[0] for s in single]
    fshapes = [tuple(s) for s in shapes]
    while min(min(s) for s in fshapes) >= 1:
        M = len(keys)
        pkeys, pnbr, dn, up, cshapes = batched_down(keys, fshapes, w)
        assert len(pkeys) <= spconv.down_rows(M, fshapes)
        ref = [R.down(v, s) for v, s in zip(fine, fshapes)]
        cbase = np.cumsum([0] + [len(r[0]) for r in ref])
        _, cvox = _unpack(pkeys, w)
        for b, (cv, cn, d, u, cs) in enumerate(ref):
            rows = slice(cbase[b], cbase[b + 1])
            assert cs == cshapes[b] and np.array_equal(cvox[rows], cv)
            assert np.array_equal(pnbr[rows], _rebase(cn, cbase[b]))
            assert np.array_equal(dn[rows], _rebase(d, base[b]))
            assert np.array_equal(up[base[b]:base[b + 1]], _rebase(u, cbase[b]))
        keys, fine, fshapes, base = pkeys, [r[0] for r in ref], cshapes, cbase


def test_field_bound_stops_the_carry():
    """x = 2^w - 1 plus one would be the next frame's x = 0, and z = 2^w - 1 plus one the next y's z = 0, without the
    bound by the field."""
    frames, shapes = _carry_frames(8)
    keys, _, nbr, w = batched_index(frames, shapes)
    frame, vox = _unpack(keys, w)
    k_x, k_z = 9 * 2 + 3 + 1, 9 + 3 + 2                           # offsets (+1, 0, 0) and (0, 0, +1)
    for k, axis in ((k_x, 0), (k_z, 2)):
        edge = vox[:, axis] == 7
        assert edge.any() and (nbr[edge, k] == -1).all()
        unbounded = keys[edge] + (np.int64(1) << (2 - axis) * w)   # what the key arithmetic alone would look up
        assert np.isin(unbounded, keys).any()


@pytest.mark.parametrize("shapes, want", [
    ([(1 << 21,) * 3], (0, 21)), ([(5, 6, 7)], (0, 21)), ([(1, 1, 1)], (0, 21)),
    ([(16, 16, 16), (3, 4, 5)], (1, 4)), ([(17, 16, 16), (3, 4, 5)], (1, 5)), ([(2, 1, 1)] * 3, (2, 1)),
    ([(1, 1, 1)] * 2, (1, 0)), ([(4, 4, 4)] * 4, (2, 2)), ([(4, 4, 4)] * 5, (3, 2)),
    ([(1 << 20,) * 3] * 8, (3, 20)), ([(1 << 20,) * 3] * 9, None), ([(1 << 21,) * 3] * 2, None),
])
def test_width_rule_and_limit(shapes, want):
    assert _layout(shapes) == want
    if want is None:
        with pytest.raises(ValueError, match="f \\+ 3 w <= 63"):
            spconv.key_layout(shapes)
    else:
        assert spconv.key_layout(shapes) == want


@pytest.mark.parametrize("shapes", [[(0, 4, 4)], [(4, 4)], [(4, 4, 1 << 21 | 1)], []])
def test_bad_shapes_are_refused(shapes):
    with pytest.raises(ValueError):
        spconv.key_layout(shapes)


@pytest.mark.parametrize("M, shapes, want", [
    (1000, [(128, 128, 128)], 1000), (10 ** 7, [(128, 128, 128)], 64 ** 3),
    (10 ** 7, [(128, 128, 128), (9, 9, 9)], 64 ** 3 + 4 ** 3), (50, [(9, 9, 9), (8, 8, 8)], 50),
    (100, [(1, 5, 5), (1, 9, 9)], 1), (100, [(1, 5, 5), (3, 3, 2)], 1), (100, [(1, 5, 5), (4, 3, 2)], 2),
    (3, [(2, 2, 2)] * 5, 3), (7, [(2, 2, 2)] * 5, 5),
])
def test_row_bound(M, shapes, want):
    assert spconv.down_rows(M, shapes) == want


def test_row_bound_holds_every_parent():
    rng = np.random.RandomState(10)
    for trial in range(20):
        B = rng.randint(1, 6)
        shapes = [tuple(int(v) for v in rng.randint(1, 12, 3)) for _ in range(B)]
        frames = [_coords(s, rng.randint(1, 200), 100 * trial + b) for b, s in enumerate(shapes)]
        keys, _, _, w = batched_index(frames, shapes)
        pkeys = batched_down(keys, shapes, w)[0]
        assert len(pkeys) <= spconv.down_rows(len(keys), shapes)
