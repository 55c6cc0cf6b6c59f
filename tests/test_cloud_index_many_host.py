"""The key layout of a many-set cloud index (cg_cloud.cu, cg_cloud_index_create_many), restated in numpy (CPU only).

A key is s << 3b | x << 2b | y << b | z with each set's own origin (its min_bound - cell/2); b is the smallest width
that holds every set's largest cell, the set field takes bit_length(S - 1) bits, and a batch needing more than 63
bits is refused.  These tests hold that restatement to the properties the device tables rely on: sorting the keys
gives each set's points as one block in the order of the set's own one-set index (whatever its own width), every
cell of a set carries the set's prefix, a coordinate at 2^b - 1 never reaches the next set, and one set is exactly
today's layout.
"""
import numpy as np
import pytest

from oracle import cloud_ref

MAX_AXIS_BITS = 21


def _set_cells(p, cell):
    """(cells (n,3) int64, largest cell per axis) of one set, in the host's float64 arithmetic."""
    o = p.min(0) - cell * 0.5
    top = np.floor((p.max(0) - o) / cell).astype(np.int64)
    cells = np.floor((p - o) / cell).astype(np.int64)
    return cells, top


def _width(maxc):
    bits = 1
    while (1 << bits) <= maxc:
        bits += 1
    return bits


def layout(sets, cell):
    """(keys (N,) uint64, b, set bits), or ValueError where the library returns CG_EINVAL."""
    if any(len(p) == 0 for p in sets):
        raise ValueError("every set needs at least one point")
    cells, tops = zip(*[_set_cells(p, cell) for p in sets])
    if any((t >= 1 << MAX_AXIS_BITS).any() for t in tops):
        raise ValueError("2^21 cells on an axis")
    b = _width(max(int(t.max()) for t in tops))
    sb = (len(sets) - 1).bit_length()
    if sb + 3 * b > 63:
        raise ValueError("63 bits")
    keys = [(np.uint64(s) << np.uint64(3 * b)) | (c[:, 0].astype(np.uint64) << np.uint64(2 * b)) |
            (c[:, 1].astype(np.uint64) << np.uint64(b)) | c[:, 2].astype(np.uint64) for s, c in enumerate(cells)]
    return np.concatenate(keys), b, sb


def one_set_keys(p, cell):
    c, top = _set_cells(p, cell)
    b = _width(int(top.max()))
    return (c[:, 0] << (2 * b)) | (c[:, 1] << b) | c[:, 2], b


def _blob(n, seed, centre=(0.1, -0.05, 0.6), spread=0.04):
    return np.random.RandomState(seed).normal(centre, spread, (n, 3))


BATCHES = {
    "sizes": ([_blob(5000, 1), _blob(3, 2), _blob(400, 3, spread=0.002)], 0.001),
    "one_point": ([np.array([[0.3, 0.2, 0.5]]), _blob(300, 4)], 0.0005),
    "identical": ([_blob(500, 5)] * 3, 0.003),
    "overlap": ([_blob(800, 6), _blob(800, 7), _blob(600, 8, centre=(0.12, -0.04, 0.61))], 0.0005),
    "far_apart": ([_blob(300, 9), _blob(300, 10, centre=(50.0, -20.0, 3.0))], 0.002),
}


@pytest.mark.parametrize("name", sorted(BATCHES))
def test_sorted_keys_give_each_set_its_one_set_order(name):
    sets, cell = BATCHES[name]
    keys, b, sb = layout(sets, cell)
    off = np.cumsum([0] + [len(p) for p in sets])
    order = np.lexsort((np.arange(len(keys)), keys))            # (key, index), as the radix sort of (key, index)
    assert sb + 3 * b <= 63
    for s, p in enumerate(sets):
        block = order[off[s]:off[s + 1]]
        assert ((block >= off[s]) & (block < off[s + 1])).all(), s          # set-major: one block per set
        k1, b1 = one_set_keys(p, cell)
        assert b1 <= b
        assert np.array_equal(block - off[s], np.lexsort((np.arange(len(p)), k1))), s
        assert (keys[block] >> np.uint64(3 * b) == np.uint64(s)).all(), s
        # the unique cells of the set are open3d's voxels of the set alone
        uk = np.unique(keys[block] & np.uint64((1 << 3 * b) - 1))
        m = np.uint64((1 << b) - 1)
        cells = np.stack([(uk >> np.uint64(2 * b)) & m, (uk >> np.uint64(b)) & m, uk & m], 1).astype(np.int64)
        assert np.array_equal(cells, np.unique(cloud_ref.voxel_cells(p, cell), axis=0)), s


@pytest.mark.parametrize("S, top, b, sb", [(1, 1, 1, 0), (1, (1 << 21) - 1, 21, 0), (2, 1, 1, 1), (3, 7, 3, 2),
                                           (8, (1 << 20) - 1, 20, 3), (5, 1000, 10, 3), (1 << 10, 1, 1, 10)])
def test_width_rule(S, top, b, sb):
    sets = [np.array([[0.0, 0.0, 0.0], [float(top) * (s == 0), 0.0, 0.0]]) for s in range(S)]
    keys, bb, ssb = layout(sets, 1.0)
    assert (bb, ssb) == (b, sb)
    assert int(keys.max()) < 1 << (sb + 3 * b)


def test_the_largest_batch_that_fits_and_one_more():
    big = [np.array([[0.0, 0.0, 0.0], [600000.0, 0.0, 0.0]])]
    layout(big * 8, 1.0)                                    # b = 20, 3 set bits: 63
    with pytest.raises(ValueError, match="63"):
        layout(big * 9, 1.0)                                # a fourth set bit: 64
    small = [np.array([[0.0, 0.0, 0.0], [3.0, 0.0, 0.0]])]  # b = 2
    layout(small * 3, 1.0)
    with pytest.raises(ValueError, match="2\\^21"):
        layout([np.array([[0.0, 0.0, 0.0], [float(1 << 21), 0.0, 0.0]])], 1.0)
    with pytest.raises(ValueError, match="at least one point"):
        layout([small[0], np.zeros((0, 3))], 1.0)


def test_top_cell_never_reaches_the_next_set():
    """A set whose cells reach 2^b - 1 on every axis: its largest key, plus one cell on any axis clamped to the
    set's range, stays below the next set's prefix."""
    b = 5
    top = float((1 << b) - 1)
    s0 = np.array([[0.0, 0.0, 0.0], [top, top, top]])
    keys, bb, _ = layout([s0, s0, s0], 1.0)
    assert bb == b
    per_set = 1 << (3 * b)
    for s in range(3):
        k = keys[2 * s:2 * s + 2].astype(np.int64)
        assert (k >= s * per_set).all() and (k < (s + 1) * per_set).all()
    assert int(keys[1]) == per_set - 1                       # (2^b - 1, 2^b - 1, 2^b - 1) of set 0
    assert int(keys[2]) == per_set                           # set 1's origin: the next key


def test_one_set_is_todays_layout():
    for name, (sets, cell) in BATCHES.items():
        for p in sets:
            keys, b, sb = layout([p], cell)
            k1, b1 = one_set_keys(p, cell)
            assert sb == 0 and b == b1 and np.array_equal(keys.astype(np.int64), k1), name
