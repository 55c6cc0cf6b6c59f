"""cg_meanshift.cu (catgrasp_b200.segment) on the paths test_meanshift_kernel.py's fixtures do not reach, against the
brute-force references of oracle/meanshift_ref.py (step_bruteforce: one ascent step over all pairs;
modes_bruteforce: the post-processing over all pairs) and, for 2^21 points, a closed form in Python integers.

  - the ascent step by step: each run at max_iter k + 1 is one brute-force step past the kernel's own run at k, bit for
    bit, and within the fixed point's bound of the set's exact mean (also with a far outlier, so E is large);
  - the modes from the kernel's own seed results: unshifted piles with thousands of mutually suppressing modes, a
    lattice of modes exactly bw apart across cell faces and one just over bw, count ties decided by y and by z;
  - equal centres reached through sets of different sizes (the count of the highest seed is kept);
  - a centre rounded one quantum past the points' bounding box into the cell after the last one;
  - exactly 2^21 points, whose per-ball fixed-point sums pass 2^53;
  - point counts around the launch widths.

Seeded mutations of cg_meanshift.cu and the test here that fails on each:
  - __ll2double_rn -> __ll2double_rz in the ascent     test_two_to_the_twenty_one_points (a dropped remainder > half)
  - the count sort's end_bit 23 -> 21                  test_two_to_the_twenty_one_points (the sentinel P + 1 = 2^21 + 1)
  - rank_kernel without its cell clamp                 test_centre_past_the_bounding_box
  - suppression `<= bw2` -> `< bw2`                    test_mode_lattice_at_bw_across_cell_faces
  - suppression scanning only C.z0 of each column      test_modes_of_unshifted_piles
  - group_kernel writing the head's count              test_equal_centres_with_different_counts
  - the seed passes in x, y, z order, not z, y, x      test_count_ties_decided_by_y_then_z
"""
import math
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import segment, synthetic   # noqa: E402
from catgrasp_b200.cloud import CloudIndex     # noqa: E402
from oracle import meanshift_ref               # noqa: E402


def _fit(X, bw, max_iter=300):
    got = segment.MeanShift(bandwidth=bw, max_iter=max_iter).fit(X)
    assert got.seed_centers_.dtype == X.dtype and got.cluster_centers_.dtype == X.dtype
    return got


def _check_modes(got, bw):
    """The kernel's kept centres == modes_bruteforce of its own seed results, bit for bit."""
    ref = meanshift_ref.modes_bruteforce(got.seed_centers_, got.seed_counts_, bw)
    assert got.cluster_centers_.tobytes() == ref.tobytes()


def _check_oracle(X, bw, max_iter=300):
    got = _fit(X, bw, max_iter)
    ref = meanshift_ref.fit(X, bw, max_iter=max_iter)
    assert got.seed_centers_.tobytes() == ref["seed_centres"].tobytes()
    assert np.array_equal(got.seed_counts_, ref["seed_counts"])
    assert np.array_equal(got.seed_iters_, ref["seed_iters"])
    assert got.cluster_centers_.tobytes() == ref["centres"].tobytes()
    assert np.array_equal(got.labels_, ref["labels"]) and got.n_iter_ == ref["n_iter"]
    _check_modes(got, bw)
    return got


def _pile(n, k, seed, pull, noise=0.0008):
    s = synthetic.make_pile(n, n_objects=k, seed=seed)
    centre = s["object_poses"][:, :3, 3][s["object_id"]]
    rng = np.random.RandomState(seed + 7)
    return s["cloud_xyz"] + pull * (centre - s["cloud_xyz"]) + rng.normal(0, noise, s["cloud_xyz"].shape)


def _index_origin(X, bw):
    ix = CloudIndex(torch.from_numpy(np.asarray(X, np.float64)).cuda(), bw)
    o = np.zeros(3)
    ix.ctx.call("cg_cloud_index_info", ix.h, None, None, None, o)
    return o


# ---------------------------------------------------------------------------------------------------- step by step

def _lattice():
    bw = 2.0 ** -7
    g = np.stack(np.meshgrid(np.arange(9), np.arange(7), np.arange(5), indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.RandomState(4)
    return 0.5 + (g * 0.75 + rng.randint(0, 4, g.shape) * 0.125) * bw, bw   # dyadic, spacing 0.75 bw +- jitter


def _with_outlier():
    X = _pile(3000, 10, seed=9, pull=0.3)
    return np.concatenate([X, X[:1] + [5.0, -0.5, 0.25]]), 0.007


STEP_CLOUDS = {
    "pile": lambda: (_pile(3000, 10, seed=5, pull=0.3), 0.007),
    "pile-bw005": lambda: (_pile(3000, 10, seed=6, pull=0.0), 0.005),
    "lattice": _lattice,
    "outlier": _with_outlier,
}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("cloud", sorted(STEP_CLOUDS))
def test_ascent_step_by_step(cloud, dtype):
    """Run k + 1 is one brute-force step past the kernel's own run k for every seed still moving after run k; every
    other seed keeps run k's result.  Each step is within the fixed point's bound of its set's mean."""
    X, bw = STEP_CLOUDS[cloud]()
    X = X.astype(dtype)
    origin, E = meanshift_ref.frame(X, bw)
    assert _index_origin(X, bw).tobytes() == origin.tobytes()
    prev_c, prev_n, prev_it = X, np.zeros(len(X), np.int64), np.zeros(len(X), np.int64)
    moving = np.ones(len(X), bool)
    worst, steps = 0.0, 0
    for k in range(8):
        got = _fit(X, bw, max_iter=k)
        c, n, it = got.seed_centers_, got.seed_counts_, got.seed_iters_
        assert c[~moving].tobytes() == prev_c[~moving].tobytes()
        assert np.array_equal(n[~moving], prev_n[~moving]) and np.array_equal(it[~moving], prev_it[~moving])
        new, cnt, mean = meanshift_ref.step_bruteforce(X, bw, prev_c[moving])
        assert new.tobytes() == c[moving].tobytes()
        assert np.array_equal(cnt, n[moving]) and (it[moving] == k).all()
        ratio = meanshift_ref.bound_ratio(new, mean, E)
        worst = max(worst, float(ratio.max()))
        steps += int(moving.sum())
        d = (new - prev_c[moving]).astype(np.float64)
        step = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        moving[np.flatnonzero(moving)[(cnt == 0) | (step <= 1e-3 * bw)]] = False
        prev_c, prev_n, prev_it = c, n, it
        if not moving.any():
            break
    print(f"{cloud} {np.dtype(dtype).name}: E = {E}, {steps} steps checked, worst |centre - mean| / bound = {worst:.3f}")
    assert worst <= 1.0


# ----------------------------------------------------------------------------------------------------------- modes

@pytest.mark.parametrize("max_iter", [0, 1, 300])
@pytest.mark.parametrize("bw, n", [(0.005, 50000), (0.007, 30000), (0.009, 20000)])
def test_modes_of_unshifted_piles(bw, n, max_iter):
    X = _pile(n, 12, seed=11, pull=0.0).astype(np.float32)
    got = _fit(X, bw, max_iter)
    n_modes = len({tuple(r) for r, k in zip(got.seed_centers_.astype(np.float64).tolist(), got.seed_counts_) if k})
    print(f"bw {bw} max_iter {max_iter}: {n} points, {n_modes} modes, {len(got.cluster_centers_)} kept")
    assert n_modes > 2 * len(got.cluster_centers_)
    _check_modes(got, bw)


@pytest.mark.parametrize("max_iter", [0, 300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mode_lattice_at_bw_across_cell_faces(dtype, max_iter):
    """Interior sites of a lattice spaced exactly bw keep their place (count 7) and lie exactly bw apart in
    neighbouring cells, so each kept one suppresses its neighbours; sites of a second lattice spaced bw (1 + 2^-16)
    are isolated modes that suppress nothing."""
    bw = 2.0 ** -7
    g = np.stack(np.meshgrid(np.arange(8), np.arange(6), np.arange(5), indexing="ij"), -1).reshape(-1, 3)
    near = 0.5 + g * bw
    far = 0.5 + g * (bw + bw * 2.0 ** -16) + [12 * bw, 0.0, 0.0]
    X = np.concatenate([near, far]).astype(dtype)
    assert np.array_equal(X.astype(np.float64), np.concatenate([near, far]))
    got = _check_oracle(X, bw, max_iter)
    kept = got.cluster_centers_.astype(np.float64)
    assert (kept[:, 0] >= far[:, 0].min()).sum() == len(far)              # no far site suppressed
    inner = got.seed_counts_[:len(near)] == 7                              # the sites' own centres, bw apart
    assert inner.sum() == 72 and got.seed_centers_[:len(near)][inner].tobytes() == X[:len(near)][inner].tobytes()
    k = kept[kept[:, 0] < far[:, 0].min()]
    d = k[:, None, :] - k[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert (d2[~np.eye(len(k), dtype=bool)] > bw * bw).all()             # kept modes are more than bw apart


def _chain(start, step, n):
    return np.asarray(start, np.float64) + np.arange(n)[:, None] * np.asarray(step, np.float64)


def test_count_ties_decided_by_y_then_z():
    """Chains of single points, dyadic and negative, whose interior points are their own means with count 3: along y
    (x tied), along z (x and y tied), and along (0, a, -a) and (a, 0, -a), where the primary key and z disagree.
    Each chain has an even number of interior points, so which end the greedy pass starts from decides the kept set."""
    bw = 2.0 ** -7
    s = 7 * 2.0 ** -10          # 0.875 bw: neighbours within bw, second neighbours not
    a = 5 * 2.0 ** -10          # (a, 0, -a) is 0.884 bw long
    X = np.concatenate([
        _chain([-0.25, -0.375, -0.125], [0, s, 0], 10),
        _chain([-0.25, -0.25, -0.125], [0, 0, s], 10),
        _chain([-0.3125, -0.375, -0.0625], [0, a, -a], 10),
        _chain([-0.375, -0.375, -0.0625], [a, 0, -a], 10),
    ])
    for dtype in (np.float32, np.float64):
        for max_iter in (0, 300):
            got = _check_oracle(X.astype(dtype), bw, max_iter)
            assert (got.seed_counts_ == 3).sum() >= 32


def test_equal_centres_with_different_counts():
    """With max_iter 0: O's set is O, the two points 1 unit off in y and the two points 2 units off in x (count 5);
    each y neighbour's set is O and both y points (count 3); both sets have mean O.  O is the lowest of the three
    seeds, so the dict rule gives the group count 3, below the 4 of a separate cluster, which then ranks first."""
    u = 2.0 ** -8
    pts = [(0, 0), (0, 1), (0, -1), (2, 0), (-2, 0)] + [(10, 10)] * 4
    X64 = np.array([(0.25 + x * u, -0.125 + y * u, 0.5) for x, y in pts])
    bw = 2 * u
    for dtype in (np.float32, np.float64):
        X = X64.astype(dtype)
        got = _check_oracle(X, bw, max_iter=0)
        c, n = got.seed_centers_, got.seed_counts_
        assert c[:3].tobytes() == np.repeat(X[:1], 3, 0).tobytes() and n[:3].tolist() == [5, 3, 3]
        head = n.copy()
        head[1:3] = n[0]
        assert meanshift_ref.modes_bruteforce(c, head, bw).tobytes() != got.cluster_centers_.tobytes()
        assert got.cluster_centers_.tobytes() == X[[5, 0]].tobytes()


def _past_the_box():
    """float64 points sharing x = hx, the max bound, with D alone at the min bound, so hi - origin = hx - x_D + bw/2
    lies just below 2 cells; hx's low bits make q(hx) round up, so a mean over those points lands past hx in cell 2,
    one after the last.  Groups A, B, C at y0, y0 - 0.6 bw, y0 - 1.2 bw (4, 3, 2 copies) give three modes within bw
    of each other (max_iter 0): B's set holds all three groups and suppresses the other two."""
    xd, y0, z0 = 0.25, -0.1, 0.4
    for j in range(64):                                # the first bw whose 2 cells end within half a quantum
        bw = 0.005 + j * 2.0 ** -50                    # of a fixed-point step above: a quarter quantum apart
        ox = xd - bw * 0.5
        hx = ox + 2 * bw                               # the first double whose cell is 2, then below it
        while math.floor((hx - ox) / bw) < 2:
            hx = np.nextafter(hx, 1.0)
        while math.floor((np.nextafter(hx, 0.0) - ox) / bw) == 2:
            hx = np.nextafter(hx, 0.0)
        for _ in range(256):
            hx = np.nextafter(hx, 0.0)
            X = np.array([[hx, y0, z0]] * 4 + [[hx, y0 - 0.6 * bw, z0]] * 3 + [[hx, y0 - 1.2 * bw, z0]] * 2
                         + [[xd, y0 - 0.6 * bw, z0]])
            c, _, _ = meanshift_ref.step_bruteforce(X, bw, X[:1])
            if c[0, 0] > hx and math.floor((c[0, 0] - ox) / bw) == 2:
                assert meanshift_ref.frame(X, bw)[0][0] == ox and math.floor((hx - ox) / bw) == 1
                return X, bw
        assert meanshift_ref.frame(X, bw)[1] == -6
    raise AssertionError("no max bound rounds into the next cell")



def test_centre_past_the_bounding_box():
    X, bw = _past_the_box()
    origin = _index_origin(X, bw)
    assert origin.tobytes() == meanshift_ref.frame(X, bw)[0].tobytes()
    got = _check_oracle(X, bw, max_iter=0)
    cx = got.seed_centers_[:9, 0]
    assert (cx > X[:, 0].max()).all() and (np.floor((cx - origin[0]) / bw) == 2).all()
    assert np.floor((X[:, 0].max() - origin[0]) / bw) == 1
    assert len(got.cluster_centers_) == 2 and got.cluster_centers_[0, 0] > X[:, 0].max()


# --------------------------------------------------------------------------------------------------- 2^21 points

def _eight_balls():
    """8 cubes of 2^18 float64 points, side bw/2 (diameter < bw), 4 bw apart: every seed's set is its whole cube on
    every step.  Returns X, bw, the cube of each point and the closed-form (centre per cube, sums, E, origin)."""
    bw = 0.005
    per = 1 << 18
    rng = np.random.RandomState(21)
    corners = np.stack(np.meshgrid([0, 1], [0, 1], [0, 1], indexing="ij"), -1).reshape(-1, 3) * 4 * bw
    base = np.array([0.125, -0.0625, 0.5])
    ball = np.repeat(np.arange(8), per)
    X = base + corners[ball] + rng.uniform(0, 0.5 * bw, (8 * per, 3))
    perm = rng.permutation(len(X))
    X, ball = X[perm], ball[perm]
    origin, E = meanshift_ref.frame(X, bw)
    q = np.rint((X - origin) * math.ldexp(1.0, meanshift_ref.QBITS - E)).astype(np.int64)
    sums = [[int(s) for s in q[ball == b].sum(axis=0)] for b in range(8)]
    unscale = math.ldexp(1.0, E - meanshift_ref.QBITS)

    def centre(to_double):
        return np.array([[to_double(s) * unscale / per + float(origin[a]) for a, s in enumerate(row)] for row in sums])

    def rz(s):                       # int -> double, rounded toward zero
        drop = max(0, s.bit_length() - 53)
        return float((s >> drop) << drop)

    return X, bw, ball, centre(float), centre(rz), sums


def test_two_to_the_twenty_one_points():
    X, bw, ball, centres, centres_rz, sums = _eight_balls()
    P, per = len(X), 1 << 18
    assert P == 1 << 21
    assert min(s for row in sums for s in row) > 2 ** 53
    above_half = [s for row in sums for s in row if (s & ((1 << (s.bit_length() - 53)) - 1)) > 1 << (s.bit_length() - 54)]
    assert above_half and not np.array_equal(centres, centres_rz)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = segment.MeanShift(bandwidth=bw).fit(X)
    torch.cuda.synchronize()
    print(f"2^21 points, 8 balls of 2^18: MeanShift.fit {time.perf_counter() - t0:.2f} s (wall clock, incl. labels)")
    d = centres[ball] - X
    step = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    assert got.seed_centers_.tobytes() == centres[ball].tobytes()
    assert (got.seed_counts_ == per).all()
    assert np.array_equal(got.seed_iters_, np.where(step <= 1e-3 * bw, 0, 1))
    order = sorted(range(8), key=lambda b: tuple(centres[b]), reverse=True)
    assert got.cluster_centers_.tobytes() == centres[order].tobytes()
    assert np.array_equal(got.labels_, np.argsort(order)[ball]) and got.n_iter_ == 1


# ------------------------------------------------------------------------------------------------- launch edges

@pytest.mark.parametrize("P", [2, 7, 8, 9, 31, 32, 33, 255, 256, 257])
def test_point_counts_around_launch_widths(P):
    rng = np.random.RandomState(P)
    bw = 0.007
    X = 0.3 + rng.uniform(0, 4 * bw, (P, 3))
    for dtype in (np.float32, np.float64):
        _check_oracle(X.astype(dtype), bw)
        _check_oracle(X.astype(dtype), bw, max_iter=0)
