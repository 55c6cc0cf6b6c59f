"""The scan occupancy grid (csrc/cg_occupancy.cu via my_cpp.makeOccupancyGridFromCloudScan) at exact geometry.

Every case runs the kernel and oracle/occupancy_ref.c and requires the same samples, bit for bit (GPU).  Both are
also held to oracle/occupancy_exact.py, an exact rational statement of the rule that shares neither their float64
arithmetic nor their early exit, on every sample it can decide (CPU for the C oracle, GPU for the kernel).  The cases:

- single-point scans, one of them on the camera axis so that samples lie at x = 0 and y = 0 exactly (step 0);
- a scan with a point at the camera and points in the camera's own cell: a sample at the origin, and an occupied
  origin cell;
- scans straddling x = 0 and y = 0, so cells have negative indices and rays step in -x and -y; one of them of
  isolated cells, whose samples just in front of a cell's far corner are reported only because the walk goes on
  past the sample (the ``+ 2r`` of the early exit);
- dyadic resolutions (2^-9, 2^-10) with scan points on cell corners and the grid origin on a corner (samples on
  corners) or on a cell centre (samples on centres): rays through cell edges and corners, crossing parameters that
  tie exactly; the exact reference counts the tied and the undecided samples;
- hex-nut piles at two new seeds and three resolutions;
- refusals: a grid of 2^31 or more samples and a resolution <= 0 (or one that rounds to 0 in float32) raise CgError.

Seeded mutations of cg_occupancy.cu / occupancy_ref.c and the test aimed at each.  Each was built once, when these
tests were written, and failed the test named for it: the first in the kernel on an H100, the next three in
occupancy_ref.c, which shares the kernel's control flow (the mutants are not built by this file):
- tmax ties broken towards the other axis (``<=`` for ``<`` in the axis choice): test_kernel_bit_exact[dyadic_*];
- the early exit without its ``+ 2r`` (``tmax > dist_q``), in both kernel and oracle:
  test_exact_reference_agrees_with_occupancy_ref[sparse];
- the step of a negative axis started at k + 1 (``step > 0 ? 1 : 0`` read as 1 for both signs), in both:
  test_exact_reference_agrees_with_occupancy_ref[straddle];
- the origin cell not tested first: test_exact_reference_agrees_with_occupancy_ref[at_camera];
- contraction re-enabled in the cast kernel: tests/test_codegen.py (this file cannot see a 1-ulp change).

No case can tell the final ``cdist <= dist_q`` (common.cpp:388-393) from ``<``: they differ only when the float64
centre distance equals the sample's float32 norm, and a cell centre's distance is never a float32.  Its square is
(res/2)^2 (a^2 + b^2 + c^2) with a, b, c odd, and a sum of three odd squares is 3 mod 8, never a perfect square; with
a dyadic res the float64 square is exact, so its rounded root has more than 24 significant bits.  For any other res a
tie needs a rounded square root that happens to fit in 24 bits.  Samples on cell centres therefore test the walk's
ties, not this comparison.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import filter_ref, occupancy_exact as ox

PAD = np.float32(0.005)


def _on_lattice(O):
    """A float32 a with float32(a - 0.005) == O exactly: the scan minimum that puts the grid origin at O."""
    a = np.float32(O + PAD)
    for _ in range(64):
        d = np.float32(a - PAD)
        if d == O:
            return a
        a = np.nextafter(a, np.float32(np.inf) if d < O else np.float32(-np.inf))
    raise AssertionError(f"no float32 scan minimum gives origin {O}")


def _lattice_case(e, seed, lat, zr, off):
    """Scan points on the corners of cells of size 2^-e, plus one point that places the grid origin on the lattice
    (off = 0: samples on corners) or half a cell off it (off = 0.5: samples on cell centres)."""
    rng = np.random.RandomState(seed)
    r = np.float32(2.0 ** -e)
    ijk = np.stack([rng.randint(-lat, lat + 1, 80), rng.randint(-lat, lat + 1, 80), rng.randint(zr[0], zr[1], 80)], 1)
    O = ((ijk.min(0) - 3 + off) * r).astype(np.float32)
    anchor = np.array([_on_lattice(o) for o in O], np.float32)
    return np.concatenate([anchor[None], (ijk * r).astype(np.float32)]), r


def _cases():
    r25 = np.float32(0.0025)
    zero = np.float32(np.float32(0.005) - np.float32(2) * r25)     # == 0; with res 0.0025 a sample lands on it
    rng, rng105 = np.random.RandomState(21), np.random.RandomState(105)
    return {
        "single_point": (np.array([[0.0123, -0.0071, 0.05]], np.float32), np.float32(0.002)),
        "axis_zero": (np.array([[zero, zero, 0.0395]], np.float32), r25),
        "at_camera": (np.array([[zero, zero, zero], [0.001, 0.0005, 0.0015], [0.003, 0.002, 0.012],
                                [0.0045, 0.004, 0.02]], np.float32), r25),
        "straddle": (np.c_[rng.uniform(-0.008, 0.008, (40, 2)), rng.uniform(0.03, 0.04, 40)].astype(np.float32),
                     np.float32(0.002)),
        # 30 isolated cells: rays that clip a cell's far corner enter it beyond the sample while its centre is nearer
        "sparse": (np.c_[rng105.uniform(-0.015, 0.015, (30, 2)), rng105.uniform(0.02, 0.035, 30)].astype(np.float32),
                   np.float32(0.002)),
        "dyadic_corner": _lattice_case(9, 22, 4, (12, 21), 0.0),
        "dyadic_centre": _lattice_case(10, 23, 3, (24, 41), 0.5),
    }


PILES = [(s, r) for s in (31, 32) for r in (0.0005, 0.001, 0.002)]


def _pile(seed):
    from catgrasp_b200.synthetic import make_pile
    return make_pile(1500, n_objects=2, seed=seed, bin_size=0.04)["cloud_xyz"]


def _pile_subset(flags, seed, n=60):
    """n reported and n unreported samples: the exact reference is too slow for whole piles."""
    rs = np.random.RandomState(seed)
    on, off = np.nonzero(flags)[0], np.nonzero(flags == 0)[0]
    return np.concatenate([rs.choice(on, min(n, len(on)), replace=False), rs.choice(off, min(n, len(off)), replace=False)])


def _samples(dims, org, r):
    idx3 = np.argwhere(np.ones(tuple(int(d) for d in dims), bool))
    return ox.samples_of(org, np.float32(r), idx3)[0]


@pytest.mark.parametrize("case", list(_cases()))
def test_exact_reference_agrees_with_occupancy_ref(case):
    """CPU: occupancy_ref.c equals the exact rule on every decided sample; the case's geometry is what it claims."""
    pts, r = _cases()[case]
    flags, org, dims = filter_ref.occupancy_ref(pts, r)
    d2, o2, _ = ox.geometry(pts, r)
    assert (d2 == dims).all() and (o2.view(np.uint32) == org.view(np.uint32)).all()
    f, decided, tied = ox.occupancy_exact(pts, r)
    fr = flags.reshape(-1)
    bad = np.nonzero((f != fr) & decided)[0]
    print(f"{case}: {fr.size} samples, {int(fr.sum())} reported, {int(tied.sum())} with an exact tie, "
          f"{int((~decided).sum())} undecided")
    assert len(bad) == 0, (bad[:10], f[bad[:10]], fr[bad[:10]])
    assert 0 < fr.sum() < fr.size
    s = _samples(dims, org, r)
    cells = np.floor(pts.astype(np.float64) / np.float64(r))
    if case == "axis_zero":
        assert (s[:, 0] == 0).any() and (s[:, 1] == 0).any() and ((s[:, 0] == 0) & (s[:, 1] == 0)).any()
    if case == "at_camera":
        assert (np.abs(s).sum(1) == 0).sum() == 1 and ((cells == 0).all(1)).any()
    if case in ("straddle", "sparse"):
        assert (cells[:, 0] < 0).any() and (cells[:, 1] < 0).any() and (cells[:, :2] >= 0).any()
    if case.startswith("dyadic"):
        assert tied.sum() > 100 and (~decided).any()
        assert decided.mean() > 0.8


@pytest.mark.parametrize("seed,res", PILES)
def test_exact_reference_agrees_with_occupancy_ref_on_piles(seed, res):
    """CPU: occupancy_ref.c equals the exact rule on a sample of a pile's reported and unreported samples."""
    pts = _pile(seed)
    flags, _, _ = filter_ref.occupancy_ref(pts, res)
    fr = flags.reshape(-1)
    sub = _pile_subset(fr, seed)
    f, decided, _ = ox.occupancy_exact(pts, res, sub)
    print(f"pile {seed} @ {res}: {fr.size} samples, {len(sub)} checked, {int((~decided).sum())} undecided")
    assert decided.mean() > 0.9
    assert (f[decided] == fr[sub][decided]).all()


def _kernel_vs_oracle(pts, r):
    from catgrasp_b200 import my_cpp
    out = my_cpp.makeOccupancyGridFromCloudScan(pts, np.eye(3), r)
    flags, org, dims = filter_ref.occupancy_ref(pts, r)
    ref = _samples(dims, org, r)[flags.reshape(-1) > 0]
    assert out.dtype == np.float32 and out.shape == ref.shape
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    return out, flags.reshape(-1), org, dims


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(_cases()))
def test_kernel_bit_exact(case):
    """GPU: the kernel reports exactly occupancy_ref.c's samples, and the exact rule's on every decided sample."""
    pts, r = _cases()[case]
    out, _, org, dims = _kernel_vs_oracle(pts, r)
    f, decided, _ = ox.occupancy_exact(pts, r)
    got = np.zeros(len(f), np.uint8)
    s = _samples(dims, org, r)
    reported = {tuple(row) for row in out.view(np.uint32)}
    got[[tuple(row) in reported for row in s.view(np.uint32)]] = 1
    assert got.sum() == len(out)
    assert (got[decided] == f[decided]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("seed,res", PILES)
def test_kernel_bit_exact_on_piles(seed, res):
    """GPU: the kernel equals occupancy_ref.c on whole piles, and the exact rule on a sample of each."""
    pts = _pile(seed)
    out, fr, org, dims = _kernel_vs_oracle(pts, res)
    assert len(out) > 100
    sub = _pile_subset(fr, seed + 1)
    f, decided, _ = ox.occupancy_exact(pts, res, sub)
    assert (f[decided] == fr[sub][decided]).all()


@pytest.mark.gpu
def test_refusals_raise_and_leave_the_context_usable():
    """A grid of 2^31 or more samples (also one whose per-axis count overflows int) and a resolution that is <= 0 in
    float32 raise CgError before anything is allocated or launched; the next call on the context still works."""
    from catgrasp_b200 import _lib, my_cpp
    big = np.array([[0.0, 0.0, 0.5], [1.3, 1.3, 1.8]], np.float32)          # 1310^3 samples at 1 mm
    with pytest.raises(_lib.CgError, match="2\\^31"):
        my_cpp.makeOccupancyGridFromCloudScan(big, np.eye(3), 0.001)
    with pytest.raises(_lib.CgError):
        my_cpp.makeOccupancyGridFromCloudScan(big, np.eye(3), 1e-12)        # (int) of 1.3e12 samples per axis
    for res in (0.0, -0.001, float("nan"), 1e-46):                          # 1e-46 rounds to 0 in float32
        with pytest.raises(_lib.CgError):
            my_cpp.makeOccupancyGridFromCloudScan(big, np.eye(3), res)
    # the C entry points refuse on their own too
    ctx = _lib.Context.get()
    p = np.ascontiguousarray(big)
    dims, org = (C.c_int * 3)(), (C.c_float * 3)()
    assert ctx.lib.cg_occupancy_grid_geometry(_lib.ptr(p), 2, C.c_float(0.0), dims, org) != 0
    assert ctx.lib.cg_occupancy_grid_geometry(_lib.ptr(p), 2, C.c_float(1e-12), dims, org) != 0
    one = np.zeros(1, np.uint8)
    ctx.use_own_stream()
    assert ctx.lib.cg_occupancy_from_scan_host(ctx.h, _lib.ptr(p), 2, C.c_float(-1.0), _lib.ptr(one)) != 0
    pts, r = _cases()["straddle"]
    _kernel_vs_oracle(pts, r)
