"""GPU tests (-m gpu) of the cone sampler's kernels (csrc/cg_cone.cu): cone_pose_kernel (R0 . R_sphere . R_inplane x
approach depths) and center_grasp_kernel (the object's y extent in the grasp frame, one 128-thread CTA per pose).

Exact checks, no tolerance: R0's own poses (rotation r = 0) are numpy's normalizeRotation and left-to-right translation
bit for bit, and the reference's recorded poses for the uncentred golden cases; with signed-permutation sphere and
in-plane tables every product is exact, so every pose is numpy's; the float32 copy is the float64 pose narrowed, with
and without centring; the bottom row is (0, 0, 0, 1); centring leaves the rotation block alone; two runs agree; and
centring gives the same bits wherever the points sit (point count around the warp, block and stride sizes; reversed,
duplicated, extremes moved).  Bounded checks: every other entry is within twice the bound of oracle/cone_ref.py's
exact evaluation (``exact_poses``, and ``exact_center`` given the kernel's own uncentred poses); each comparison prints
its largest error / (2 x bound) ratio.  Refusals go through the C ABI with small dummy buffers and launch nothing.

Seeded mutations of cg_cone.cu, each with the first test that fails on it (others that fail too in brackets):
  sphere and in-plane indices swapped (/ <-> %)      test_golden_r0_poses_bit_exact_with_reference_run, on its bound
                                                     (test_signed_permutation_tables_bit_exact,
                                                     test_poses_within_exact_bound at NS, NI > 1)
  translation re-associated, p + (b a + a d)         test_r0_poses_bit_exact_with_numpy (test_golden_r0_...,
                                                     test_signed_permutation_tables_bit_exact)
  fma in the column norm                             test_r0_poses_bit_exact_with_numpy (test_golden_r0_..., case 2;
                                                     test_signed_permutation_tables_bit_exact)
  centring combines warp 0's min / max only          test_narrowing_centring_and_repeat, on its bound
                                                     (test_center_independent_of_point_order from M = 33)
  centring loop not strided (one point per thread)   test_narrowing_centring_and_repeat, on its bound
                                                     (test_center_independent_of_point_order from M = 129)
  row 0 of the inverse instead of row 1              test_narrowing_centring_and_repeat, on its bound
                                                     (test_center_independent_of_point_order, on its bound)
  poses32 not updated by centring                    test_narrowing_centring_and_repeat
                                                     (test_poses_within_exact_bound)
"""
import os

import numpy as np
import pytest
import torch

from catgrasp_b200 import _lib
from catgrasp_b200 import grasp_sampler as gs
from oracle import cone_ref
from oracle.encoder_ref import bound_ratio

pytestmark = pytest.mark.gpu

INIT_BITE = 0.002
CT = 128          # threads per block of both kernels


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return _lib.Context.get(0)


def _dev(a):
    return None if a is None or len(a) == 0 else torch.from_numpy(np.array(a, np.float64, order="C")).cuda()


def run(ctx, surf, R0s, Rs, Ri, depths, pts=None, bite=INIT_BITE):
    """cg_cone_poses_dev, then cg_center_grasps_dev if ``pts`` is given, with explicit tables (an empty table is
    passed as NULL).  Returns (poses64, poses32) as numpy (P,4,4); the outputs start as NaN."""
    S, NS, NI, ND = len(surf), len(Rs), len(Ri), len(depths)
    P = S * (1 + NS * NI) * ND
    o64 = torch.full((P, 4, 4), float("nan"), dtype=torch.float64, device="cuda")
    o32 = torch.full((P, 4, 4), float("nan"), dtype=torch.float32, device="cuda")
    ctx.call("cg_cone_poses_dev", ctx.h, _dev(surf), _dev(R0s), S, _dev(Rs), NS, _dev(Ri), NI, _dev(depths), ND,
             float(bite), o64, o32)
    if pts is not None:
        ctx.call("cg_center_grasps_dev", ctx.h, o64, o32, P, _dev(pts), len(pts))
    torch.cuda.synchronize()
    return o64.cpu().numpy(), o32.cpu().numpy()


def tables(dirs, inplane_deg):
    """R_sphere and R_inplane as grasp_sampler.enumerate_poses builds them."""
    ref = np.array([1, 0, 0])
    Rs = np.stack([gs.directionVecToRotation(direction=d.copy(), ref=ref) for d in dirs]) if len(dirs) \
        else np.zeros((0, 3, 3))
    Ri = np.stack([gs.euler_matrix(x * np.pi / 180, 0, 0, axes="sxyz")[:3, :3] for x in inplane_deg])
    return Rs, Ri


def cone_dirs(rng, n):
    """n directions within 60 degrees of +x, like the view-sphere subset turned onto +x."""
    v = rng.normal(size=(16 * n + 64, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    v = v[v[:, 0] >= 0.5][:n]
    assert len(v) == n
    return v


def frames(kind, rng, S, z):
    """(surface points (S,3), R0s (S,3,3), object points (M,3)) around (0, 0, z)."""
    shift = np.array([0.0, 0.0, z - 0.7])
    if kind == "pile":
        from catgrasp_b200.synthetic import make_pile
        scene = make_pile(2400, n_objects=6, seed=43)
        m = scene["object_id"] == 3
        pts, nrm = scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
        np.random.seed(int(rng.randint(1 << 30)))
        ids, R0s, _ = gs.cone_frames(pts, nrm, S + 8, 1)      # a sample whose frame is complex is dropped
        return pts[ids[:S]] + shift, R0s[:S], pts + shift
    pts = np.array([0.0, 0.0, 0.7]) + rng.uniform(-0.04, 0.04, (300, 3)) + shift
    surf = pts[rng.choice(len(pts), S, replace=False)]
    from catgrasp_b200.synthetic import random_rotation
    if kind == "orthonormal":
        return surf, np.stack([random_rotation(rng) for _ in range(S)]), pts
    # unit columns, the minor axis tilted off the plane normal to the approach axis: det = sin(tilt) from 1 to 1e-3,
    # the frames cone_frames returns when the smallest principal direction is almost the approach axis
    R0s = []
    for det in np.geomspace(1.0, 1e-3, S):
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        m = np.cross(a, rng.normal(size=3))
        m /= np.linalg.norm(m)
        minor = np.sqrt(1 - det * det) * a + det * m
        minor /= np.linalg.norm(minor)
        major = np.cross(minor, a)
        major /= np.linalg.norm(major)
        R0s.append(np.stack([a, major, minor], 1))
    return surf, np.array(R0s), pts


def ratio(label, got, ref, err):
    assert np.isfinite(got).all(), label
    r = float(bound_ratio(got, ref, err).max())
    print(f"\nRATIO cone {label} = {r:.3g}")
    assert r <= 1.0, (label, r)
    return r


def check_center(label, uncentred, centred, pts, sel=None):
    """The centred poses against exact_center applied to the kernel's own uncentred poses (rows ``sel``)."""
    sel = np.arange(len(uncentred)) if sel is None else sel
    ref, err = cone_ref.exact_center(uncentred[sel], pts)
    return ratio(label + " centred", centred[sel], ref, err)


# ------------------------------------------------------------------------------------------ exact checks
@pytest.mark.parametrize("kind", ["orthonormal", "pile", "skewed"])
@pytest.mark.parametrize("z", [0.7, 10.0])
def test_r0_poses_bit_exact_with_numpy(ctx, kind, z):
    """Rotation r = 0 is R0 itself: numpy's column normalisation and p + b a + a d, bit for bit, at every depth."""
    rng = np.random.RandomState(int(z * 10) + len(kind))
    surf, R0s, _ = frames(kind, rng, 40, z)
    Rs, Ri = tables(cone_dirs(rng, 2), np.arange(0, 180, 30))
    depths = np.arange(0, 0.012, 0.003)
    got64, got32 = run(ctx, surf, R0s, Rs, Ri, depths)
    want = cone_ref.poses_from_tables(surf, R0s, Rs[:0], Ri, depths, INIT_BITE)
    r0 = got64.reshape(len(surf), 1 + len(Rs) * len(Ri), len(depths), 4, 4)[:, 0].reshape(-1, 4, 4)
    assert np.array_equal(r0.view(np.uint64), want.view(np.uint64))


@pytest.mark.parametrize("k", [0, 2])
def test_golden_r0_poses_bit_exact_with_reference_run(ctx, golden_dir, k):
    """The uncentred golden cases through grasp_sampler.enumerate_poses: R0's poses are the recorded reference poses
    bit for bit, and every pose is within the exact oracle's bound."""
    import test_cone_golden as tc
    c = tc.CASES[k]
    surf, R0s, sph, Rs, Ri, dep, _ = tc.golden_tables(c)
    got64, got32 = gs.enumerate_poses(surf, R0s, sph, tc.HAND_DEPTH, c["approach_step"], tc.INIT_BITE)
    got64 = got64.cpu().numpy()
    gold = np.load(os.path.join(golden_dir, "cone_poses.npz"))[f"poses_{k}"]
    shape = (len(surf), 1 + len(Rs) * len(Ri), len(dep), 4, 4)
    assert np.array_equal(got64.reshape(shape)[:, 0].view(np.uint64), gold.reshape(shape)[:, 0].view(np.uint64))
    ref, err = cone_ref.exact_poses(surf, R0s, Rs, Ri, dep, tc.INIT_BITE, np.arange(len(gold)))
    ratio(f"golden case {k}", got64, ref, err)
    print(f"cone golden case {k}: {np.mean(got64 == gold):.4f} of entries equal the reference run's bits")


def _signed_permutations(rng, n):
    out = []
    for _ in range(n):
        M = np.zeros((3, 3))
        M[np.arange(3), rng.permutation(3)] = rng.choice([-1.0, 1.0], 3)
        out.append(M)
    return np.array(out)


@pytest.mark.parametrize("kind", ["orthonormal", "skewed"])
def test_signed_permutation_tables_bit_exact(ctx, kind):
    """Sphere and in-plane tables of signed permutations make every product exact, so every pose (each rotation,
    each depth, in the kernel's order) equals numpy's bit for bit; distinct tables tell the indices apart."""
    rng = np.random.RandomState(17)
    surf, R0s, _ = frames(kind, rng, 5, 0.7)
    Rs, Ri = _signed_permutations(rng, 7), _signed_permutations(rng, 5)
    depths = np.arange(0, 0.012, 0.004)
    got64, got32 = run(ctx, surf, R0s, Rs, Ri, depths)
    want = cone_ref.poses_from_tables(surf, R0s, Rs, Ri, depths, INIT_BITE)
    assert np.array_equal(got64.view(np.uint64), want.view(np.uint64))
    assert np.array_equal(got32.view(np.uint32), want.astype(np.float32).view(np.uint32))


def test_narrowing_centring_and_repeat(ctx):
    """The float32 copy is the float64 pose narrowed (with and without centring), the bottom row is exactly
    (0, 0, 0, 1), centring moves only the translation and moves it as the exact oracle does, and a second run is
    bitwise the first."""
    rng = np.random.RandomState(23)
    surf, R0s, pts = frames("pile", rng, 9, 0.7)
    Rs, Ri = tables(cone_dirs(rng, 8), np.arange(0, 180, 30))
    depths = np.arange(0, 0.012, 0.002)
    u64, u32 = run(ctx, surf, R0s, Rs, Ri, depths)
    c64, c32 = run(ctx, surf, R0s, Rs, Ri, depths, pts=pts)
    for a64, a32 in ((u64, u32), (c64, c32)):
        assert np.array_equal(a32.view(np.uint32), a64.astype(np.float32).view(np.uint32))
        assert (a64[:, 3] == np.array([0.0, 0.0, 0.0, 1.0])).all()
        assert not np.signbit(a64[:, 3]).any()
    assert np.array_equal(c64[:, :, :3].view(np.uint64), u64[:, :, :3].view(np.uint64))
    assert (c64[:, :3, 3] != u64[:, :3, 3]).any(axis=1).mean() > 0.99
    check_center("repeat case", u64, c64, pts)
    again64, again32 = run(ctx, surf, R0s, Rs, Ri, depths, pts=pts)
    assert np.array_equal(again64.view(np.uint64), c64.view(np.uint64))
    assert np.array_equal(again32.view(np.uint32), c32.view(np.uint32))


def moved(pts, a, pos, b, other):
    """``pts`` with point ``a`` moved to index ``pos`` and then point ``b`` to ``other``, each by a swap."""
    order = np.arange(len(pts))
    for src, dst in ((a, pos), (b, other)):
        i = int(np.nonzero(order == src)[0][0])
        order[[i, dst]] = order[[dst, i]]
    return pts[order]


CENTER_M = [1, 2, 31, 32, 33, 127, 128, 129, 255, 257, 4097, 1 << 20]


@pytest.mark.parametrize("M", CENTER_M)
def test_center_independent_of_point_order(ctx, M):
    """The y of each point is computed the same way whichever thread reads it, and min / max are exact, so the
    centred poses do not depend on where a point sits: in order, reversed, every point twice, and the highest and
    lowest points (planted along the frame's y axis) moved to 0, 31, 32, 127, 128 and M - 1 (each with the other
    extreme half the array away) must all give the same bits."""
    from catgrasp_b200.synthetic import random_rotation
    rng = np.random.RandomState(M % 1000003)
    R = random_rotation(rng)
    centre = np.array([0.01, -0.02, 0.7])
    surf = centre + rng.uniform(-0.02, 0.02, (4, 3))
    depths = np.arange(0, 0.012, 0.004)
    R0s = np.stack([R] * 4)
    Ri = np.eye(3)[None]
    u64, _ = run(ctx, surf, R0s, np.zeros((0, 3, 3)), Ri, depths)
    pts = centre + rng.uniform(-0.03, 0.03, (M, 3))
    hi, lo = 0, min(1, M - 1)
    pts[hi] = centre + 0.25 * R[:, 1]
    if M > 1:
        pts[lo] = centre - 0.3 * R[:, 1]
    arrangements = {"reversed": pts[::-1], "duplicated": np.concatenate([pts, pts])}
    for pos in sorted({p for p in (0, 31, 32, 127, 128, M - 1) if p < M}):
        other = (pos + M // 2) % M
        arrangements[f"hi@{pos}"] = moved(pts, hi, pos, lo, other)
        arrangements[f"lo@{pos}"] = moved(pts, lo, pos, hi, other)
    base64, base32 = run(ctx, surf, R0s, np.zeros((0, 3, 3)), Ri, depths, pts=pts)
    for name, q in arrangements.items():
        g64, g32 = run(ctx, surf, R0s, np.zeros((0, 3, 3)), Ri, depths, pts=np.ascontiguousarray(q))
        assert np.array_equal(g64.view(np.uint64), base64.view(np.uint64)), (M, name)
        assert np.array_equal(g32.view(np.uint32), base32.view(np.uint32)), (M, name)
    if M <= 4097:
        check_center(f"M={M}", u64, base64, pts)


# ------------------------------------------------------------------------------------------ bounded checks
SHAPES = [(1, 0, 6, 1),      # R0 only, NULL sphere table
          (1, 1, 1, 1),
          (3, 8, 6, 6),
          (5, 4, 6, 3)]      # S * NR = 125: the only block ends inside
FRAMES = ["orthonormal", "pile", "skewed"]


@pytest.mark.parametrize("kind", FRAMES)
@pytest.mark.parametrize("z", [0.7, 10.0])
@pytest.mark.parametrize("S,NS,NI,ND", SHAPES)
def test_poses_within_exact_bound(ctx, kind, z, S, NS, NI, ND):
    """Every entry of every pose, uncentred and centred, within twice the exact oracle's bound."""
    rng = np.random.RandomState(S * 1000 + NS * 100 + NI * 10 + ND + int(z))
    surf, R0s, pts = frames(kind, rng, S, z)
    Rs, Ri = tables(cone_dirs(rng, NS), np.arange(NI) * 30.0 + (45.0 if NI == 1 else 0.0))
    depths = np.arange(ND) * 0.002
    u64, u32 = run(ctx, surf, R0s, Rs, Ri, depths)
    c64, c32 = run(ctx, surf, R0s, Rs, Ri, depths, pts=pts)
    P = S * (1 + NS * NI) * ND
    assert u64.shape == (P, 4, 4)
    ref, err = cone_ref.exact_poses(surf, R0s, Rs, Ri, depths, INIT_BITE, np.arange(P))
    label = f"{kind} z={z} S,NS,NI,ND={S},{NS},{NI},{ND}"
    ratio(label, u64, ref, err)
    check_center(label, u64, c64, pts)
    assert np.array_equal(c32.view(np.uint32), c64.astype(np.float32).view(np.uint32))


def test_pick_sized_launch(ctx):
    """compute_candidate_grasp's size: every surface sample of a pile object (about 400), 30 sphere directions x 6
    in-plane angles (NR = 181), a 2 mm approach step (ND = 15), centred over the object's points: about 10^6 poses
    over thousands of blocks.  A sample of about 2 000 poses, with the first and last blocks of the enumeration, is
    compared with the exact oracle; the float32 copy of every pose with the float64 pose narrowed."""
    from catgrasp_b200.synthetic import make_pile
    scene = make_pile(2400, n_objects=6, seed=21)
    sizes = np.bincount(scene["object_id"])
    obj = int(np.argmin(np.abs(sizes - 400)))
    m = scene["object_id"] == obj
    pts, nrm = scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
    np.random.seed(5)
    ids, R0s, sph = gs.cone_frames(pts, nrm, np.inf, 30)
    surf = pts[ids]
    hand_depth, step = 0.03, 0.002
    u64, u32 = gs.enumerate_poses(surf, R0s, sph, hand_depth, step, INIT_BITE)
    c64, c32 = gs.enumerate_poses(surf, R0s, sph, hand_depth, step, INIT_BITE, points_for_center=pts)
    u64, c64, c32 = (a.cpu().numpy() for a in (u64, c64, c32))
    S, NS, ND = len(surf), len(sph), len(np.arange(0, hand_depth, step))
    NR = 1 + NS * 6
    assert S > 300 and len(pts) > 300 and NS == 30 and ND == 15 and len(c64) == S * NR * ND
    threads = S * NR
    last = (threads - 1) // CT * CT
    rng = np.random.RandomState(0)
    t = np.unique(np.concatenate([[0, 1, 31, 32, CT - 1, CT, CT + 1, last, last + 1, threads - 2, threads - 1],
                                  rng.choice(threads, 120, replace=False)]))
    sel = (t[:, None] * ND + np.arange(ND)).reshape(-1)
    Rs, Ri = tables(sph, np.arange(0, 180, 30))
    ref, err = cone_ref.exact_poses(surf, R0s, Rs, Ri, np.arange(0, hand_depth, step), INIT_BITE, sel)
    print(f"\ncone pick-sized launch: S={S} NR={NR} ND={ND} P={len(c64)} M={len(pts)}, {len(sel)} poses sampled")
    ratio("pick-sized", u64[sel], ref, err)
    check_center("pick-sized", u64, c64, pts, sel)
    assert np.array_equal(c32.view(np.uint32), c64.astype(np.float32).view(np.uint32))


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_before_any_launch(ctx):
    """Argument errors come back as CG_EINVAL before anything is launched (the context's launch count stays put),
    with buffers far too small for the sizes asked: 2^31 poses or more, including sizes whose product overflows 64
    bits; sphere or in-plane tables missing; no object points; empty or negative sizes.  P = 0 poses to centre is a successful no-op."""
    d = torch.zeros(64, dtype=torch.float64, device="cuda")
    f = torch.zeros(64, dtype=torch.float32, device="cuda")
    ctx.use_torch_stream()
    n0 = ctx.launch_count()
    big = (1 << 31) - 1

    def cone(S, NS, NI, ND, sph=d, inp=d):
        return ctx.lib.cg_cone_poses_dev(ctx.h, d, d, S, sph, NS, inp, NI, d, ND, INIT_BITE, d, f)

    for S, NS, NI, ND in [(1 << 16, 1 << 8, 1 << 7, 1),      # S * NR = 2^31 + 2^16
                          (1 << 15, 1 << 16, 1, 1),           # S * NR = 2^31 + 2^15
                          (2, 0, 0, 1 << 30),                 # P = 2^31 exactly
                          (1, 1 << 16, 1 << 15, 1),           # NR = 2^31 + 1
                          (big, 0, 0, big),
                          (3, big, 2, big),
                          (big, big, big, big)]:              # S * NR * ND overflows 64 bits
        assert S * (1 + NS * NI) * ND >= 1 << 31
        assert cone(S, NS, NI, ND) == _lib.CG_EINVAL, (S, NS, NI, ND)
    for sph, inp in ((None, d), (d, None), (None, None)):
        assert cone(1, 2, 3, 1, sph, inp) == _lib.CG_EINVAL
    assert cone(0, 0, 0, 1) == _lib.CG_EINVAL and cone(1, 0, 0, 0) == _lib.CG_EINVAL and cone(1, -1, 1, 1) == _lib.CG_EINVAL
    center = ctx.lib.cg_center_grasps_dev
    assert center(ctx.h, d, f, 4, d, 0) == _lib.CG_EINVAL
    assert center(ctx.h, d, f, 4, d, -1) == _lib.CG_EINVAL
    assert center(ctx.h, d, f, -1, d, 4) == _lib.CG_EINVAL
    assert center(ctx.h, d, f, 0, d, 4) == _lib.CG_OK
    assert ctx.launch_count() == n0
