"""CPU: the host half of the cone sampler (catgrasp_b200.grasp_sampler: view sphere, local frames, numpy-RNG stream)
and the enumeration oracle (oracle/cone_ref.py) against poses recorded from the reference's own
PointConeGraspSampler.sample_grasps (tests/golden/make_golden_cone.py)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

from catgrasp_b200 import grasp_sampler as gs  # noqa: E402
from oracle import cone_ref  # noqa: E402

CASES = [dict(n_pts=60, seed=4, n_sphere_dir=8, approach_step=0.005, center=False, max_num_samples=9),
         dict(n_pts=40, seed=5, n_sphere_dir=5, approach_step=0.004, center=True, max_num_samples=np.inf),
         dict(pile=(2400, 6, 43, 3), n_sphere_dir=6, approach_step=0.004, center=False, max_num_samples=12)]
HAND_DEPTH, INIT_BITE = 0.012, 0.002


def case_inputs(c):
    from catgrasp_b200 import synthetic
    if "pile" in c:
        n, k, seed, obj = c["pile"]
        scene = synthetic.make_pile(n, n_objects=k, seed=seed)
        m = scene["object_id"] == obj
        return scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
    rng = np.random.RandomState(c["seed"])
    pts, nrm = synthetic.sample_hex_nut(c["n_pts"], rng)
    R = synthetic.random_rotation(rng)
    return pts @ R.T + np.array([0.01, -0.02, 0.70]), nrm @ R.T


def test_view_sphere_matches_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "cone_poses.npz"))
    pts, level = gs.hinter_sampling(1000, radius=1)
    assert pts.shape == g["hinter_1000"].shape
    np.testing.assert_array_equal(pts, g["hinter_1000"])


def test_host_frames_and_enumeration_match_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "cone_poses.npz"))
    for k, c in enumerate(CASES):
        pts, nrm = case_inputs(c)
        np.random.seed(7)
        ids, R0s, sph = gs.cone_frames(pts, nrm, c["max_num_samples"], c["n_sphere_dir"])
        np.testing.assert_array_equal(np.random.rand(2), g[f"next_rand_{k}"])          # same RNG consumption
        poses = cone_ref.enumerate_poses(pts[ids], R0s, sph, HAND_DEPTH, c["approach_step"], INIT_BITE,
                                         points_for_center=pts if c["center"] else None)
        assert poses.shape == g[f"poses_{k}"].shape
        np.testing.assert_allclose(poses, g[f"poses_{k}"], rtol=0, atol=1e-14)


def golden_tables(c):
    """A golden case's enumeration inputs, with the rotation tables as the device wrapper builds them: (surface
    points, R0s, sphere directions, R_sphere, R_inplane, depths, object points)."""
    pts, nrm = case_inputs(c)
    np.random.seed(7)
    ids, R0s, sph = gs.cone_frames(pts, nrm, c["max_num_samples"], c["n_sphere_dir"])
    Rs = np.stack([gs.directionVecToRotation(sp.copy(), np.array([1, 0, 0])) for sp in sph])
    Ri = np.stack([gs.euler_matrix(x * np.pi / 180, 0, 0)[:3, :3] for x in np.arange(0, 180, 30)])
    return pts[ids], R0s, sph, Rs, Ri, np.arange(0, HAND_DEPTH, c["approach_step"]), pts


def test_exact_oracle_vs_numpy_and_reference_runs(golden_dir):
    """The exact enumeration (oracle/cone_ref.exact_poses) and centring (exact_center) against the numpy restatement
    and the recorded reference poses, every pose.  numpy's rotations and translations follow the kernel's operation
    classes (3-term products, the same normalisation and translation order), so they must lie within the kernel's
    bound; its centring inverts the 4x4 pose by LU and sums [p, 1] against the inverse's row, whose rounding is of
    order u |row| (|p| + |t|), so the recorded centred translations get that much more."""
    from oracle.encoder_ref import bound_ratio
    g = np.load(os.path.join(golden_dir, "cone_poses.npz"))
    worst = 0.0
    for k, c in enumerate(CASES):
        surf, R0s, sph, Rs, Ri, dep, pts = golden_tables(c)
        P = len(surf) * (1 + len(Rs) * len(Ri)) * len(dep)
        ref, err = cone_ref.exact_poses(surf, R0s, Rs, Ri, dep, INIT_BITE, np.arange(P))
        raw = cone_ref.poses_from_tables(surf, R0s, Rs, Ri, dep, INIT_BITE)
        assert np.array_equal(raw, cone_ref.enumerate_poses(surf, R0s, sph, HAND_DEPTH, c["approach_step"], INIT_BITE))
        r = {"numpy": bound_ratio(raw, ref, err).max()}
        gold = g[f"poses_{k}"]
        if c["center"]:
            cref, cerr = cone_ref.exact_center(raw, pts)
            row, _ = cone_ref._cofactor_row(raw)
            lu = 16 * cone_ref.U * (np.abs(row) @ np.abs(pts).T + (np.abs(row) * np.abs(raw[:, :3, 3])).sum(1)[:, None])
            cerr[:, :3, 3] += lu.max(1)[:, None] * np.abs(raw[:, :3, 1])
            r["reference run, centred"] = bound_ratio(gold, cref, cerr).max()
            r["numpy, centred"] = bound_ratio(cone_ref.enumerate_poses(surf, R0s, sph, HAND_DEPTH, c["approach_step"],
                                                                       INIT_BITE, pts), cref, cerr).max()
        else:
            r["reference run"] = bound_ratio(gold, ref, err).max()
        print(f"\nRATIO cone case {k} P={P} " + " ".join(f"{n}={v:.3g}" for n, v in r.items()))
        assert max(r.values()) <= 1.0, (k, r)
        worst = max(worst, *r.values())
        # not vacuous: unit-scale rotations are bounded well below the old flat 1e-13
        assert err[:, :3, :3].max() < 1e-14 and err[:, :3, 3].max() < 1e-15, k
    print(f"\nRATIO cone oracle largest {worst:.3g}")


def test_exact_oracle_on_known_values():
    """The oracle's own claims, on values whose exact results are known: a rotation it is given exactly (the bound then
    is only the normalisation's rounding and the rounded exact value's half ulp), a signed-permutation product, a
    non-orthonormal frame's columns, and a centring whose extreme points and shift are exact in float64."""
    rng = np.random.RandomState(3)
    R0 = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    Rs = np.array([[[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]]])
    Ri = np.array([[[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]]])
    surf = np.array([[0.25, -0.5, 0.75]])
    ref, err = cone_ref.exact_poses(surf, R0[None] * 2.0, Rs, Ri, [0.0, 0.5], 0.25, np.arange(4))
    want = np.stack([np.eye(4)] * 4)
    for n, R in enumerate([R0, R0, R0 @ Rs[0] @ Ri[0], R0 @ Rs[0] @ Ri[0]]):
        want[n, :3, :3] = R
        want[n, :3, 3] = surf[0] + (0.25 + 0.5 * (n % 2)) * R[:, 0]
    assert np.array_equal(ref, want)
    assert (err[:, 3] == 0).all() and err[:2, :3, :3].max() < 6e-16 and err.max() < 2e-15
    # unit columns at 60 degrees: R0 is not orthonormal, its columns stay where they are
    R1 = np.array([[1.0, 0.0, 0.5], [0.0, 1.0, 0.0], [0.0, 0.0, np.sqrt(0.75)]])
    ref, err = cone_ref.exact_poses(surf, R1[None], np.zeros((0, 3, 3)), Ri, [0.0], 0.0, [0])
    assert np.abs(ref[0, :3, :3] - R1).max() <= 1.2e-16 and np.array_equal(ref[0, :3, 3], surf[0])
    # centring: with R = I the grasp frame's y is the camera's, the extent of points y in {-0.25, ..., 0.5} is
    # centred at 0.125
    T = np.eye(4)[None].copy()
    T[0, :3, 3] = [0.5, 0.25, 0.75]
    pts = rng.uniform(-0.2, 0.2, (50, 3)) + T[0, :3, 3]
    pts[7, 1], pts[31, 1] = 0.25 - 0.25, 0.25 + 0.5
    ref, err = cone_ref.exact_center(T, pts)
    assert np.array_equal(ref[0, :3, 3], [0.5, 0.25 + 0.125, 0.75]) and np.array_equal(ref[0, :, :3], T[0, :, :3])
    assert err[0, :3, 3].max() < 1e-15 and (err[0, :, :3] == 0).all() and err[0, 3, 3] == 0
