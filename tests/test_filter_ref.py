"""CPU: the float32 filter oracle (oracle/filter_ref.c) against the float64 predicate of oracle/filter64.py.

filter_ref.c is pinned to the reference build's survivors, but in that build the geometry predicate is filter_ref.c's
own fp32 code.  filter64 states the predicate plainly in float64 (pose composition, inv(cur @ gripper_in_grasp),
(p - origin) / res, meshpy's lookups) with a rigorous bound on the float32 pipeline, so a mistake shared by both float32
copies shows up here on every pose whose verdict the bound decides."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_mycpp as mk  # noqa: E402  (case tables + input builders shared with the generator)

from oracle import filter64, filter_ref, sdf_ref  # noqa: E402


def test_trilinear64_is_sdf_ref():
    from catgrasp_b200.synthetic import make_gripper_proxy
    rng = np.random.RandomState(0)
    grids = [make_gripper_proxy()["open"]["sdf"]] + [rng.normal(size=s) for s in [(1, 5, 5), (2, 3, 1), (1, 1, 1), (4, 2, 3)]]
    for d in grids:
        d = np.asarray(d, np.float64)
        c = rng.uniform(-3, max(d.shape) + 3, (3, 20000))
        c[:, :500] = np.round(c[:, :500])                       # lattice points, incl. the last cell on every axis
        c[:, 500:600] = (np.array(d.shape) - 1)[:, None]
        got, ref = filter64.trilinear64(d, c), sdf_ref.signed_distance(d, c)
        assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))


@pytest.mark.parametrize("k", range(len(mk.FILTER_CASES)))
def test_filter_oracle_agrees_with_float64_predicate(k):
    S, scale, mode, adjust, fdir = mk.FILTER_CASES[k]
    (p1, p2, poses, sym, nocs_pose, c2n, g), _ = mk.filter_inputs(S, scale)
    args = (poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], fdir, adjust, mode, g["open"], p1, g["enclosed"], p2)
    st, off, out = filter_ref.filter_ref(*args)
    r = filter64.filter64(*args)
    bad, undecided = filter64.compare(r, st, off, out)
    print(f"case {k}: {len(st)} poses, {undecided} undecided")
    assert bad == 0
    assert undecided <= 0.02 * len(st)
    dec = r["decided"]
    assert (r["status"][dec] == 0).any() and (r["status"][dec] == 3).any()
    if fdir:
        assert (r["status"][dec] == 1).any()
    if adjust:
        assert len(set(r["offset"][dec & (r["status"] == 0)].tolist())) >= 2


def test_float64_predicate_split_status():
    """split status (3 = the object's points hit, 4 = only the background does) on the sideways-shifted inputs"""
    S, scale, mode, adjust, fdir = mk.FILTER_CASES[1]
    (p1, p2, poses, sym, nocs_pose, c2n, g), _ = mk.filter_inputs(S, scale)
    poses = mk.shift_sideways(poses, 0.02)
    args = (poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], fdir, adjust, mode, g["open"], p1, g["enclosed"], p2)
    st, off, out = filter_ref.filter_ref(*args, split=True)
    r = filter64.filter64(*args, split=True)
    assert filter64.compare(r, st, off, out)[0] == 0
    dec = r["decided"]
    assert (r["status"][dec] == 3).any() and (r["status"][dec] == 4).any()


def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _grid_coords32(g32, gig, sdf, pts, mutation):
    """The kernel's camera -> grid chain in numpy float32 (affine_inverse, fold_grid, three fmas) at offset 0."""
    from catgrasp_b200.my_cpp import _mm4_f32
    A = _mm4_f32(g32, np.asarray(gig, np.float32)).reshape(-1, 16)
    a, b, c, d, e, f, g, h, i = (A[:, j] for j in (0, 1, 2, 4, 5, 6, 8, 9, 10))
    c00, c01, c02 = e * i - f * h, f * g - d * i, d * h - e * g
    r = np.float32(1) / ((a * c00 + b * c01) + c * c02)
    R = np.stack([c00 * r, (c * h - b * i) * r, (b * f - c * e) * r, c01 * r, (a * i - c * g) * r, (c * d - a * f) * r,
                  c02 * r, (b * g - a * h) * r, (a * e - b * d) * r], 1)
    t = np.stack([-((R[:, 3 * k] * A[:, 3] + R[:, 3 * k + 1] * A[:, 7]) + R[:, 3 * k + 2] * A[:, 11]) for k in range(3)], 1)
    inv_res = np.float32(1) / np.float32(sdf["res"])
    org = np.asarray(sdf["origin"], np.float32)
    if mutation == "transposed_rotation":
        R = R.reshape(-1, 3, 3).transpose(0, 2, 1).reshape(-1, 9)
    G = R * inv_res
    T = ((t + org) if mutation == "origin_added" else (t - org)) * inv_res
    x, y, z = (np.asarray(pts, np.float32)[None, :, k] for k in range(3))
    out = []
    for k in range(3):
        out.append(_fma32(G[:, 3 * k + 2, None], z, _fma32(G[:, 3 * k + 1, None], y, _fma32(G[:, 3 * k, None], x,
                                                                                       T[:, k, None]))))
    return np.stack(out, -1)                                  # (Q, P, 3)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("mutation", [None, "transposed_rotation", "origin_added"])
def test_float64_bound_rejects_a_wrong_grid_transform(mode, mutation):
    """The per-pose minimum of sd - margin over the object's points, computed by a float32 copy of the kernel's chain,
    lies inside the float64 interval [lo, hi] for every pose; with the fold_grid rotation transposed or the origin
    added instead of subtracted it does not.  Both mutations stay bit-identical between kernel and filter_ref.c, so
    only this check can see them."""
    from catgrasp_b200.my_cpp import grasp_in_cam_unshifted
    S, scale = 12, (1.0, 1.1, 0.9)
    (p1, p2, poses, sym, nocs_pose, c2n, g), _ = mk.filter_inputs(S, scale)
    poses = mk.shift_sideways(poses, 0.02)[:32]          # the open gripper lands in the object on every third pose
    margin = np.float32(0.0004)
    r = filter64.filter64(poses, sym, nocs_pose, c2n, g["gripper_in_grasp"], False, False, mode, g["open"], p1, None,
                          np.zeros((0, 3)), margin=margin)
    g32 = grasp_in_cam_unshifted(poses, sym, nocs_pose, c2n)
    gc = _grid_coords32(g32, g["gripper_in_grasp"], g["open"], p1, mutation)
    sd = filter_ref.sdf_lookup_ref(g["open"]["sdf"], gc.reshape(-1, 3), mode).reshape(gc.shape[:2]).astype(np.float64)
    if mode == 1:                                          # nearest: points outside the grid are dropped
        R = np.rint(gc)
        inb = ((R >= 0) & (R < np.array(g["open"]["sdf"].shape))).all(-1)
        sd = np.where(inb, sd, np.inf)
    m32 = (sd - float(margin)).min(1)
    lo, hi = r["open"]["lo"][:, 0], r["open"]["hi"][:, 0]
    outside = (m32 < lo) | (m32 > hi)
    if mutation is None:
        assert not outside.any()
        assert (hi < 0).any() and (lo >= 0).any()          # both verdicts occur among the decided poses
    else:
        assert outside.sum() >= len(m32) // 4, (mutation, int(outside.sum()))
