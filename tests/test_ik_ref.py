"""The closed-form iiwa14 IK restatement (oracle/ik_ref.py, the CPU twin of csrc/cg_ik.cu) against the reference's
generated ikfast solver, as pinned in tests/golden/ik_iiwa14.npz (tests/golden/make_golden_ik.py) and, where the
oracle/_ref build exists, live."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_ik import (IK_LOWER, IK_UPPER, TIGHT_LOWER, TIGHT_UPPER, digest,  # noqa: E402
                            inputs)
from oracle import ik_ref  # noqa: E402
from catgrasp_b200 import ik as cg_ik  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ik_iiwa14.npz"))
FAMILIES = ["fk", "rigid", "shoulder", "wrist", "elbow", "reach", "limit"]


@pytest.fixture(scope="module")
def data():
    P, fam, fk_q = inputs()
    assert (digest(P, fam, fk_q, IK_UPPER, IK_LOWER, TIGHT_UPPER, TIGHT_LOWER) == GOLD["inputs_sha"]).all(), \
        "the input generator drifted from the fixture"
    ca, sol = ik_ref.iiwa14_ik(P, IK_UPPER, IK_LOWER)
    cb, _ = ik_ref.iiwa14_ik(P, TIGHT_UPPER, TIGHT_LOWER)
    return P, fam, fk_q, ca, cb, sol, ik_ref.in_band(P)


def same_set(mine, ref, tol):
    """Solution sets equal within tol (angles compared modulo 2 pi); returns the worst matched deviation or None."""
    if len(mine) != len(ref):
        return None
    worst = 0.0
    used = np.zeros(len(mine), bool)
    for r in ref:
        d = np.abs(np.angle(np.exp(1j * (mine - r)))).max(axis=1)
        d[used] = np.inf
        k = int(np.argmin(d))
        if d[k] > tol:
            return None
        used[k] = True
        worst = max(worst, float(d[k]))
    return worst


def test_fk_matches_ikfast():
    assert np.abs(ik_ref.iiwa14_fk(GOLD["fk_q"]) - GOLD["fk_T"]).max() < 1e-12
    assert np.abs(cg_ik.iiwa14_fk(GOLD["fk_q"]) - GOLD["fk_T"]).max() < 1e-12
    T0 = ik_ref.iiwa14_fk(np.zeros(7))
    assert np.allclose(T0[:3, 3], [0, 0, 1.261], atol=1e-15) and np.allclose(T0[:3, :3], np.eye(3), atol=1e-15)


def test_shoulder_band_bisection():
    assert np.abs(GOLD["shoulder_bisect"] - ik_ref.SHOULDER_BAND).max() < 1e-6


def test_solution_sets_match_outside_bands(data):
    P, fam, _, _, _, sol, band = data
    idx = GOLD["sol_index"]
    nsol = GOLD["nsol"].astype(int)
    starts = np.concatenate([[0], np.cumsum(nsol[idx])])
    worst, checked, skipped = 0.0, 0, 0
    for n, i in enumerate(idx):
        if band[i]:
            skipped += 1
            continue
        ref = GOLD["sol"][starts[n]:starts[n + 1]].astype(np.float64)
        mine = sol[i][~np.isnan(sol[i][:, 0])]
        w = same_set(mine, ref, 1e-6)
        assert w is not None, (i, FAMILIES[fam[i]], mine, ref)
        worst = max(worst, w)
        checked += 1
    print(f"solution sets: {checked} poses equal to ikfast's within {worst:.2e} rad, {skipped} inside the bands")
    # every pose's solution count, stored for all of them
    ok = ~band
    assert ((~np.isnan(sol[ok][:, :, 0])).sum(axis=1) == nsol[ok]).all()


@pytest.mark.parametrize("which", ["a", "b"])
def test_counts_and_verdicts_match_outside_bands(data, which):
    P, fam, _, ca, cb, _, band = data
    mine = ca if which == "a" else cb
    ref = GOLD[f"count_{which}"]
    ok = ~band
    for f, name in enumerate(FAMILIES):
        m = fam == f
        print(f"{name}: {m.sum()} poses, {(m & band).sum()} inside the bands")
    assert (fam[band] != 1).all(), "random rigid poses should lie outside every band"
    assert (mine[ok] == ref[ok]).all(), np.nonzero(ok & (mine != ref))[0][:10]
    assert ((mine[ok] > 0) == (ref[ok] > 0)).all()
    # the families exercise what they are meant to: both verdicts occur
    assert (ref[fam == 6] > 0).any() and (ref[fam == 6] == 0).any()


def test_special_cases():
    eye = np.eye(4)
    nan = eye.copy()
    nan[0, 3] = np.nan
    inf = eye.copy()
    inf[1, 1] = np.inf
    c, s = ik_ref.iiwa14_ik(np.stack([nan, inf]), IK_UPPER, IK_LOWER)
    assert (c == 0).all() and np.isnan(s).all()
    q = np.array([0.3, 0.5, 0.0, 1.0, 0.2, 0.7, -0.4])
    T = ik_ref.iiwa14_fk(q).astype(np.float32)
    assert ik_ref.iiwa14_ik(T[None], IK_UPPER, IK_LOWER)[0][0] == 8
    assert ik_ref.iiwa14_ik(T[None], IK_LOWER, IK_UPPER)[0][0] == 0        # lower > upper
    with pytest.raises(ValueError):
        cg_ik.joint_limits(IK_UPPER[:6], IK_LOWER[:6])
    up, lo = cg_ik.joint_limits(list(IK_UPPER) + [9.0], list(IK_LOWER) + [-9.0])
    assert up.shape == (7,) and (up == IK_UPPER).all()


def test_live_reference_build(data):
    from oracle import mycpp_ref_ik
    if not mycpp_ref_ik.available():
        pytest.skip("oracle/_ref is not built (no reference checkout)")
    P, fam, _, ca, _, sol, band = data
    rng = np.random.RandomState(0)
    pick = np.concatenate([np.nonzero(fam >= 2)[0], rng.choice(np.nonzero(fam < 2)[0], 1500, replace=False)])
    worst = 0.0
    for i in pick:
        if band[i]:
            continue
        ref = mycpp_ref_ik.ik_solutions(P[i])
        w = same_set(sol[i][~np.isnan(sol[i][:, 0])], ref, 1e-6)
        assert w is not None, i
        worst = max(worst, w)
        assert len(mycpp_ref_ik.ik_within_limits(P[i], IK_UPPER, IK_LOWER)) == ca[i]
    print(f"live ikfast: worst deviation {worst:.2e} rad")


@pytest.mark.parametrize("k", [0, 1])
def test_counts_on_filter_ik_cases(k):
    """The in-limit counts the compiled reference's ikfast gave on the collision survivors of the filter_ik cases of
    mycpp_filter.npz (their poses are float32 products of scaled poses, which ikfast rejects when not orthonormal)."""
    from make_golden_mycpp import IK_CASES, filter_inputs, ik_frames
    from oracle import filter_ref
    from catgrasp_b200.my_cpp import _mm4_f32, grasp_in_cam_unshifted
    S, scale, mode, adjust, fdir = IK_CASES[k]
    (p1, p2, P, sym, nocs, c2n, g), _ = filter_inputs(S, scale)
    cam, ee = ik_frames()
    st, _, _ = filter_ref.filter_ref(P, sym, nocs, c2n, g["gripper_in_grasp"], fdir, adjust, mode, g["open"], p1,
                                     g["enclosed"], p2)
    u = grasp_in_cam_unshifted(P, sym, nocs, c2n)
    f = lambda m: np.asarray(m, np.float64).astype(np.float32)      # noqa: E731
    eb = np.array([_mm4_f32(_mm4_f32(f(cam), u[q]), f(ee)) for q in np.nonzero(st == 0)[0]])
    runs = np.load(os.path.join(HERE, "golden", "mycpp_ref_runs.npz"))
    assert not ik_ref.in_band(eb).any()
    assert (ik_ref.iiwa14_ik(eb, IK_UPPER, IK_LOWER)[0].astype(np.int64) == runs[f"ik_counts_{k}"]).all()
