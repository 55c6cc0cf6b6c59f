"""CPU: pin oracle/ransac64.py (one RANSAC hypothesis in high precision, with margins and error bounds) against the
reference's own hypothesis code with real cv2 (oracle/aligning_ref._hypothesis), hypothesis by hypothesis, and
replay the reference's selection rule over it to reproduce both RANSAC goldens."""
import copy
import os

import mpmath as mp
import numpy as np
import pytest

from oracle import aligning_ref, ransac64, transforms_ref

THR = 0.003
MIN_S, MAX_S, MAX_D = np.array([0.005, 0.005, 0.001]), np.array([0.05] * 3), np.array([1.2] * 3)


def golden_ransac_case(golden_dir):
    """host_ransac9d.npz and the 3000 seed-3 draws of its reference run."""
    g = np.load(os.path.join(golden_dir, "host_ransac9d.npz"))
    np.random.seed(3)
    ids = np.array([np.random.choice(len(g["source"]), 4, replace=False) for _ in range(3000)], np.int32)
    return g, ids


def lattice_case(golden_dir, n_draws):
    """host_nunocs_lattice.npz: the NOCS cloud (0.01 lattice, many repeated points) against the observed cloud, and
    the first n_draws of the reference's first RANSAC call (threshold 0.003) under its seed."""
    g = np.load(os.path.join(golden_dir, "host_nunocs_lattice.npz"))
    cfg = {"n_pts": 8192, "ce_loss_bins": 100, "mean": g["mean"], "std": g["std"]}
    data = {"cloud_xyz": g["cloud_xyz"], "cloud_normal": g["cloud_normal"].astype(np.float64)}
    np.random.seed(0)
    dt = transforms_ref.nunocs_transform(copy.deepcopy(data), cfg)
    np.testing.assert_array_equal(dt["keep_ids"], g["keep_ids"])
    src = g["nocs_cloud"].astype(np.float64)
    tgt = dt["cloud_xyz_original"]
    ids = np.array([np.random.choice(len(src), 4, replace=False) for _ in range(n_draws)], np.int32)
    return g, src, tgt, ids


def _agree_with_cv2(src, tgt, ids, max_dims=MAX_D, min_s=MIN_S, max_s=MAX_S):
    """oracle vs aligning_ref._hypothesis (cv2) on every hypothesis; returns (#decided, #undecided, #valid)."""
    res = ransac64.evaluate(src, tgt, ids, THR, min_s, max_s, max_dims)
    und = nval = 0
    sh = np.c_[src, np.ones(len(src))]
    for h, r in enumerate(res):
        Tr = aligning_ref._hypothesis(src[ids[h]], tgt[ids[h]], tgt, THR, max_s, min_s, max_dims)
        if r["valid"] is None:
            und += 1
            continue
        assert (Tr is not None) == r["valid"], (h, r["gates"], r["info"])
        if Tr is not None:
            nval += 1
            assert np.abs(Tr - r["T"]).max() <= r["bound"], h
            cnt = int(np.count_nonzero(np.linalg.norm(sh @ Tr[:3].T - tgt, axis=1) <= THR))
            assert r["lo"] <= cnt <= r["hi"], (h, cnt, r["lo"], r["hi"])
    return len(res) - und, und, nval


def test_oracle_agrees_with_cv2_on_golden_draws(golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    dec, und, nval = _agree_with_cv2(g["source"], g["target"], ids)
    assert und <= len(ids) // 100 and nval >= 10


def test_oracle_agrees_with_cv2_on_lattice_draws(golden_dir):
    """NOCS points sit on a 0.01 lattice: 4-subsets with a repeated source point are singular, and cv2 answers them
    with the minimum-norm affine."""
    g, src, tgt, ids = lattice_case(golden_dir, 2000)
    s, _ = ransac64.narrow(src, tgt, ids)
    dup = sum(len(np.unique(q, axis=0)) < 4 for q in s)
    assert dup >= 3
    dec, und, nval = _agree_with_cv2(src, tgt, ids)
    assert und <= len(ids) // 100 and nval >= 10


def singular_subsets(src, rng, inliers, n):
    """Hand-built singular 4-subsets (index lists into src): a point, two inliers, and a second point with the same
    narrowed source value as the first (a duplicate NOCS value)."""
    key = {}
    s32 = src.astype(np.float32)
    for i, p in enumerate(map(bytes, s32)):
        key.setdefault(p, []).append(i)
    dups = [v for v in key.values() if len(v) > 1]
    out = []
    while len(out) < n:
        grp = dups[rng.randint(len(dups))]
        a, b = rng.choice(grp, 2, replace=False)
        c, d = rng.choice(inliers, 2, replace=False)
        out.append([a, c, d, b])
    return np.array(out, np.int32)


def test_oracle_agrees_with_cv2_on_singular_subsets(golden_dir):
    g, src, tgt, _ = lattice_case(golden_dir, 0)
    T = g["call_transforms"][0]
    err = np.linalg.norm(np.c_[src, np.ones(len(src))] @ T[:3].T - tgt, axis=1)
    rng = np.random.RandomState(5)
    ids = singular_subsets(src, rng, np.nonzero(err <= THR)[0], 400)
    res = ransac64.evaluate(src, tgt, ids, THR, MIN_S, MAX_S, MAX_D)
    assert all(r["info"]["singular"] for r in res)
    dec, und, nval = _agree_with_cv2(src, tgt, ids)
    assert nval >= 1 and und <= 4
    # coplanar (z = 0) and collinear subsets near the golden's true transform: a zero or rank-deficient affine
    truth = np.load(os.path.join(golden_dir, "host_ransac9d.npz"))["truth"]
    q = rng.uniform(-0.5, 0.5, (80, 3))
    q[:40, 2] = 0.0
    q[40:] = q[40:, :1].astype(np.float32).astype(np.float64) * [1.0, 0.5, -0.25]     # collinear after narrowing too
    d = np.c_[q, np.ones(len(q))] @ truth[:3].T + rng.normal(0, 1e-4, q.shape)
    ids = np.arange(80, dtype=np.int32).reshape(20, 4)
    for mdims in (MAX_D, None):
        assert all(r["info"]["singular"] for r in ransac64.evaluate(q, d, ids, THR, MIN_S, MAX_S, mdims))
        dec, und, nval = _agree_with_cv2(q, d, ids, max_dims=mdims)
        assert und == 0


def test_cv2_truncation_cut():
    """The cut of the minimum-norm solve (6 DBL_EPSILON x sum of M's singular values) against cv2: a subset whose
    smallest singular value is 0.7x the cut is truncated by both, one at 1.4x is solved in full by both."""
    import cv2
    d = np.random.RandomState(1).uniform(-0.5, 0.5, (4, 3)).astype(np.float32).astype(np.float64)
    for f, truncated in ((0.7, True), (1.4, False)):
        # [0, e1, e2, e3 * e]: sigma_min ~ e * const; solve for e at the wanted multiple of the cut
        lo, hi = 1e-17, 1e-12
        for _ in range(200):
            e = float(np.float32(np.sqrt(lo * hi)))
            s4 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, e]], np.float64)
            sv = np.linalg.svd(np.c_[s4, np.ones(4)], compute_uv=False)
            r = sv[-1] / (ransac64.CV2_CUT * sv.sum())
            if abs(r - f) < 0.02:
                break
            lo, hi = (e, hi) if r < f else (lo, e)
        assert abs(r - f) < 0.05
        X, info = ransac64.solve_affine(s4, d)
        assert not info["cut_undecided"] and info["singular"] == truncated
        _, Tc, _ = cv2.estimateAffine3D(s4, d, confidence=0.999, ransacThreshold=THR)
        assert (np.abs(Tc).max() < 10) == truncated
        if truncated:
            assert np.abs(np.array(X.tolist(), float).T - Tc).max() < 1e-12


def test_replay_reproduces_goldens(golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    res = ransac64.evaluate(g["source"], g["target"], ids, THR, MIN_S, MAX_S, MAX_D)
    w = ransac64.replay_winner(res)
    np.testing.assert_allclose(res[w]["T"], g["transform"], rtol=0, atol=1e-9)
    sh = np.c_[g["source"], np.ones(len(g["source"]))]
    inl = np.nonzero(np.linalg.norm(sh @ res[w]["T"][:3].T - g["target"], axis=1) <= THR)[0]
    np.testing.assert_array_equal(inl, g["inliers"])
    gl, src, tgt, ids = lattice_case(golden_dir, 10000)
    res = ransac64.evaluate(src, tgt, ids, THR, MIN_S, MAX_S, MAX_D, stop_at_full=True)
    w = ransac64.replay_winner(res)
    assert res[w]["lo"] == len(src)                         # ratio exactly 1.0: the first holder wins the tie
    np.testing.assert_allclose(res[w]["T"], gl["call_transforms"][0], rtol=0, atol=1e-9)


@pytest.mark.parametrize("mutation", ["swapped_scale_axes", "no_det", "transposed_inverse"])
def test_perturbed_oracle_is_caught(golden_dir, monkeypatch, mutation):
    """Each gate matters on the golden draws: a deliberately wrong copy of the oracle disagrees with cv2."""
    g, ids = golden_ransac_case(golden_dir)
    # plus 5 subsets through the true transform mirrored in z (det < 0, every other gate passes)
    q = np.random.RandomState(9).uniform(-0.5, 0.5, (20, 3))
    mirrored = np.c_[q, np.ones(20)] @ (g["truth"] @ np.diag([1.0, 1.0, -1.0, 1.0]))[:3].T
    src, tgt = np.r_[g["source"], q], np.r_[g["target"], mirrored]
    ids = np.r_[ids, len(g["source"]) + np.arange(20, dtype=np.int32).reshape(5, 4)]
    if mutation == "swapped_scale_axes":             # row norms instead of column norms
        monkeypatch.setattr(ransac64, "column_scales", lambda A: [mp.sqrt(sum(A[j, i] ** 2 for i in range(3))) for j in range(3)])
    elif mutation == "no_det":
        monkeypatch.setattr(ransac64, "polar_det", lambda Ro: abs(ransac64.mp.det(Ro)))
    else:
        right = ransac64.canonical_inverse

        def transposed(Ro, sc, t):
            return right(Ro.T, sc, t)
        monkeypatch.setattr(ransac64, "canonical_inverse", transposed)
    with pytest.raises(AssertionError):         # (the mirrored subsets fail max_dims in z, so no_det runs without it)
        _agree_with_cv2(src, tgt, ids, max_dims=None if mutation == "no_det" else MAX_D)
