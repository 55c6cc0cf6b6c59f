"""CPU: the kd-tree evaluation of the 9-DoF RANSAC (aligning.py:68-79) in oracle/aligning_kdtree_ref.py against the
reference's own estimate9DTransform(use_kdtree_for_eval=True) (tests/golden/host_ransac9d_kdtree.npz, written by
tests/golden/make_golden_kdtree.py), and the argument checks of the product's kd-tree mode.

The oracle must reproduce the golden exactly (per-hypothesis ratios, the winner's T, its inliers, numpy's generator);
transforming the source in the kernel's operation order instead of numpy's matmul gives the same counts on every golden
hypothesis; and a restatement of the rule with one seeded mutation (denominator N, no dists2 term, origin without the
half voxel, strict `<`) misses the golden."""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import aligning_kdtree_ref

MIN_S, MAX_D = np.array([0.005, 0.005, 0.001]), np.array([1.2, 1.2, 1.2])
N_CASES = 5
MAX_ITER = 1000


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "host_ransac9d_kdtree.npz"))


def case(g, c):
    return (g[f"c{c}_source"], g[f"c{c}_target"], float(g[f"c{c}_thr"]), float(g[f"c{c}_res"]),
            g[f"c{c}_max_scale"], int(g[f"c{c}_seed"]))


@pytest.mark.parametrize("c", range(N_CASES))
def test_oracle_reproduces_golden(golden, c):
    src, tgt, thr, res, max_s, seed = case(golden, c)
    np.random.seed(seed)
    seen = []
    tf, inl = aligning_kdtree_ref.estimate9DTransform(src, tgt, thr, res, max_iter=MAX_ITER, max_scale=max_s,
                                                      min_scale=MIN_S, max_dimensions=MAX_D, ratios_out=seen)
    assert np.array_equal(np.random.rand(2), golden[f"c{c}_next_rand"])
    assert [i for i, _, _ in seen] == golden[f"c{c}_iters"].tolist()
    assert np.array([r for _, r, _ in seen]).tobytes() == golden[f"c{c}_ratios"].tobytes()
    assert np.array([T for _, _, T in seen]).tobytes() == golden[f"c{c}_T"].tobytes()
    assert tf.tobytes() == golden[f"c{c}_transform"].tobytes()
    assert np.array_equal(inl, golden[f"c{c}_inliers"])


@pytest.mark.parametrize("c", range(N_CASES))
def test_kernel_order_gives_the_same_counts(golden, c):
    src, tgt, thr, res, _, _ = case(golden, c)
    for T in golden[f"c{c}_T"]:
        a, ia = aligning_kdtree_ref.kdtree_eval(T, src, tgt, thr, res, order="matmul")
        b, ib = aligning_kdtree_ref.kdtree_eval(T, src, tgt, thr, res, order="kernel")
        assert a == b and np.array_equal(ia, ib)


def _down(p, r, mutation):
    origin = p.min(axis=0) - (0.0 if mutation == "origin_without_half_voxel" else r * 0.5)
    cells = np.floor((p - origin) / r).astype(np.int64)
    _, inv, counts = np.unique(cells, axis=0, return_inverse=True, return_counts=True)
    sums = np.zeros((len(counts), 3))
    np.add.at(sums, inv.reshape(-1), p)          # unbuffered: each voxel summed in ascending point index
    return sums / counts[:, None].astype(np.float64)


def restated_ratio(T, src, tgt, thr, r, mutation=None):
    """aligning.py:68-78 restated, with at most one seeded mutation."""
    src_t = (T @ np.c_[src, np.ones(len(src))].T).T[:, :3]
    d1 = cKDTree(_down(tgt, r, mutation)).query(src_t)[0]
    d2 = cKDTree(_down(src_t, r, mutation)).query(tgt)[0]
    ok = (lambda d: d < thr) if mutation == "strict_less" else (lambda d: d <= thr)
    count = int(ok(d1).sum()) + (0 if mutation == "no_dists2" else int(ok(d2).sum()))
    return count / (len(src) if mutation == "denominator_n" else 2 * len(src))


def _golden_ratios(golden, mutation):
    out = []
    for c in range(N_CASES):
        src, tgt, thr, res, _, _ = case(golden, c)
        out.append(np.array([restated_ratio(T, src, tgt, thr, res, mutation) for T in golden[f"c{c}_T"]]))
    return out


def test_restatement_matches_golden(golden):
    for c, got in enumerate(_golden_ratios(golden, None)):
        assert got.tobytes() == golden[f"c{c}_ratios"].tobytes(), c


@pytest.mark.parametrize("mutation", ["denominator_n", "no_dists2", "origin_without_half_voxel", "strict_less"])
def test_seeded_mutation_is_caught(golden, mutation):
    got = _golden_ratios(golden, mutation)
    assert any(g.tobytes() != golden[f"c{c}_ratios"].tobytes() for c, g in enumerate(got)), mutation


@pytest.mark.parametrize("r", [None, 0.0, -0.003, float("nan"), float("inf"), "abc"])
def test_bad_resolution_raises_before_the_device(r):
    from catgrasp_b200 import aligning
    from catgrasp_b200.predicter import NunocsPredicter
    src = np.random.RandomState(0).uniform(-0.5, 0.5, (16, 3))
    state = np.random.get_state()
    with pytest.raises(ValueError):
        aligning.estimate9DTransform(src, src, 0.003, max_iter=4, use_kdtree_for_eval=True, kdtree_eval_resolution=r)
    assert np.array_equal(np.random.get_state()[1], state[1])          # no draw was made
    if r is not None:                                                   # None: ransac9d_pose's residual mode
        with pytest.raises(ValueError):
            aligning.ransac9d_pose(src, src, np.zeros((4, 4), np.int32), (0.003,), kdtree_eval_resolution=r)
    p = NunocsPredicter.__new__(NunocsPredicter)
    p.subsample, p.use_kdtree_for_eval, p.kdtree_eval_resolution = "host", True, r
    with pytest.raises(ValueError):
        p.predict({})

