"""oracle/meanshift_ref.py (the kernel's arithmetic restated in numpy) against the real sklearn MeanShift and the
reference's PointGroupPredictor.predict, and catgrasp_b200.segment's argument checks (CPU only)."""
import os

import numpy as np
import pytest

from catgrasp_b200 import segment, synthetic
from oracle import meanshift_ref

sklearn_cluster = pytest.importorskip("sklearn.cluster")


def shifted_pile(n_points, n_objects, seed, pull, noise=0.0008):
    """A pile whose points are pulled `pull` of the way to their object's centre, plus noise (float64)."""
    s = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    centre = s["object_poses"][:, :3, 3][s["object_id"]]
    rng = np.random.RandomState(seed + 7)
    return s["cloud_xyz"] + pull * (centre - s["cloud_xyz"]) + rng.normal(0, noise, s["cloud_xyz"].shape)


@pytest.mark.parametrize("pull", [0.85, 0.3], ids=["tight", "loose"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("bw", [0.005, 0.007, 0.009])
def test_oracle_matches_sklearn(bw, dtype, pull):
    X = shifted_pile(1500, 8, seed=1, pull=pull).astype(dtype)
    sk = sklearn_cluster.MeanShift(bandwidth=bw, cluster_all=True, n_jobs=-1, seeds=None).fit(X)
    o = meanshift_ref.fit(X, bw)
    assert np.array_equal(o["labels"], sk.labels_)
    assert o["n_iter"] == sk.n_iter_
    assert o["centres"].shape == sk.cluster_centers_.shape and o["centres"].dtype == sk.cluster_centers_.dtype
    tol = 1e-6 if dtype == np.float32 else 1e-12
    assert np.abs(o["centres"].astype(np.float64) - sk.cluster_centers_).max() <= tol


def test_oracle_is_independent_of_row_order():
    X = shifted_pile(1200, 6, seed=2, pull=0.6).astype(np.float32)
    perm = np.random.RandomState(0).permutation(len(X))
    a = meanshift_ref.fit(X, 0.007)
    b = meanshift_ref.fit(X[perm], 0.007)
    assert a["centres"].tobytes() == b["centres"].tobytes()
    assert np.array_equal(b["labels"], a["labels"][perm])
    assert b["seed_centres"].tobytes() == a["seed_centres"][perm].tobytes()


def test_oracle_composition_reproduces_reference_predict(golden_dir):
    g = np.load(os.path.join(golden_dir, "segment.npz"))
    for cls, bw in segment.MEANSHIFT_BANDWIDTH.items():
        labels_all, shifted = meanshift_ref.pointgroup_labels(g[f"{cls}_xyz_original_all"], g[f"{cls}_pt_offsets"],
                                                              g[f"{cls}_cloud_xyz"], bw)
        assert shifted.dtype == np.float32 and shifted.tobytes() == g[f"{cls}_xyz_shifted"].tobytes(), cls
        assert np.array_equal(labels_all, g[f"{cls}_labels_all"]), cls


def test_max_iter_zero_and_empty_sets_follow_sklearn():
    X = shifted_pile(600, 4, seed=3, pull=0.3).astype(np.float64)
    for max_iter in (0, 1):
        sk = sklearn_cluster.MeanShift(bandwidth=0.007, max_iter=max_iter).fit(X)
        o = meanshift_ref.fit(X, 0.007, max_iter=max_iter)
        assert o["n_iter"] == sk.n_iter_ == max_iter
        assert np.array_equal(o["labels"], sk.labels_)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_step_bruteforce_is_one_step_of_the_ascent(dtype):
    """The ascent at max_iter k, seed by seed: a seed still moving after run k - 1 (X itself before run 0) takes one
    step_bruteforce step from its centre there, and stops at k when that step is empty or shorter than 1e-3 bw; every
    other seed keeps run k - 1's result.  Each step lands within the fixed point's bound of its set's mean."""
    bw = 0.007
    X = shifted_pile(1500, 8, seed=1, pull=0.3).astype(dtype)
    origin, E = meanshift_ref.frame(X, bw)
    o, e, _ = meanshift_ref.quantise(X.astype(np.float64), bw)
    assert E == e and origin.tobytes() == o.tobytes()
    c_prev, n_prev, it_prev = X, np.zeros(len(X), np.int64), np.zeros(len(X), np.int64)
    moving = np.ones(len(X), bool)
    for k in range(5):
        c, n, it = meanshift_ref.ascent(X, bw, max_iter=k)
        assert c[~moving].tobytes() == c_prev[~moving].tobytes()
        assert np.array_equal(n[~moving], n_prev[~moving]) and np.array_equal(it[~moving], it_prev[~moving])
        new, cnt, mean = meanshift_ref.step_bruteforce(X, bw, c_prev[moving])
        assert new.tobytes() == c[moving].tobytes() and np.array_equal(cnt, n[moving]) and (it[moving] == k).all()
        assert (meanshift_ref.bound_ratio(new, mean, E) <= 1.0).all()
        d = (new - c_prev[moving]).astype(np.float64)
        step = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        moving[np.flatnonzero(moving)[(cnt == 0) | (step <= 1e-3 * bw)]] = False
        c_prev, n_prev, it_prev = c, n, it
    assert moving.any() and not moving.all()


@pytest.mark.parametrize("max_iter", [0, 300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("bw", [0.005, 0.007, 0.009])
def test_modes_bruteforce_equals_modes(bw, dtype, max_iter):
    X = shifted_pile(1500, 8, seed=1, pull=0.0).astype(dtype)
    c, n, _ = meanshift_ref.ascent(X, bw, max_iter=max_iter)
    got = meanshift_ref.modes_bruteforce(c, n, bw)
    assert got.dtype == X.dtype and got.tobytes() == meanshift_ref.modes(c, n, bw).tobytes()


def test_modes_bruteforce_dict_rule():
    """Equal centres (+0.0 and -0.0 among them) collapse to the first seed's value with the last seed's count."""
    c = np.array([[-0.0, 1.0, 2.0], [5.0, 5.0, 5.0], [0.0, 1.0, 2.0], [9.0, 9.0, 9.0]])
    assert meanshift_ref.modes_bruteforce(c, [1, 2, 3, 0], 0.5).tobytes() == np.array(
        [[-0.0, 1.0, 2.0], [5.0, 5.0, 5.0]]).tobytes()
    assert meanshift_ref.modes_bruteforce(c, [3, 2, 1, 0], 0.5).tobytes() == np.array(
        [[5.0, 5.0, 5.0], [-0.0, 1.0, 2.0]]).tobytes()


X_OK = np.zeros((4, 3), np.float32) + np.arange(4, dtype=np.float32)[:, None] * 0.01


@pytest.mark.parametrize("kw, exc", [
    ({"bandwidth": None}, NotImplementedError),
    ({"bandwidth": 0.007, "seeds": X_OK}, NotImplementedError),
    ({"bandwidth": 0.007, "bin_seeding": True}, NotImplementedError),
    ({"bandwidth": 0.007, "cluster_all": False}, NotImplementedError),
    ({"bandwidth": 0.0}, ValueError),
    ({"bandwidth": -1.0}, ValueError),
    ({"bandwidth": float("nan")}, ValueError),
    ({"bandwidth": 0.007, "max_iter": -1}, ValueError),
    ({"bandwidth": 0.007, "max_iter": 1.5}, ValueError),
])
def test_unsupported_or_bad_arguments_raise_before_the_device(kw, exc):
    with pytest.raises(exc):
        segment.MeanShift(**kw).fit(X_OK)


@pytest.mark.parametrize("X", [np.zeros((0, 3)), np.zeros((5, 2)), np.zeros(6), np.zeros((2, 3, 1)),
                               np.array([[0.0, 0.0, np.nan]]), np.array([[np.inf, 0.0, 0.0]])],
                         ids=["empty", "two-columns", "flat", "3d", "nan", "inf"])
def test_bad_points_raise_value_error(X):
    with pytest.raises(ValueError):
        segment.MeanShift(bandwidth=0.007).fit(X)
    with pytest.raises(ValueError):
        segment.pointgroup_labels(X, X, X_OK, 0.007)


def test_n_jobs_is_accepted():
    assert segment.MeanShift(0.007, n_jobs=-1).n_jobs == -1
