"""cg_meanshift.cu (catgrasp_b200.segment) against oracle/meanshift_ref.py, bit for bit: per-seed centres, counts and
iterations, the kept centres, the labels and n_iter_; and pointgroup_labels against the reference's
PointGroupPredictor.predict (tests/golden/segment.npz).

Seeded mutations and the test that catches each:
  - membership `d2 < bw2` for `<=`                   test_dyadic_lattice_on_the_boundary (neighbours at d2 == bw^2)
  - FMA contraction in the ascent's distance        test_codegen.py::test_entry_contract (ascent_kernel's no_fma)
  - a float64 sum in place of the int64 sum         test_piles, test_numpy_and_tensor_input_agree (centres move)
  - suppression without the (count, x, y, z) order  test_chain_of_equal_count_modes (the greedy order decides)
  - centres collapsed by bit pattern, not value     test_signed_zeros_and_duplicates
  - label ties to the larger index                  test_dyadic_lattice_on_the_boundary (exactly tied centres)
  - max_iter off by one (it > max_iter)             test_max_iter_zero_and_one
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import segment, synthetic   # noqa: E402
from oracle import meanshift_ref               # noqa: E402


def _check(X, bw, max_iter=300):
    got = segment.MeanShift(bandwidth=bw, max_iter=max_iter).fit(X)
    ref = meanshift_ref.fit(X, bw, max_iter=max_iter)
    assert got.seed_centers_.dtype == X.dtype and got.cluster_centers_.dtype == X.dtype
    assert got.seed_centers_.tobytes() == ref["seed_centres"].tobytes()
    assert np.array_equal(got.seed_counts_, ref["seed_counts"])
    assert np.array_equal(got.seed_iters_, ref["seed_iters"])
    assert got.cluster_centers_.tobytes() == ref["centres"].tobytes()
    assert got.labels_.dtype == np.int64 and np.array_equal(got.labels_, ref["labels"])
    assert got.n_iter_ == ref["n_iter"]
    return got


def _pile(n, k, seed, pull, noise=0.0008):
    s = synthetic.make_pile(n, n_objects=k, seed=seed)
    centre = s["object_poses"][:, :3, 3][s["object_id"]]
    rng = np.random.RandomState(seed + 7)
    return s["cloud_xyz"] + pull * (centre - s["cloud_xyz"]) + rng.normal(0, noise, s["cloud_xyz"].shape)


@pytest.mark.parametrize("pull", [0.85, 0.3], ids=["tight", "loose"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("bw", [0.005, 0.007, 0.009])
def test_piles(bw, dtype, pull):
    _check(_pile(3000, 12, seed=5, pull=pull).astype(dtype), bw)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_dyadic_lattice_on_the_boundary(dtype):
    bw = 2.0 ** -7                                   # spacing == bw: axis neighbours at d2 == bw*bw exactly
    g = np.stack(np.meshgrid(np.arange(12), np.arange(10), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    X = (0.5 + g * bw).astype(dtype)
    got = _check(X, bw)
    assert got.seed_counts_.max() == 7


def test_chain_of_equal_count_modes():
    bw = 0.007
    x = np.arange(24) * 0.9 * bw
    X = np.repeat(np.stack([x, np.zeros_like(x), np.full_like(x, 0.7)], 1), 5, axis=0)
    _check(X, bw)
    _check(X[::-1].copy(), bw)


def test_signed_zeros_and_duplicates():
    bw = 0.007
    rng = np.random.RandomState(3)
    X = rng.normal(0, 0.002, (400, 3))
    X[::3, 0] = 0.0
    X[1::3, 0] = -0.0
    X[::5, 2] = -0.0
    X = np.concatenate([X, X[:150], X[:40]])          # exact duplicates
    _check(X, bw)
    _check(X.astype(np.float32), bw)


@pytest.mark.parametrize("X", [np.array([[0.1, -0.2, 0.7]]), np.full((1000, 3), 0.3125)],
                         ids=["single", "identical"])
def test_degenerate_clouds(X):
    got = _check(X, 0.005)
    assert len(got.cluster_centers_) == 1 and (got.labels_ == 0).all()


@pytest.mark.parametrize("max_iter", [0, 1])
def test_max_iter_zero_and_one(max_iter):
    got = _check(_pile(2000, 8, seed=6, pull=0.3).astype(np.float32), 0.007, max_iter=max_iter)
    assert got.n_iter_ == max_iter


def test_two_to_the_twenty_points():
    """2^17 separated groups of 8 points: 2^20 seeds, 2^17 modes."""
    bw = 0.005
    g = np.stack(np.meshgrid(np.arange(64), np.arange(64), np.arange(32), indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.RandomState(7)
    X = (np.repeat(g * 3 * bw, 8, axis=0) + rng.uniform(-0.3 * bw, 0.3 * bw, (len(g) * 8, 3))).astype(np.float32)
    X = X[rng.permutation(len(X))]
    assert len(X) == 1 << 20
    got = _check(X, bw)
    assert len(got.cluster_centers_) == len(g)


def test_numpy_and_tensor_input_agree():
    X = _pile(2500, 10, seed=8, pull=0.6).astype(np.float32)
    a = segment.MeanShift(bandwidth=0.007).fit(X)
    b = segment.MeanShift(bandwidth=0.007).fit(torch.from_numpy(X).cuda())
    assert isinstance(b.labels_, torch.Tensor) and b.labels_.is_cuda and b.cluster_centers_.dtype == torch.float32
    assert b.cluster_centers_.cpu().numpy().tobytes() == a.cluster_centers_.tobytes()
    assert np.array_equal(b.labels_.cpu().numpy(), a.labels_) and b.n_iter_ == a.n_iter_
    assert np.array_equal(segment.MeanShift(0.007).fit_predict(X), a.labels_)


def test_pointgroup_labels_reproduce_reference_predict(golden_dir):
    g = np.load(os.path.join(golden_dir, "segment.npz"))
    for cls, bw in segment.MEANSHIFT_BANDWIDTH.items():
        labels_all, shifted = segment.pointgroup_labels(g[f"{cls}_xyz_original_all"], g[f"{cls}_pt_offsets"],
                                                        g[f"{cls}_cloud_xyz"], bw)
        assert shifted.dtype == np.float32 and shifted.tobytes() == g[f"{cls}_xyz_shifted"].tobytes(), cls
        assert labels_all.dtype == np.int64 and np.array_equal(labels_all, g[f"{cls}_labels_all"]), cls


def test_too_many_points_is_refused():
    from catgrasp_b200 import _lib
    X = np.random.RandomState(0).uniform(0, 1, ((1 << 21) + 1, 3)).astype(np.float32)
    with pytest.raises(_lib.CgError, match="2\\^21"):
        segment.MeanShift(bandwidth=0.05).fit(X)
