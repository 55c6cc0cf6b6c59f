"""CPU tests of the PointNet++ oracle pieces that tests/test_pn2_kernels.py relies on.

1. The fp32 three_nn restatement (oracle/pn2_ref.py) reproduces the 3-NN indices and weights of the golden module run,
   which used the reference's own square_distance.
2. The float64 shared-MLP reference (SharedMLP64) computes the same stacks as the golden run (torch fp32, unfolded BN).
3. Its error bound is tight enough to catch localized kernel bugs: a group max that drops its last member, a skipped
   last 64-row tile, two swapped output channels, rows offset by one.
"""
import os

import numpy as np
import pytest

from oracle import pn2_ref
from oracle.encoder_ref import bound_ratio
from test_pn2_modules import _sd

T = lambda a: np.ascontiguousarray(np.swapaxes(a, 1, 2))   # noqa: E731  (B,C,N) <-> (B,N,C)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "pn2_modules.npz"))


def test_three_nn_reproduces_golden(golden):
    """Indices exact; weights exact too: torch sums the three reciprocals in index order, as the kernel does."""
    for dense, sparse, i, w in (("xyz", "l1_xyz", "idx1", "w1"), ("l1_xyz", "l2_xyz", "idx2", "w2")):
        idx, wt = pn2_ref.three_nn(T(golden[dense]), T(golden[sparse]))
        assert np.array_equal(idx, golden[i]), i
        assert np.array_equal(wt.view(np.uint32), golden[w].view(np.uint32)), w


def test_three_nn_two_neighbours_and_ties():
    """S = 2 keeps two neighbours normalised over two; equal distances go to the lower index."""
    dense = np.array([[[0, 0, 0], [1, 0, 0]]], np.float32)
    sparse = np.array([[[0.5, 0, 0], [-0.5, 0, 0]]], np.float32)
    idx, w = pn2_ref.three_nn(dense, sparse)
    assert idx.shape == (1, 2, 2) and (idx[0, 0] == [0, 1]).all() and (idx[0, 1] == [0, 1]).all()
    assert w[0, 0, 0] == w[0, 0, 1] == np.float32(0.5) and np.isclose(w[0, 1].sum(), 1.0)
    sparse4 = np.array([[[0, 0, 1], [0, 1, 0], [2, 0, 0], [1, 0, 0], [0, 0, -1]]], np.float32)
    idx, _ = pn2_ref.three_nn(dense[:, :1], sparse4)
    assert (idx[0, 0] == [0, 1, 3]).all()                 # four at distance 1: the three lowest indices


def _stages(g):
    """(name, SharedMLP64, input, is_group) for the six golden stages, each from the golden inputs of its layer."""
    stages = []
    mlp = lambda n: pn2_ref.SharedMLP64(*_sd(n))          # noqa: E731
    _, grouped, _, _ = pn2_ref.sample_and_group(256, 0.2, 32, T(g["xyz"]), T(g["nrm"]), g["start1"])
    stages.append(("l1_pts", mlp("sa1"), grouped, True))
    _, grouped, _, _ = pn2_ref.sample_and_group(64, 0.4, 16, T(g["l1_xyz"]), T(g["l1_pts"]), g["start2"])
    stages.append(("l2_pts", mlp("sa2"), grouped, True))
    stages.append(("l3_pts", mlp("sa3"), np.concatenate([T(g["l2_xyz"]), T(g["l2_pts"])], -1)[:, None], True))
    l3 = np.repeat(T(g["l3_pts"]), g["l2_xyz"].shape[2], axis=1)
    stages.append(("f2", mlp("fp3"), np.concatenate([T(g["l2_pts"]), l3], -1), False))
    idx, w = pn2_ref.three_nn(T(g["l1_xyz"]), T(g["l2_xyz"]))
    stages.append(("f1", mlp("fp2"), pn2_ref.three_interp(T(g["l1_pts"]), T(g["f2"]), idx, w), False))
    idx, w = pn2_ref.three_nn(T(g["xyz"]), T(g["l1_xyz"]))
    stages.append(("f0", mlp("fp1"), pn2_ref.three_interp(T(g["nrm"]), T(g["f1"]), idx, w), False))
    return stages


def _run(m, x, is_group, engine):
    if is_group:
        B, S, K, C = x.shape
        y, e = m.group_max(x.reshape(B * S, K, C), engine)
        return y.reshape(B, S, -1), e.reshape(B, S, -1)
    B, N, C = x.shape
    y, e = m.rows(x.reshape(B * N, C), engine)
    return y.reshape(B, N, -1), e.reshape(B, N, -1)


def test_float64_mlp_matches_golden_stacks(golden):
    """Every SA / FP stage of the golden run.  The golden is torch fp32 with BatchNorm unfolded: a conv rounding plus
    four BN roundings per layer on top of the accumulation, i.e. of the order of the fp32 bound itself, so it must
    lie within 4x the engine-0 bound, and within 1e-5 of the largest value."""
    for name, m, x, is_group in _stages(golden):
        y, e = _run(m, x, is_group, engine=0)
        want = T(golden[name]).astype(np.float64)
        d = np.abs(y - want)
        print(f"{name}: max |float64 - golden| {d.max():.3g}, max bound {e.max():.3g}, ratio {bound_ratio(want, y, e, 4).max():.3g}")
        assert d.max() <= 4 * e.max(), name
        assert bound_ratio(want, y, e, 4).max() <= 1, name
        assert d.max() < 1e-5 * max(1.0, np.abs(want).max()), name


@pytest.mark.parametrize("engine", [0, 1])
def test_bound_rejects_localized_mlp_bugs(engine):
    """G = 40 groups of K = 20 members (800 rows, the last 64-row tile is rows 768-799), stack 6 -> 64 -> 64 -> 128:
    each perturbed group max lies outside twice the bound of the unperturbed one."""
    m = pn2_ref.SharedMLP64(*_sd("sa1"))
    G, K = 40, 20
    x = np.random.RandomState(3).normal(0, 0.3, (G * K, 6)).astype(np.float32)
    y, e = m.rows(x, engine)
    out, eo = y.reshape(G, K, -1).max(1), e.reshape(G, K, -1).max(1)
    assert bound_ratio(out, out, eo).max() == 0

    def skip_last_tile(z):
        z = z.copy()
        z[(G * K - 1) // 64 * 64:] = 0.0                # rows never written: a zero-initialised buffer
        return z

    def swap(o):
        o = o.copy()
        o[:, [5, 6]] = o[:, [6, 5]]
        return o

    shift = np.minimum(np.arange(G * K) + 1, G * K - 1)
    perturbed = {"group max drops member K-1": y.reshape(G, K, -1)[:, :K - 1].max(1),
                 "last 64-row tile skipped": skip_last_tile(y).reshape(G, K, -1).max(1),
                 "output channels 5 and 6 swapped": swap(out),
                 "rows offset by one": y[shift].reshape(G, K, -1).max(1)}
    for name, got in perturbed.items():
        r = bound_ratio(got, out, eo)
        print(f"engine {engine} {name}: {int((r > 1).sum())} values past 2x the bound, max ratio {r.max():.3g}")
        assert r.max() > 1, (engine, name)


def test_fps_config_ranges():
    """The launch rule of cg_fps_dev at the range edges of its nine (cluster, points per thread) combinations."""
    edges = {2048: (2, 4), 2049: (2, 8), 4096: (2, 8), 4097: (2, 16), 5632: (2, 16), 5633: (4, 8), 8192: (4, 8),
             8193: (4, 16), 13312: (4, 16), 13313: (8, 8), 16384: (8, 8), 16385: (8, 16), 32768: (8, 16),
             32769: (8, 32), 65536: (8, 32), 65537: (16, 32), 131072: (16, 32)}
    for n, cfg in edges.items():
        assert pn2_ref.fps_config(n) == cfg, n
    assert pn2_ref.fps_config(1) == (2, 4) and pn2_ref.fps_config(131073) is None
    assert pn2_ref.fps_config(65537, max_cluster=8) is None
