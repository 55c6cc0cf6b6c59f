"""GPU (-m gpu): cg_ransac9d_host (csrc/cg_ransac.cu) hypothesis by hypothesis against oracle/ransac64.py.

Per hypothesis: the valid flag equals the oracle's wherever the oracle decides it; the kernel's count ratio * N lies
in the oracle's [lo, hi]; a valid T is within the oracle's bound of the high-precision T; an invalid hypothesis has
ratio 0 and an all-zero T (include/catgrasp_b200.h).  Undecided hypotheses are counted and capped at 1 %."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import ransac64
from test_ransac_ref import MAX_D, MAX_S, MIN_S, THR, golden_ransac_case, lattice_case, singular_subsets

pytestmark = pytest.mark.gpu
RATIOS = []        # kernel |T - T*| / bound over every valid hypothesis checked (printed by the last test)
UNDECIDED = [0, 0]  # undecided hypotheses, hypotheses checked


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def kernel(src, tgt, ids, thr=THR, min_s=MIN_S, max_s=MAX_S, max_dims=MAX_D):
    from catgrasp_b200 import _lib
    src = np.ascontiguousarray(src, np.float64)
    tgt = np.ascontiguousarray(tgt, np.float64)
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1, 4)
    H = len(ids)
    mins = np.ascontiguousarray(min_s, np.float64).reshape(3)
    maxs = np.ascontiguousarray(max_s, np.float64).reshape(3)
    mdim = None if max_dims is None else np.ascontiguousarray(max_dims, np.float64).reshape(3)
    ratio, T, valid = np.empty(H), np.empty((H, 4, 4)), np.empty(H, np.uint8)
    ctx = _lib.Context.get()
    ctx.use_own_stream()
    ctx.check(ctx.lib.cg_ransac9d_host(ctx.h, _lib.ptr(src), _lib.ptr(tgt), len(src), _lib.ptr(ids), H, C.c_double(thr),
                                       _lib.ptr(mins), _lib.ptr(maxs), _lib.ptr(mdim), _lib.ptr(ratio), _lib.ptr(T),
                                       _lib.ptr(valid)))
    return ratio, T, valid


def check(src, tgt, ids, thr=THR, min_s=MIN_S, max_s=MAX_S, max_dims=MAX_D, res=None, cap=0.01):
    """kernel vs oracle on every hypothesis; returns (oracle results, kernel ratio, kernel valid)."""
    ratio, T, valid = kernel(src, tgt, ids, thr, min_s, max_s, max_dims)
    if res is None:
        res = ransac64.evaluate(src, tgt, ids, thr, min_s, max_s, max_dims)
    N = len(src)
    und = 0
    for h, r in enumerate(res):
        if not valid[h]:
            assert ratio[h] == 0.0 and not T[h].any(), h
        if r["valid"] is None or r["info"]["lu_may_differ"]:
            und += 1
            continue
        assert bool(valid[h]) == r["valid"], (h, r["gates"], r["info"])
        if r["valid"]:
            err = np.abs(T[h] - r["T"]).max()
            assert err <= r["bound"], (h, err, r["bound"])
            RATIOS.append(err / r["bound"])
            np.testing.assert_array_equal(T[h][3], [0, 0, 0, 1])
            cnt = ratio[h] * N
            assert cnt == np.rint(cnt) and r["lo"] <= cnt <= r["hi"], (h, cnt, r["lo"], r["hi"])
    assert und <= cap * len(res), und
    UNDECIDED[0] += und
    UNDECIDED[1] += len(res)
    return res, ratio, valid


def test_golden_draws(cuda, golden_dir):
    g, ids = golden_ransac_case(golden_dir)
    res, ratio, valid = check(g["source"], g["target"], ids)
    w = ransac64.replay_winner(res)
    keep = np.nonzero(valid)[0]
    assert keep[np.argmax(ratio[keep])] == w                # the host's first-maximum rule picks the oracle's winner
    res, _, _ = check(g["source"], g["target"], ids[:500], max_dims=None)


def test_lattice_draws(cuda, golden_dir):
    g, src, tgt, ids = lattice_case(golden_dir, 2000)
    check(src, tgt, ids)


def test_singular_subsets(cuda, golden_dir):
    """Repeated NOCS points (three inliers + a duplicate of one), coplanar z = 0 and collinear subsets: cv2's
    minimum-norm affine.  The lattice's duplicate subsets include hypotheses that pass every gate."""
    g, src, tgt, _ = lattice_case(golden_dir, 0)
    T = g["call_transforms"][0]
    err = np.linalg.norm(np.c_[src, np.ones(len(src))] @ T[:3].T - tgt, axis=1)
    ids = singular_subsets(src, np.random.RandomState(5), np.nonzero(err <= THR)[0], 400)
    res, ratio, valid = check(src, tgt, ids)
    assert all(r["info"]["singular"] for r in res) and valid.sum() >= 1
    truth = np.load(os.path.join(golden_dir, "host_ransac9d.npz"))["truth"]
    rng = np.random.RandomState(6)
    q = rng.uniform(-0.5, 0.5, (80, 3))
    q[:40, 2] = 0.0
    q[40:] = q[40:, :1].astype(np.float32).astype(np.float64) * [1.0, 0.5, -0.25]
    d = np.c_[q, np.ones(80)] @ truth[:3].T + rng.normal(0, 1e-4, q.shape)
    for mdims in (MAX_D, None):
        check(q, d, np.arange(80).reshape(20, 4), max_dims=mdims, cap=0.1)


def _exact_case(N, rng, inlier_frac=0.7):
    """N correspondences through a known affine-similarity with noise and outliers, the first 4 points exact."""
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    R *= np.sign(np.linalg.det(R))
    T = np.eye(4)
    T[:3, :3] = R @ np.diag([0.02, 0.025, 0.01])
    T[:3, 3] = [0.05, -0.02, 0.7]
    src = rng.uniform(-0.5, 0.5, (N, 3))
    tgt = np.c_[src, np.ones(N)] @ T[:3].T + rng.normal(0, 0.001, (N, 3))
    bad = rng.rand(N) > inlier_frac
    tgt[bad] += rng.normal(0, 0.05, (bad.sum(), 3))
    return src, tgt


@pytest.mark.parametrize("N", [4, 127, 128, 129, 4097, 2 ** 20 + 3])
def test_point_counts(cuda, N):
    """The 128-thread stride, the warp reductions and the four-warp combine, with and without max_dims."""
    rng = np.random.RandomState(N)
    src, tgt = _exact_case(N, rng)
    H = 40 if N < 2 ** 20 else 6
    ids = np.array([rng.choice(N, 4, replace=False) for _ in range(H)], np.int32)
    ids[0] = [N - 1, N - 2, N - 3, N - 4]
    for mdims in (MAX_D, None):
        check(src, tgt, ids, max_dims=mdims, cap=0.05 if H < 100 else 0.01)


def _gate_points():
    """4 points through an exactly representable similarity (unit vectors -> columns): the solve is exact, so every
    gate quantity is known in closed form; 1000 more points around it for the residual and extent passes."""
    A = np.array([[0.015625, -0.0078125, 0.0], [0.0078125, 0.015625, 0.0], [0.0, 0.0, 0.0078125]])
    t = np.array([0.125, -0.25, 0.5])
    s4 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    rng = np.random.RandomState(3)
    q = rng.uniform(-0.5, 0.5, (1000, 3))
    src = np.r_[s4, q]
    tgt = src @ A.T + t
    return A, t, src, tgt


def test_gates_at_their_edges(cuda):
    """Scale gates at (1 -+ 1e-9) of the exact quantity, dimensions and the threshold at (1 -+ 1e-7), a mirrored target."""
    A, t, src, tgt = _gate_points()
    ids = np.array([[0, 1, 2, 3]], np.int32)
    sc = np.linalg.norm(A, axis=0)
    for j in range(3):
        for side, f, expect in (("min", 1 - 1e-9, 1), ("min", 1 + 1e-9, 0), ("max", 1 + 1e-9, 1), ("max", 1 - 1e-9, 0)):
            mins, maxs = np.array(MIN_S, float), np.array(MAX_S, float)
            (mins if side == "min" else maxs)[j] = sc[j] * f
            res, ratio, valid = check(src, tgt, ids, min_s=mins, max_s=maxs, max_dims=None, cap=0)
            assert valid[0] == expect and res[0]["valid"] == bool(expect)
    Ti = np.linalg.inv(np.r_[np.c_[A, t], [[0, 0, 0, 1]]])
    c = tgt @ Ti[:3, :3].T + Ti[:3, 3]
    ext = c.max(0) - c.min(0)
    for j in range(3):
        for f, expect in ((1 + 1e-7, 1), (1 - 1e-7, 0)):     # the extent's bound (through 1 / scale^2) is ~1e-8
            md = np.full(3, 10.0)
            md[j] = ext[j] * f
            _, _, valid = check(src, tgt, ids, max_dims=md, cap=0)
            assert valid[0] == expect
    # residuals: points at thr (1 -+ 1e-7) off the model (the count's slack, from the T bound, is ~1e-8 thr here),
    # and points exactly on it (residual 0)
    rng = np.random.RandomState(4)
    u = rng.normal(size=(200, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    k = np.arange(200)
    off = np.where(k % 2 == 0, 1 - 1e-7, 1 + 1e-7)[:, None] * THR * u
    tg = tgt.copy()
    tg[4:204] += off
    res, ratio, valid = check(src, tg, ids, max_dims=None, cap=0)
    assert valid[0] and res[0]["lo"] == res[0]["hi"] == len(src) - 100 and ratio[0] * len(src) == len(src) - 100
    _, ratio, _ = check(src, tgt, ids, max_dims=None, cap=0)
    assert ratio[0] == 1.0                                   # all points inliers
    far = tgt.copy()
    far[4:] += 1.0
    _, ratio, valid = check(src, far, ids, max_dims=None, cap=0)
    assert valid[0] and ratio[0] == 4 / len(src)             # only the 4 sample points
    _, ratio, valid = check(src, tgt, ids, thr=-1.0, max_dims=None, cap=0)
    assert valid[0] and ratio[0] == 0.0                       # a valid hypothesis with no inliers
    mirrored = tgt * [1, 1, -1]
    res, ratio, valid = check(src, mirrored, ids, max_dims=None, cap=0)
    assert valid[0] == 0 and res[0]["gates"]["det"][0] < -0.5


def test_residual_exactly_at_threshold(cuda):
    """A diagonal dyadic affine (the polar step is exact: R = I, Jacobi does nothing, T = A bit for bit), dyadic
    points and a dyadic threshold: 100 points sit at a residual of exactly thr (|T s - tgt| = thr along x, computed
    exactly), 100 at thr + 2^-30.  The kernel's `<=` counts the first 100 and not the second."""
    A = np.diag([1 / 64, 1 / 32, 1 / 128])
    t = np.array([0.125, -0.25, 0.5])
    thr = 1 / 64
    rng = np.random.RandomState(8)
    src = np.r_[[[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], rng.randint(-32, 33, (1000, 3)) / 64.0]
    tgt = src @ A.T + t
    tgt[4:104, 0] += thr
    tgt[104:204, 0] += thr + 2.0 ** -30
    ratio, T, valid = kernel(src, tgt, [[0, 1, 2, 3]], thr=thr, max_dims=None)
    assert valid[0] and np.array_equal(T[0][:3, :3], A) and np.array_equal(T[0][:3, 3], t)
    assert ratio[0] * len(src) == len(src) - 100


def _sv_edge_affine(edge, side):
    """Columns of a float32 affine whose R = A / scales has its smallest (edge 0.8) or largest (edge 1.2) singular
    value at edge * (1 + side * [2e-10, 2e-9]): R^T R = (1 - c) I + c 11^T (eigenvalues 1 + 2c, 1 - c, 1 - c), then
    two entries are nudged by float32 ulps until the singular value lands in the window."""
    c = -0.18 if edge == 0.8 else 0.22
    G = (1 - c) * np.eye(3) + c * np.ones((3, 3))
    A0 = (0.02 * np.linalg.cholesky(G).T).astype(np.float32)
    k = np.arange(-60, 61)
    k1, k2 = np.meshgrid(k, k, indexing="ij")
    B = np.repeat(A0.astype(np.float64)[None], k1.size, 0)
    B[:, 0, 1] = (A0[0, 1] + k1.ravel() * np.spacing(A0[0, 1])).astype(np.float32)
    B[:, 1, 2] = (A0[1, 2] + k2.ravel() * np.spacing(A0[1, 2])).astype(np.float32)
    sv = np.linalg.svd(B / np.linalg.norm(B, axis=1, keepdims=True), compute_uv=False)
    v = sv[:, -1] if edge == 0.8 else sv[:, 0]
    rel = side * (v / edge - 1)
    i = np.nonzero((rel > 2e-10) & (rel < 2e-9))[0]
    assert i.size
    return B[i[np.argmin(rel[i])]]


@pytest.mark.parametrize("edge", [0.8, 1.2])
def test_singular_value_gate_at_its_edges(cuda, edge):
    """Sheared affines with a singular value of R at 0.8 / 1.2 (1 -+ 2e-9): inside passes, outside fails."""
    s4 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    for side in (1, -1):
        A = _sv_edge_affine(edge, side if edge == 0.8 else -side)
        tgt = s4 @ A.T                                      # float32 values: the narrowing is exact
        res, ratio, valid = check(s4, tgt, [[0, 1, 2, 3]], max_dims=None, cap=0)
        margin = res[0]["gates"]["sv_min" if edge == 0.8 else "sv_max"][0]
        assert 0 < side * margin < 3e-9 and valid[0] == (side > 0)


def test_hypothesis_counts(cuda, golden_dir):
    """H = 1 and H = 70 000 (the same 35 subsets repeated, each copy scored alike)."""
    g, ids = golden_ransac_case(golden_dir)
    check(g["source"], g["target"], ids[:1], cap=1)
    base = ids[:35]
    res = ransac64.evaluate(g["source"], g["target"], base, THR, MIN_S, MAX_S, MAX_D)
    rep = np.tile(base, (2000, 1))
    ratio, T, valid = kernel(g["source"], g["target"], rep)
    check(g["source"], g["target"], base, res=res)
    r0, T0, v0 = kernel(g["source"], g["target"], base)
    assert np.array_equal(valid.reshape(2000, 35), np.tile(v0, (2000, 1)))
    assert np.array_equal(ratio.reshape(2000, 35), np.tile(r0, (2000, 1)))
    assert np.array_equal(T.reshape(2000, 35, 4, 4), np.tile(T0, (2000, 1, 1, 1)))


def test_host_selection_rule(cuda, golden_dir):
    """The first maximum among valid hypotheses: tied maximal ratios (the lattice golden, ratio exactly 1.0; then the
    same draws rotated so that the first holder is not at index 0) and the seeded draws of the reference run."""
    from catgrasp_b200.aligning import estimate9DTransform
    gl, src, tgt, ids = lattice_case(golden_dir, 10000)
    res = ransac64.evaluate(src, tgt, ids, THR, MIN_S, MAX_S, MAX_D, stop_at_full=True)
    w = ransac64.replay_winner(res)
    ratio, T, valid = kernel(src, tgt, ids[:len(res)])
    assert ratio[w] == 1.0 and not (ratio[:w][valid[:w] == 1] == 1.0).any()
    # the same draws rotated so that the first full holder is not at index 0: later full holders tie with it
    tail = ids[w + 1:w + 400]
    rt = ransac64.evaluate(src, tgt, tail, THR, MIN_S, MAX_S, MAX_D)
    lower = [h for h, r in enumerate(rt) if r["valid"] is False or (r["valid"] and r["hi"] < len(src))]
    rot = np.r_[tail[lower[:10]], tail]
    res = ransac64.evaluate(src, tgt, rot, THR, MIN_S, MAX_S, MAX_D)
    w2 = ransac64.replay_winner(res)
    ratio, T, valid = kernel(src, tgt, rot)
    keep = np.nonzero(valid)[0]
    assert w2 > 0 and ratio[w2] == 1.0 and keep[np.argmax(ratio[keep])] == w2
    # the seeded draws of the reference run give the oracle-replayed winner
    g, ids3 = golden_ransac_case(golden_dir)
    np.random.seed(3)
    tf, inl = estimate9DTransform(source=g["source"], target=g["target"], PassThreshold=THR, max_iter=3000,
                                  max_scale=MAX_S, min_scale=MIN_S, max_dimensions=MAX_D)
    res3 = ransac64.evaluate(g["source"], g["target"], ids3, THR, MIN_S, MAX_S, MAX_D)
    np.testing.assert_allclose(tf, res3[ransac64.replay_winner(res3)]["T"], rtol=0, atol=1e-9)


def test_host_selection_skips_invalid_higher_raw_ratio(cuda, monkeypatch):
    """aligning.estimate9DTransform with chosen subsets (np.random.choice replaced by a list): hypothesis 0 is a
    mirrored fit (det < 0) whose raw inlier count, 1007, beats the true fit's 1004; hypotheses 1 and 2 are the true
    fit, tied.  The host must return hypothesis 1's transform and its inliers."""
    from catgrasp_b200.aligning import estimate9DTransform
    A, t, _, _ = _gate_points()
    rng = np.random.RandomState(12)
    q = np.c_[rng.randint(-32, 33, (1000, 2)) / 64.0, np.zeros(1000)]          # z = 0: fits the mirror as well
    e = np.array([[0.25, 0.25, 0.5], [-0.25, 0.25, 0.5], [0.25, -0.25, 0.5], [0.25, 0.25, -0.5]])
    s4 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    src = np.r_[s4, q, e]
    tgt = np.r_[s4 @ A.T + t, q @ A.T + t, e @ (A @ np.diag([1.0, 1.0, -1.0])).T + t]
    draws = [np.arange(1004, 1008), np.arange(4), np.arange(4)]
    ratio, T, valid = kernel(src, tgt, draws, max_dims=None)
    assert list(valid) == [0, 1, 1] and ratio[0] == 0.0 and ratio[1] == ratio[2] == 1004 / 1008
    Am = np.c_[A @ np.diag([1.0, 1.0, -1.0]), t]
    assert np.count_nonzero(np.linalg.norm(np.c_[src, np.ones(1008)] @ Am.T - tgt, axis=1) <= THR) == 1007
    it = iter(draws)
    monkeypatch.setattr(np.random, "choice", lambda *a, **k: next(it))
    tf, inl = estimate9DTransform(source=src, target=tgt, PassThreshold=THR, max_iter=3, max_scale=MAX_S,
                                  min_scale=MIN_S, max_dimensions=None)
    assert np.array_equal(tf, T[1]) and np.array_equal(inl, np.arange(1004))


def test_report_error_over_bound(cuda):
    """Runs last: the largest kernel |T - T*| / bound over every valid hypothesis checked above."""
    assert RATIOS and max(RATIOS) <= 1.0
    print(f"ransac9d: {len(RATIOS)} valid hypotheses, max |T - T*| / bound = {max(RATIOS):.3e}; "
          f"{UNDECIDED[0]} of {UNDECIDED[1]} hypotheses undecided")
