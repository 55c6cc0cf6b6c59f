"""Several point sets in one cloud index (cg_cloud_index_create_many), one nearest-point pass over them
(cg_cloud_nearest_many_dev), mean shift per set in one pass (cg_meanshift_many_dev), and the batched front and
clustering of PointGroupPredictor.predict_many, each held bit for bit to the one-set calls.

  - tables: set s's sorted points, perm minus its first point, cell keys without the set field and cell starts minus
    its first point equal the one-set index over set s alone, and so do its voxel means; for sets of very different
    sizes, a one-point set, identical sets, sets overlapping in space, sets in the top cell of a 2^b-wide field next to
    the following set, and the largest batch whose keys fit in 63 bits (one more set is refused);
  - nearest_many: ties to the smaller index, misses that stay -1 while another set has a point in range, and answers
    never taken from a neighbouring set;
  - mean shift: seeds, counts, iterations, centres, labels and n_iter_ per set, float32 and float64;
  - predictor: device_front_many, pointgroup_labels_many and predict_many against their per-frame calls, and the
    number of index builds predict_many makes does not grow with the number of frames.
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from catgrasp_b200 import _lib, cloud, segment, synthetic   # noqa: E402
from catgrasp_b200.predicter import PointGroupPredictor      # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
SEG = np.load(os.path.join(GOLDEN, "segment.npz"))


def _bit_length(v):
    return int(v).bit_length()


def _one_set_bits(p, cell):
    """The per-axis key width a one-set index over p uses (cg_cloud.cu's host arithmetic, in float64)."""
    o = p.min(0) - cell * 0.5
    top = np.floor((p.max(0) - o) / cell).astype(np.int64).max()
    return max(1, _bit_length(top))


def _tables(ix):
    dev = torch.device("cuda", ix.device)
    P, U = ix.n_points, ix.n_cells
    pts = torch.empty((P, 3), dtype=torch.float64, device=dev)
    perm = torch.empty((P,), dtype=torch.int32, device=dev)
    keys = torch.empty((U,), dtype=torch.int64, device=dev)
    start = torch.empty((U + 1,), dtype=torch.int32, device=dev)
    ix.ctx.call("cg_cloud_index_tables_dev", ix.h, pts, perm, keys, start)
    return pts.cpu().numpy(), perm.cpu().numpy(), keys.cpu().numpy().view(np.uint64), start.cpu().numpy()


def _unpack(keys, b):
    m = np.uint64((1 << b) - 1)
    return np.stack([(keys >> np.uint64(2 * b)) & m, (keys >> np.uint64(b)) & m, keys & m], 1)


def check_index(sets, cell):
    """The many-set index over `sets` (float64 arrays) against one one-set index per set."""
    pts = np.concatenate(sets)
    off = np.cumsum([0] + [len(s) for s in sets])
    ix = cloud.CloudIndex(pts, cell, set_offsets=off)
    assert ix.n_sets == len(sets) and np.array_equal(ix.set_offsets, off)
    spts, perm, keys, start = _tables(ix)
    b = max(_one_set_bits(s, cell) for s in sets)
    S = len(sets)
    assert _bit_length(S - 1) + 3 * b <= 63
    means, _ = ix.voxel_means()
    means = means.cpu().numpy()
    coff = ix.cell_offsets
    assert coff[0] == 0 and coff[-1] == ix.n_cells
    for s, p in enumerate(sets):
        one = cloud.CloudIndex(p, cell)
        o_pts, o_perm, o_keys, o_start = _tables(one)
        a, e, c, d = off[s], off[s + 1], coff[s], coff[s + 1]
        assert d - c == one.n_cells, s
        assert spts[a:e].tobytes() == o_pts.tobytes(), s
        assert np.array_equal(perm[a:e] - a, o_perm), s
        assert ((keys[c:d] >> np.uint64(3 * b)) == np.uint64(s)).all(), s
        lo = keys[c:d] & np.uint64((1 << (3 * b)) - 1)
        assert np.array_equal(_unpack(lo, b), _unpack(o_keys, _one_set_bits(p, cell))), s
        assert np.array_equal(start[c:d + 1] - a, o_start), s
        assert means[c:d].tobytes() == one.voxel_means()[0].cpu().numpy().tobytes(), s
    return ix


def _blob(n, seed, centre=(0.1, -0.05, 0.6), spread=0.04):
    return np.random.RandomState(seed).normal(centre, spread, (n, 3))


def _top_cell_sets(b, cell):
    """Set 0 fills the top cell of a 2^b-wide field on every axis; set 1 sits at set 0's origin, so a key of set 0 that
    carried past 2^b - 1 would land among set 1's cells."""
    top = (2 ** b - 1) * cell
    s0 = np.array([[0.0, 0.0, 0.0], [top, top, top], [top, 0.0, top], [0.0, top, top], [top, top, 0.0]])
    s1 = np.array([[0.0, 0.0, 0.0], [cell * 0.25, 0.0, 0.0], [top, top, top]])
    return [s0, s1, s0 + 0.5 * cell]


CASES = {
    "sizes": ([_blob(20000, 1), _blob(3, 2), _blob(700, 3, spread=0.01)], 0.002),
    "one_point": ([np.array([[0.3, 0.2, 0.5]]), _blob(500, 4), np.array([[-1.0, 2.0, 3.0]])], 0.0005),
    "identical": ([_blob(900, 5)] * 3, 0.003),
    "overlap": ([_blob(3000, 6), _blob(3000, 7), _blob(2000, 8, centre=(0.12, -0.04, 0.61))], 0.0005),
    "top_cell": (_top_cell_sets(5, 0.25), 0.25),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_tables_equal_the_sets(name):
    sets, cell = CASES[name]
    check_index(sets, cell)


def test_one_set_is_the_one_set_index():
    p = _blob(5000, 9)
    ix = cloud.CloudIndex(p, 0.001, set_offsets=[0, len(p)])
    one = cloud.CloudIndex(p, 0.001)
    for a, b in zip(_tables(ix), _tables(one)):
        assert a.tobytes() == b.tobytes()
    assert np.array_equal(ix.cell_offsets, [0, one.n_cells])


def test_largest_batch_that_fits_and_one_more():
    """b = 20 (a set spans 600001 cells): 3 * 20 + 3 set bits = 63 holds 8 sets; a ninth needs a fourth set bit."""
    cell = 1.0
    sets = [np.array([[0.0, 0.0, 0.0], [600000.0, 3.0 * s, 1.0]]) + 7.0 * s for s in range(8)]
    check_index(sets, cell)
    ix = cloud.CloudIndex(np.concatenate(sets), cell, set_offsets=np.arange(0, 17, 2))
    ctx = ix.ctx
    pts = np.concatenate(sets + [sets[0]])
    torch.cuda.synchronize()
    ctx.reset_launch_count()
    with pytest.raises(_lib.CgError, match="63"):
        cloud.CloudIndex(pts, cell, set_offsets=np.arange(0, 19, 2))
    assert ctx.launch_count() == 2          # the bounds pass alone: no key, sort or table launch, no allocation


def test_refusals():
    p = _blob(10, 10)
    with pytest.raises(ValueError, match="at least one point"):
        cloud.CloudIndex(p, 0.01, set_offsets=[0, 4, 4, 10])
    with pytest.raises(ValueError):
        cloud.CloudIndex(p, 0.01, set_offsets=[0, 4, 9])
    ix = cloud.CloudIndex(p, 0.01, set_offsets=[0, 4, 10])
    with pytest.raises(_lib.CgError, match="several sets"):
        ix.nearest(p, 0.1)
    with pytest.raises(_lib.CgError, match="several sets"):
        ix.within(p, 0.1, False)
    with pytest.raises(_lib.CgError, match="several sets"):
        ix.normals(0.01, 10)
    with pytest.raises(ValueError):
        ix.nearest_many(p, [0, 10], 0.1)


def _nearest_ref(ref, q, max_dist):
    """scipy-free brute force: float64 (dx*dx + dy*dy) + dz*dz, ties to the smaller index."""
    d = ref[None, :, :] - q[:, None, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    i = np.argmin(d2, 1)                     # first minimum: the smaller index on a tie
    dist = np.sqrt(d2[np.arange(len(q)), i])
    ok = dist <= max_dist
    return np.where(ok, i, -1), np.where(ok, dist, np.inf)


def check_nearest_many(sets, queries, cell, max_dist):
    off = np.cumsum([0] + [len(s) for s in sets])
    qoff = np.cumsum([0] + [len(q) for q in queries])
    ix = cloud.CloudIndex(np.concatenate(sets), cell, set_offsets=off)
    dist, idx = ix.nearest_many(np.concatenate(queries), qoff, max_dist)
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    for s, (p, q) in enumerate(zip(sets, queries)):
        if len(q) == 0:
            continue
        a, b = qoff[s], qoff[s + 1]
        d1, i1 = cloud.CloudIndex(p, cell).nearest(q, max_dist)
        i1 = i1.cpu().numpy()
        want = np.where(i1 < 0, -1, i1 + off[s])
        assert np.array_equal(idx[a:b], want), s
        assert dist[a:b].tobytes() == d1.cpu().numpy().tobytes(), s
        ri, rd = _nearest_ref(p, q, max_dist)
        assert np.array_equal(i1, ri) and np.array_equal(d1.cpu().numpy(), rd), s
        hit = idx[a:b] >= 0
        assert ((idx[a:b][hit] >= off[s]) & (idx[a:b][hit] < off[s + 1])).all(), s
    return idx


def test_nearest_many_ties_to_the_smaller_index():
    g = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(-1, 3) * 0.001
    sets = [g, np.concatenate([g, g]), g[::-1].copy()]
    q = g + 0.0005                                           # equidistant from 8 lattice points
    check_nearest_many(sets, [q, q, q], 0.001, 0.002)


def test_nearest_many_misses_stay_misses():
    far = np.array([[1.0, 1.0, 1.0]])
    near = _blob(300, 11, centre=(0.0, 0.0, 0.5), spread=0.01)
    q = near[:40] + 0.0001
    # set 0 is far from its queries; set 1 holds points right on them: set 0's answers must stay -1
    idx = check_nearest_many([far, near, far + 0.5], [q, q, np.zeros((0, 3))], 0.001, 0.005)
    assert (idx[:40] == -1).all() and (idx[40:] >= 1).all()


def test_nearest_many_never_crosses_into_the_next_set():
    sets = _top_cell_sets(4, 0.5)
    top = (2 ** 4 - 1) * 0.5
    q0 = np.array([[top, top, top + 0.3], [top + 0.2, top, top], [0.1, 0.1, 0.1]])
    check_nearest_many(sets, [q0, q0, q0], 0.5, 2.0)
    check_nearest_many(sets, [q0, q0, q0], 0.5, 1e3)


# --------------------------------------------------------------------------------------------------------- mean shift


def _pile(n, k, seed, pull, noise=0.0008):
    s = synthetic.make_pile(n, n_objects=k, seed=seed)
    centre = s["object_poses"][:, :3, 3][s["object_id"]]
    rng = np.random.RandomState(seed + 7)
    return s["cloud_xyz"] + pull * (centre - s["cloud_xyz"]) + rng.normal(0, noise, s["cloud_xyz"].shape)


def _lattice(dtype):
    bw = 2.0 ** -7
    g = np.stack(np.meshgrid(np.arange(12), np.arange(10), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    return (0.5 + g * bw).astype(dtype)


def _chain(dtype):
    x = np.arange(24) * 0.9 * 0.007
    return np.repeat(np.stack([x, np.zeros_like(x), np.full_like(x, 0.7)], 1), 5, axis=0).astype(dtype)


def check_meanshift_many(Xs, bw, max_iter=300):
    got = segment.MeanShift(bandwidth=bw, max_iter=max_iter).fit_many(Xs)
    assert len(got) == len(Xs)
    for s, (X, g) in enumerate(zip(Xs, got)):
        w = segment.MeanShift(bandwidth=bw, max_iter=max_iter).fit(X)
        for a in ("seed_centers_", "seed_counts_", "seed_iters_", "cluster_centers_", "labels_"):
            x, y = getattr(g, a), getattr(w, a)
            if isinstance(x, torch.Tensor):
                x, y = x.cpu().numpy(), y.cpu().numpy()
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (s, a)
        assert g.n_iter_ == w.n_iter_, s
    return got


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_meanshift_many_piles(dtype):
    Xs = [_pile(3000, 12, seed=5, pull=0.85), _pile(1500, 6, seed=6, pull=0.3), _pile(200, 2, seed=7, pull=0.6),
          _pile(3000, 12, seed=5, pull=0.85)]
    for bw in (0.005, 0.009):
        check_meanshift_many([X.astype(dtype) for X in Xs], bw)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_meanshift_many_lattice_and_chain(dtype):
    """The dyadic lattice (neighbours at d2 == bw*bw exactly) and the chain of equal-count modes in one batch, with a
    one-point set and the chain reversed."""
    check_meanshift_many([_lattice(dtype), _chain(dtype)[::-1].copy(), np.array([[0.1, 0.2, 0.3]], dtype),
                          _chain(dtype)], 2.0 ** -7)
    check_meanshift_many([_chain(dtype), _lattice(dtype), _chain(dtype)[::-1].copy()], 0.007)


@pytest.mark.parametrize("max_iter", [0, 1])
def test_meanshift_many_max_iter_zero_and_one(max_iter):
    Xs = [_pile(2000, 8, seed=6, pull=0.3).astype(np.float32), _pile(900, 4, seed=9, pull=0.5).astype(np.float32)]
    got = check_meanshift_many(Xs, 0.007, max_iter=max_iter)
    assert all(g.n_iter_ == max_iter for g in got)


def test_meanshift_many_cuda_input():
    Xs = [torch.from_numpy(_pile(1200, 5, seed=s, pull=0.6).astype(np.float32)).cuda() for s in (11, 12)]
    got = check_meanshift_many(Xs, 0.007)
    assert got[0].labels_.is_cuda and got[0].cluster_centers_.dtype == torch.float32


def test_meanshift_many_two_to_the_twenty_one_points_per_set():
    """One set at the 2^21-point limit next to small ones; a set one point over it is refused."""
    bw = 0.005
    g = np.stack(np.meshgrid(np.arange(64), np.arange(64), np.arange(64), indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.RandomState(7)
    big = (np.repeat(g * 3 * bw, 8, axis=0) + rng.uniform(-0.3 * bw, 0.3 * bw, (len(g) * 8, 3))).astype(np.float32)
    assert len(big) == 1 << 21
    small = [_pile(500, 3, seed=3, pull=0.7).astype(np.float32), _pile(80, 1, seed=4, pull=0.7).astype(np.float32)]
    check_meanshift_many([small[0], big, small[1]], bw)
    over = np.concatenate([big, big[:1]])
    with pytest.raises(_lib.CgError, match="2\\^21"):
        segment.MeanShift(bandwidth=bw).fit_many([small[0], over])


# ---------------------------------------------------------------------------------------------------------- predictor


@pytest.fixture(scope="module")
def predictor(tmp_path_factory):
    import json
    import yaml
    from oracle import pointgroup_ref as PR
    G = np.load(os.path.join(GOLDEN, "pointgroup.npz"))
    key_shapes = [(k, tuple(s)) for k, s in json.loads(str(G["key_shapes"]))]
    d = tmp_path_factory.mktemp("artifacts-pg-front-many")
    cfg = {"downsample_size": 0.0005,
           "GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": int(G["m"]), "block_residual": True, "block_reps": int(G["block_reps"]),
                         "use_coords": True},
           "GROUP": {"prepare_epochs": 999999}}
    (d / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    sd = PR.synthetic_state_dict(key_shapes, int(G["seed"]))
    torch.save({"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}}, str(d / "best_val.pth.tar"))
    return PointGroupPredictor("nut", artifact_dir=str(d), device=0)


def _frames(n):
    out = []
    seg = SEG["nut_cloud_xyz"].copy()
    out.append({"cloud_xyz": seg, "cloud_normal": np.tile(np.float32([0, 0, -1]), (len(seg), 1))})
    for i in range(n - 1):
        sc = synthetic.make_pile(3000 + 2500 * (i % 3), n_objects=2 + i % 4, seed=40 + i)
        dt = np.float64 if i == 2 else np.float32
        out.append({"cloud_xyz": sc["cloud_xyz"].astype(dt), "cloud_normal": sc["cloud_normal"].astype(dt)})
    return out[:n]


def _same(a, b):
    if isinstance(a, torch.Tensor):
        assert a.is_cuda and b.is_cuda
        a, b = a.cpu().numpy(), b.cpu().numpy()
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def test_device_front_many_equals_the_frames(predictor):
    frames = _frames(5)
    xo, locs, feats, shapes, off = predictor.device_front_many(frames)
    assert len(shapes) == len(frames) and off[-1] == len(xo) == len(locs) == len(feats)
    for b, d in enumerate(frames):
        w = predictor.device_front(d)
        a, e = off[b], off[b + 1]
        assert _same(xo[a:e], w[0]) and _same(locs[a:e], w[1]) and _same(feats[a:e], w[2]), b
        assert shapes[b] == w[3], b


def test_pointgroup_labels_many_equals_the_frames():
    rng = np.random.RandomState(3)
    xos, offs, clouds = [], [], []
    for cls in ("hnm", "nut", "screw"):
        xos.append(SEG[f"{cls}_xyz_original_all"])
        offs.append(SEG[f"{cls}_pt_offsets"])
        clouds.append(SEG[f"{cls}_cloud_xyz"])
    xos.append(xos[1] + np.float32(0.25))
    offs.append(offs[1][::-1].copy())
    clouds.append(rng.uniform(-1, 1, (500, 3)))                  # far from its frame: the fallback query
    for bw in (0.005, 0.007):
        got = segment.pointgroup_labels_many(xos, offs, clouds, bw)
        for b in range(len(xos)):
            w = segment.pointgroup_labels(xos[b], offs[b], clouds[b], bw)
            assert _same(got[b][0], w[0]) and _same(got[b][1], w[1]), (bw, b)
    g = segment.pointgroup_labels_many([xos[1]], [offs[1]], [clouds[1]], 0.007)[0]
    assert _same(g[0], SEG["nut_labels_all"]) and _same(g[1], SEG["nut_xyz_shifted"])


@pytest.mark.parametrize("kind", ["numpy", "cuda"])
def test_predict_many_equals_the_loop(predictor, kind):
    frames = _frames(5)
    if kind == "cuda":
        frames = [{k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in d.items()} for d in frames]
    want = []
    for d in frames:
        want.append(predictor.predict(d))
    shifted = predictor.xyz_shifted
    predictor.xyz_shifted = None
    got = predictor.predict_many(frames)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert _same(g, w)
    assert _same(predictor.xyz_shifted, shifted)


@pytest.mark.parametrize("B", [1, 2, 8])
def test_predict_many_index_builds_do_not_grow_with_frames(predictor, monkeypatch, B):
    """Two builds in the front, one 2 mm, one snap and one mean-shift index, and one per nearest-label stage, each of
    the two stages with at most one more for the batch's far queries: at most 9 whatever B is."""
    frames = _frames(B)
    calls = []
    real = _lib.Context.call

    def counting(self, name, *args):
        calls.append(name)
        return real(self, name, *args)
    monkeypatch.setattr(_lib.Context, "call", counting)
    predictor.predict_many(frames)
    builds = [c for c in calls if c.startswith("cg_cloud_index_create")]
    assert 7 <= len(builds) <= 9, builds
    assert all(c == "cg_cloud_index_create_many" for c in builds)
