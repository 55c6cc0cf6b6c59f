"""GPU tests (-m gpu) of the several-frame pick: CloudIndex.normals_many and estimate_normals_many against the
one-set normals set by set, segment_table_many against segment_table frame by frame and against oracle.pick_ref,
both new entries under the poisoned-memory protocol, and compute_candidate_grasp_many against a loop of
compute_candidate_grasp from the same numpy state, every yield and every generator state bit for bit."""
import copy
import hashlib

import numpy as np
import pytest
import torch

from catgrasp_b200 import _lib, cloud, pick, synthetic
from oracle import pick_ref
from test_cloud_index_many import _blob, _pile, _top_cell_sets
from test_pick import CFG_RUN, K, N_CLASSES, _compare, _scene, predicters, straight_line  # noqa: F401
from test_poisoned_memory import _protocol, poison  # noqa: F401

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------ normals over several sets
def _bytes(t):
    return t.cpu().numpy().tobytes()


def check_normals_many(sets, radius, max_nn, cells=()):
    """normals_many on one index of the non-empty sets, at the largest of their query cells and at each of ``cells``,
    against normals on a one-set index of each set alone: normals, counts and neighbour lists, bit for bit."""
    off = np.cumsum([0] + [len(s) for s in sets])
    pts = np.concatenate(sets)
    shared = cloud._query_cell_many(pts, off, radius)
    for cell in (shared,) + tuple(cells):
        ix = cloud.CloudIndex(pts, cell, set_offsets=off)
        n, nbr, cnt = ix.normals_many(radius, max_nn, neighbours=True)
        for s, p in enumerate(sets):
            a, b = off[s], off[s + 1]
            one_n, one_nbr, one_cnt = cloud.CloudIndex(p, cloud._query_cell(p, radius)).normals(radius, max_nn,
                                                                                                  neighbours=True)
            assert _bytes(n[a:b]) == _bytes(one_n), (cell, s)
            assert _bytes(cnt[a:b]) == _bytes(one_cnt), (cell, s)
            got = nbr[a:b].cpu().numpy()
            assert (got[got >= 0] >= a).all() and (got[got >= 0] < b).all(), (cell, s)   # never another set's point
            assert np.array_equal(np.where(got >= 0, got - a, -1), one_nbr.cpu().numpy()), (cell, s)
    got = cloud.estimate_normals_many(pts, off, radius, max_nn)
    for s, p in enumerate(sets):
        assert got[off[s]:off[s + 1]].tobytes() == cloud.estimate_normals(p, radius, max_nn).tobytes(), s


def _faces(cell):
    """Two sets whose points coincide at cell faces: a lattice of pitch `cell`, and every other point of it plus a
    second lattice shifted by half a cell; neighbours at exactly the radius tie with d2 = r*r."""
    g = np.arange(6) * cell
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + [0.1, -0.05, 0.6]
    return [lat, np.concatenate([lat[::2], lat[1::3] + cell / 2])]


NORMAL_CASES = {
    "piles": ([_pile(3000, 5, 81, 0.6), _pile(2000, 4, 82, 0.6), _blob(1500, 3, spread=0.01)], 0.002, 30),
    "identical": ([_blob(2000, 5, spread=0.01)] * 2, 0.002, 30),
    "faces": (_faces(0.002), 0.002, 30),
    "top_cell": (_top_cell_sets(5, 0.25), 0.25, 30),
    "one_point": ([np.array([[0.3, 0.2, 0.5]]), _blob(800, 4, spread=0.01), np.array([[0.1, -0.05, 0.6]])], 0.003, 30),
    "max_nn_1": ([_blob(1000, 6, spread=0.01), _blob(900, 7, spread=0.01)], 0.002, 1),
    "max_nn_max": ([_blob(3000, 8, spread=0.005), _blob(2500, 9, spread=0.005)], 0.002, 64),
    # radius 0: the shared cell is the largest set's span / 2^20, so a set with extent takes 21 bits per axis and
    # fits only alone; coincident points keep the cell at its floor
    "radius_0": ([np.tile([[0.1, 0.2, 0.6]], (50, 1)), np.array([[0.3, 0.2, 0.5]]), np.tile([[0.1, 0.2, 0.6]], (31, 1))],
                 0.0, 30),
    "radius_0_one_set": ([_blob(500, 10, spread=0.01)], 0.0, 30),
}


@pytest.mark.parametrize("name", sorted(NORMAL_CASES))
def test_normals_many_equals_the_sets(name):
    sets, radius, max_nn = NORMAL_CASES[name]
    check_normals_many(sets, radius, max_nn, cells=() if radius == 0 else (radius, 3 * radius))


def test_normals_many_largest_batch_and_one_more():
    """8 sets of 600001 cells fill the 63-bit key (3 * 20 + 3 set bits); a ninth set is refused."""
    sets = [np.concatenate([np.array([[0.0, 0.0, 0.0], [600000.0, 3.0 * s, 1.0]]) + 7.0 * s,
                            _blob(40, s, centre=(7.0 * s, 7.0 * s, 7.0 * s), spread=0.5)]) for s in range(8)]
    check_normals_many(sets, 1.0, 30)
    pts = np.concatenate(sets + [sets[0]])
    with pytest.raises(_lib.CgError, match="63"):
        cloud.estimate_normals_many(pts, np.arange(0, 42 * 9 + 1, 42), 1.0, 30)


def test_estimate_normals_many_empty_sets_and_cuda_input():
    sets = [np.zeros((0, 3)), _blob(700, 11, spread=0.01), np.zeros((0, 3)), _blob(300, 12, spread=0.01),
            np.zeros((0, 3))]
    off = np.cumsum([0] + [len(s) for s in sets])
    pts = torch.from_numpy(np.concatenate(sets)).float().cuda()
    got = cloud.estimate_normals_many(pts, off, 0.002, 30)
    assert got.is_cuda and got.shape == (1000, 3)
    for s in (1, 3):
        assert _bytes(got[off[s]:off[s + 1]]) == _bytes(cloud.estimate_normals(pts[off[s]:off[s + 1]], 0.002, 30))
    assert cloud.estimate_normals_many(np.zeros((0, 3)), [0, 0, 0], 0.002, 30).shape == (0, 3)


# ------------------------------------------------------------------------------------------ segment table of frames
def _frame(M, L, seed, ltype=np.int64, xtype=np.float32, ties=False, outside=False):
    rng = np.random.RandomState(seed)
    if ties:
        labels = np.repeat(np.arange(L), M // L)[rng.permutation(M // L * L)]
    else:
        w = rng.uniform(0.2, 3, L)
        labels = rng.choice(L, M, p=w / w.sum())
        labels[:min(L, M)] = np.arange(min(L, M))
    if outside and M:
        labels[rng.choice(len(labels), max(1, M // 50), replace=False)] = rng.choice([-1, -7, L, L + 3], max(1, M // 50))
    n = len(labels)
    centre = rng.uniform(-0.1, 0.1, (L, 3))[np.clip(labels, 0, L - 1)]
    size = rng.uniform(0.001, 0.2, (L, 3))[np.clip(labels, 0, L - 1)]
    return labels.astype(ltype), (centre + size * rng.uniform(-0.5, 0.5, (n, 3))).astype(xtype), L


def _table_many(frames):
    labels = torch.from_numpy(np.concatenate([f[0] for f in frames])).cuda()
    xyz = torch.from_numpy(np.concatenate([f[1] for f in frames])).cuda()
    off = np.cumsum([0] + [len(f[0]) for f in frames])
    return pick.segment_table_many(labels, xyz, off, [f[2] for f in frames])


def check_table_many(frames):
    got = {k: v.cpu().numpy() for k, v in _table_many(frames).items()}
    po, lo = 0, 0
    for b, (labels, xyz, L) in enumerate(frames):
        M = len(labels)
        one = pick.segment_table(torch.from_numpy(labels).cuda(), torch.from_numpy(xyz).cuda(), L)
        one = {k: v.cpu().numpy() for k, v in one.items()}
        blocks = {"labels": (po, po + M), "index": (po, po + M), "count": (lo, lo + L), "min": (lo, lo + L),
                  "max": (lo, lo + L), "inlier": (lo, lo + L), "order": (lo, lo + L), "n_kept": (b, b + 1),
                  "offsets": (lo + b, lo + b + L + 1)}
        for k, (a, e) in blocks.items():
            assert got[k][a:e].dtype == one[k].dtype and got[k][a:e].tobytes() == one[k].tobytes(), (b, k)
        if M and labels.min() >= 0:                    # pick_ref sizes the table from the labels themselves
            ref = pick_ref.segment_table(labels, xyz)
            n = int(one["n_kept"][0])
            assert one["order"][:n].tolist() == ref["order"] and (one["order"][n:] == -1).all()
            assert np.array_equal(one["labels"], ref["labels"])
            for k, idx in enumerate(ref["indices"]):
                assert np.array_equal(one["index"][one["offsets"][k]:one["offsets"][k + 1]], idx)
        po, lo = po + M, lo + L
    assert po == len(got["labels"]) and lo + len(frames) == len(got["offsets"])


TABLE_CASES = {
    "small_tables": [_frame(5000, 7, 1), _frame(0, 3, 2), _frame(1, 1, 3), _frame(3000, 1, 4), _frame(8000, 20, 5)],
    "wide_tables": [_frame(200_000, 300, 6), _frame(50_000, 600, 7), _frame(0, 1, 8), _frame(30_000, 2, 9)],
    "ties": [_frame(64 * 600, 64, 10, ties=True), _frame(20 * 700, 20, 11, ties=True)],
    "outside": [_frame(20_000, 10, 12, outside=True), _frame(10_000, 5, 13, outside=True), _frame(0, 2, 14)],
    "int32_float64": [_frame(9000, 9, 15, np.int32, np.float64), _frame(0, 4, 16, np.int32, np.float64),
                      _frame(40_000, 513, 17, np.int32, np.float64)],
    "int64_float64": [_frame(9000, 9, 18, np.int64, np.float64), _frame(12_000, 30, 19, np.int64, np.float64)],
    "int32_float32": [_frame(9000, 9, 20, np.int32), _frame(700, 1, 21, np.int32)],
}


@pytest.mark.parametrize("name", sorted(TABLE_CASES))
def test_segment_table_many_equals_the_frames(name):
    check_table_many(TABLE_CASES[name])


def test_segment_table_many_one_frame_is_segment_table():
    check_table_many([_frame(20_000, 12, 22)])


# ------------------------------------------------------------------------------------------ poisoned memory
def test_poisoned_normals_many(poison):
    sets = [np.array([[0.3, 0.2, 0.5]]), _pile(2000, 4, 82, 0.6), _blob(600, 3, spread=0.01)]
    off = np.cumsum([0] + [len(s) for s in sets])
    pts = np.concatenate(sets)

    def run():
        return list(cloud.CloudIndex(pts, 0.002, set_offsets=off).normals_many(0.002, 30, neighbours=True))

    def check(A):
        check_normals_many(sets, 0.002, 30)
        one = [cloud.CloudIndex(s, 0.002).normals(0.002, 30, neighbours=True) for s in sets]
        assert A[0].tobytes() == np.concatenate([o[0].cpu().numpy() for o in one]).tobytes()
    _protocol(poison, run, check)


def test_poisoned_segment_table_many(poison):
    frames = [_frame(5000, 7, 23), _frame(0, 2, 24), _frame(30_000, 600, 25, outside=True), _frame(4000, 1, 26)]

    def run():
        return _table_many(frames)
    _protocol(poison, run, lambda A: check_table_many(frames))


# ------------------------------------------------------------------------------------------ the pick over frames
class ContentSegmenter:
    """A segmenter stand-in: fixed labels per frame, found by the frame's points (frames with the same points get the
    same labels)."""

    def __init__(self):
        self.by_key, self.calls = {}, 0

    @staticmethod
    def _key(xyz):
        x = xyz.cpu().numpy() if isinstance(xyz, torch.Tensor) else np.asarray(xyz)
        return hashlib.sha1(np.ascontiguousarray(x).tobytes()).hexdigest()

    def add(self, xyz, labels):
        self.by_key[self._key(xyz)] = labels

    def predict(self, data):
        self.calls += 1
        return self.by_key[self._key(data["cloud_xyz"])].copy()


class ContentSegmenterMany(ContentSegmenter):
    def predict_many(self, datas):
        self.many = getattr(self, "many", 0) + 1
        return [ContentSegmenter.predict(self, d) for d in datas]


def _pts_of(depth, Km, bg):
    xyz = cloud.depth2xyzmap(depth, Km)
    return xyz[bg == 0].reshape(-1, 3)


@pytest.fixture(scope="module")
def frames():
    """(name, depth, K, bg, env, labels) for every kind of frame the pick must handle."""
    sc, plain = _scene(True), _scene(False)
    out = [("shaped", sc["depth"], K, sc["bg"], sc["env"], sc["labels"]),
           ("plain", plain["depth"].astype(np.float64), K, plain["bg"], plain["env"], plain["labels"])]
    K2 = np.array([[5100.0, 0, 300.0], [0, 5102.0, 240.0], [0, 0, 1]])
    d2, ids2 = synthetic.render_depth(K2, 480, 600, n_objects=6, seed=41)
    out.append(("smaller", d2, K2, ids2 < 0, sc["env"], ids2[ids2 >= 0].astype(np.int64)))
    out.append(("background", sc["depth"], K, np.ones_like(sc["bg"]), sc["env"], np.zeros(0, np.int64)))
    shallow = np.where(sc["bg"], sc["depth"], np.float32(0.05))       # every object pixel below 0.1
    out.append(("shallow", shallow, K, sc["bg"], sc["env"], sc["labels"]))
    d3, ids3 = synthetic.render_depth(K2, 480, 600, n_objects=6, seed=42)   # 400-point segments: no inlier
    out.append(("no_inlier", d3, K2, ids3 < 0, sc["env"], np.arange(int((ids3 >= 0).sum()), dtype=np.int64) // 400))
    out.append(("shaped_again", sc["depth"], K, sc["bg"], sc["env"], sc["labels"]))
    return out, sc


def _segmenter(frames, many):
    seg = ContentSegmenterMany() if many else ContentSegmenter()
    for _, d, Km, bg, _, labels in frames:
        if (bg == 0).any():
            seg.add(_pts_of(d, Km, bg), labels)
    return seg


def _run(gen):
    out = []
    for r in gen:
        out.append((r, np.random.get_state()))
    return out


def _same_yields(got, want, where):
    assert len(got) == len(want), where
    for (r, st), (w, wst) in zip(got, want):
        assert r.keys() == w.keys(), where
        for k in r:
            if k == "data":
                assert r[k].keys() == w[k].keys()
                for kk in r[k]:
                    assert np.asarray(r[k][kk]).tobytes() == np.asarray(w[k][kk]).tobytes(), (where, k, kk)
            else:
                a, b = r[k], w[k]
                a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
                b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (where, k)
        assert np.array_equal(st[1], wst[1]) and st[2] == wst[2], where


def _args(fr):
    return [f[1] for f in fr], [f[2] for f in fr], [f[3] for f in fr], [f[4] for f in fr]


def _loop(fr, seg, npd, gp, sc, order):
    res = {}
    for b in order:
        _, d, Km, bg, env, _ = fr[b]
        res[b] = _run(pick.compute_candidate_grasp(d, Km, bg, seg, npd, gp, sc["gripper"], env, sc["canonical"],
                                                   [np.eye(4)], CFG_RUN, n_classes=N_CLASSES))
    return res, np.random.get_state()


def _many(fr, seg, npd, gp, sc, order, starts=None):
    gens = pick.compute_candidate_grasp_many(*_args(fr), seg, npd, gp, sc["gripper"], sc["canonical"], [np.eye(4)],
                                             CFG_RUN, n_classes=N_CLASSES)
    res = {}
    for b in order:
        if starts is not None:
            starts[b] = copy.deepcopy(np.random.get_state())
        res[b] = _run(gens[b])
    return res, np.random.get_state()


@pytest.mark.parametrize("many_segmenter", [False, True])
def test_pick_many_equals_the_loop(frames, predicters, many_segmenter):
    fr, sc = frames
    gp, npd = predicters
    orders = [list(range(len(fr)))] + ([list(range(len(fr)))[::-1]] if not many_segmenter else [])
    for order in orders:
        np.random.seed(11)
        want, want_end = _loop(fr, _segmenter(fr, False), npd, gp, sc, order)
        np.random.seed(11)
        seg = _segmenter(fr, many_segmenter)
        starts = {}
        got, got_end = _many(fr, seg, npd, gp, sc, order, starts)
        for b in order:
            _same_yields(got[b], want[b], (fr[b][0], order[0]))
        assert np.array_equal(got_end[1], want_end[1]) and got_end[2] == want_end[2]
        assert seg.calls == sum(1 for f in fr if (f[3] == 0).any())
        assert getattr(seg, "many", 1) == 1
        names = {fr[b][0]: len(got[b]) for b in order}
        assert names["background"] == names["no_inlier"] == 0, names
        assert sum(names.values()) >= 1, names   # which frames yield depends on numpy's state at their start
        if order[0] == 0 and not many_segmenter:
            for b in (0, 1, 2):       # each distinct frame with objects against test_pick's straight line
                np.random.set_state(starts[b])
                one = {"depth": fr[b][1], "bg": fr[b][3], "env": fr[b][4], "gripper": sc["gripper"],
                       "canonical": sc["canonical"]}
                want_b = []
                with _intrinsics(fr[b][2]):
                    for seg_id, branch, res in straight_line(one, _segmenter(fr, False), npd, gp):
                        if branch == "accepted":
                            want_b.append((seg_id, branch, res, np.random.get_state()))
                _compare(got[b], want_b)


class _intrinsics:
    """test_pick.straight_line reads the module's K: point it at a frame's own intrinsics for the block."""

    def __init__(self, Km):
        import test_pick
        self.mod, self.Km, self.old = test_pick, Km, test_pick.K

    def __enter__(self):
        self.mod.K = self.Km

    def __exit__(self, *exc):
        self.mod.K = self.old


def test_pick_many_shared_stage_errors_reach_every_generator(frames, predicters):
    fr, sc = frames
    gp, npd = predicters
    seg = _segmenter(fr, False)
    bad = fr[2][5].copy()
    bad[5] = -1
    seg.add(_pts_of(fr[2][1], fr[2][2], fr[2][3]), bad)
    gens = pick.compute_candidate_grasp_many(*_args(fr[:3]), seg, npd, gp, sc["gripper"], sc["canonical"],
                                             [np.eye(4)], CFG_RUN, n_classes=N_CLASSES)
    st = np.random.get_state()
    for g in gens[::-1]:
        with pytest.raises(ValueError, match="negative label"):
            next(g)
    assert seg.calls == 3                                   # the shared stages ran once
    assert np.array_equal(np.random.get_state()[1], st[1])  # and drew nothing


class _StopAtFirstObject(Exception):
    pass


@pytest.mark.parametrize("B", [1, 2, 8])
def test_pick_many_index_builds_do_not_grow_with_frames(frames, predicters, monkeypatch, B):
    """Up to the first object's stages: two index builds (normals and 1 mm scenes), one segment table, and one
    back-projection launch per frame."""
    fr, sc = frames
    gp, npd = predicters
    sel = [fr[1]] * B
    seg = _segmenter(sel, False)
    calls = []
    real = _lib.Context.call

    def counting(self, name, *args):
        calls.append(name)
        return real(self, name, *args)

    def stop(*a, **k):
        raise _StopAtFirstObject

    monkeypatch.setattr(_lib.Context, "call", counting)
    monkeypatch.setattr(cloud, "prepare_object", stop)
    gens = pick.compute_candidate_grasp_many(*_args(sel), seg, npd, gp, sc["gripper"], sc["canonical"], [np.eye(4)],
                                             CFG_RUN, n_classes=N_CLASSES)
    with pytest.raises(_StopAtFirstObject):
        next(gens[0])
    builds = [c for c in calls if c.startswith("cg_cloud_index_create")]
    assert builds == ["cg_cloud_index_create_many"] * 2, builds
    assert [c for c in calls if c.startswith("cg_segment_table")] == ["cg_segment_table_many_dev"]
    assert calls.count("cg_depth2xyz_dev") == B
