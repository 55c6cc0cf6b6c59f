"""GPU: GraspPredicter.predict_batch_many against a loop of predict_batch, and its device entries against the
per-object ones.

- Equivalence with the loop, bit for bit: every [label, conf, probs], numpy's generator afterwards and the
  predicter's engine, on engines 0-3, with host-drawn, device-drawn and given subsets.  Per-object candidate counts
  cover every FC kernel-selection edge (0, 1, 7, 8, 9, 63, 64, 65, 1023, 1024, 1025), objects with fewer points than
  n_pts are included, and one list holds more than CHUNK_B candidates in all.
- More than one launch's worth of few-row groups (150 objects of 1-8 candidates), and far fewer launches than the loop.
- The fp16 fallback: one object's cloud is scaled out of the fp16 range; only that object is scored again on
  engine 1, as in the loop; a flag left set before the call sends the first object to engine 1, as in the loop.
- cg_draw_ids_many_dev equals per-object cg_draw_ids_dev plus each object's base row, and the CPU restatement of
  the single-object draw (oracle.draw_ref.draw_ids) plus the base, object by object.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ENGINES = [int(e) for e in os.environ.get("CG_TEST_ENGINES", "0,1,2,3").split(",")]
N_PTS = 128
EDGES = (0, 1, 7, 8, 9, 63, 64, 65, 1023, 1024, 1025)


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need an H100; there is no CPU fallback")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def predicter(cuda, tmp_path_factory):
    from catgrasp_b200.predicter import GraspPredicter
    from catgrasp_b200.synthetic import write_artifacts
    adir = write_artifacts(str(tmp_path_factory.mktemp("many") / "artifacts-47"), "cls", n_pts=N_PTS, seed=0)
    return GraspPredicter("nut", artifact_dir=adir, engine=3)


@pytest.fixture(scope="module")
def pile():
    from catgrasp_b200.synthetic import make_pile
    scene = make_pile(16000, n_objects=16, seed=4)
    out = []
    for k in range(16):
        m = scene["object_id"] == k
        xyz, nrm = scene["cloud_xyz"][m].copy(), scene["cloud_normal"][m].copy()
        xyz[:2, 2] = 0.05                                        # masked out
        out.append({"cloud_xyz": xyz, "cloud_normal": nrm})
    out[3] = {k: v[:60] for k, v in out[3].items()}              # 58 valid points < n_pts: drawn with replacement
    out[5] = {k: v[:N_PTS + 2] for k, v in out[5].items()}       # exactly n_pts valid points
    return out


def _objects(pile, counts, seed=0):
    from catgrasp_b200.synthetic import make_candidates
    datas, grasps = [], []
    for o, B in enumerate(counts):
        d = pile[o % len(pile)]
        datas.append(d)
        grasps.append(list(make_candidates(d["cloud_xyz"][2:], d["cloud_normal"][2:], B, seed=seed + o))[:B]
                      if B else [])
    return datas, grasps


def _state():
    s = np.random.get_state()
    return s[0], s[1].copy(), s[2], s[3], s[4]


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _same_results(a, b):
    assert len(a) == len(b)
    for o, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), o
        for i, (u, v) in enumerate(zip(x, y)):
            assert type(u[0]) is type(v[0]) and u[0] == v[0], (o, i)
            assert u[1].dtype == v[1].dtype and u[1].tobytes() == v[1].tobytes(), (o, i)
            assert u[2].dtype == v[2].dtype and u[2].tobytes() == v[2].tobytes(), (o, i)


def _compare(gp, datas, grasps, mode, ids=None, capsys=None):
    engine = gp.engine
    np.random.seed(21)
    loop = [gp.predict_batch(d, g, ids=None if ids is None else ids[o], subsample=mode)
            for o, (d, g) in enumerate(zip(datas, grasps))]
    after = _state()
    printed = capsys.readouterr().out if capsys else None
    np.random.seed(21)
    many = gp.predict_batch_many(datas, grasps, ids=ids, subsample=mode)
    assert _same_state(after, _state())
    assert gp.engine == engine
    _same_results(loop, many)
    if capsys:
        assert capsys.readouterr().out == printed
    return loop, printed


def _given(datas, grasps, seed=3):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, int((d["cloud_xyz"][:, 2] >= 0.1).sum()), (len(g), N_PTS)).astype(np.int32)
            for d, g in zip(datas, grasps)]


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("mode", ["host", "device", "given"])
def test_many_equals_loop_at_every_kernel_edge(predicter, pile, engine, mode):
    gp = predicter
    counts = list(EDGES) + [5, 2, 0, 3, 64]                        # 16 objects: the edges, and M < n_pts / M == n_pts
    datas, grasps = _objects(pile, counts)
    keep = gp.engine
    gp.engine = engine
    try:
        ids = _given(datas, grasps) if mode == "given" else None
        _compare(gp, datas, grasps, "host" if mode == "given" else mode, ids=ids)
    finally:
        gp.engine = keep


@pytest.mark.parametrize("mode", ["host", "device", "given"])
def test_many_over_chunk_b_in_all(predicter, pile, mode):
    from catgrasp_b200.predicter import GRASPQ_CHUNK_B
    counts = [9000, 3, 8000, 1, 0, 700]
    assert sum(counts) > GRASPQ_CHUNK_B
    datas, grasps = _objects(pile, counts, seed=40)
    ids = _given(datas, grasps) if mode == "given" else None
    _compare(predicter, datas, grasps, "host" if mode == "given" else mode, ids=ids)


def test_many_small_objects_share_fc_launches(predicter, pile):
    gp = predicter
    counts = [1 + o % 8 for o in range(150)]                       # more few-row groups than one launch takes
    datas, grasps = _objects(pile, counts, seed=7)
    _compare(gp, datas, grasps, "device")
    ctx = gp.model.ctx
    ctx.reset_launch_count()
    np.random.seed(1)
    [gp.predict_batch(d, g, subsample="device") for d, g in zip(datas, grasps)]
    loop_launches = ctx.launch_count()
    ctx.reset_launch_count()
    np.random.seed(1)
    gp.predict_batch_many(datas, grasps, subsample="device")
    many_launches = ctx.launch_count()
    # the loop: per object a draw, three trunks, nine FC layers and a softmax; the batched call: one draw, three
    # trunks, two few-row launches per FC layer (150 groups, 128 per launch) and one softmax
    assert many_launches * 20 < loop_launches, (many_launches, loop_launches)


def _scaled(d, s):
    return {"cloud_xyz": d["cloud_xyz"] * s, "cloud_normal": d["cloud_normal"]}


@pytest.mark.parametrize("mode", ["host", "device"])
def test_fp16_fallback_redoes_only_the_overflowing_object(predicter, pile, mode, capsys):
    gp = predicter
    assert gp.engine == 3
    datas, grasps = _objects(pile, [4, 9, 70, 2], seed=11)
    datas[2] = _scaled(datas[2], 1e6)                              # its activations leave the fp16 range
    grasps[2] = [g * np.array([[1, 1, 1, 1e6]] * 3 + [[0, 0, 0, 1]]) for g in grasps[2]]
    capsys.readouterr()
    _, printed = _compare(gp, datas, grasps, mode, capsys=capsys)
    assert printed.count("re-running on engine 1") == 1
    # the same list without the scaled object never leaves the fp16 range
    _, printed = _compare(gp, datas[:2] + datas[3:], grasps[:2] + grasps[3:], mode, capsys=capsys)
    assert printed.count("re-running on engine 1") == 0


def test_fp16_flag_set_before_the_call(predicter, pile, capsys):
    """The flag belongs to the context: a clamp by earlier work that nobody read sends the loop's first call (and only
    it) to engine 1; the batched call does the same."""
    gp = predicter
    datas, grasps = _objects(pile, [0, 3, 5], seed=12)
    big = _scaled(pile[0], 1e6)
    bg = [g * np.array([[1, 1, 1, 1e6]] * 3 + [[0, 0, 0, 1]])
          for g in _objects([pile[0]], [2], seed=13)[1][0]]
    ctx = gp.model.ctx

    def clamp():   # engine-3 work that sets the flag and leaves it set
        ctx.set_engine(3)
        np.random.seed(0)
        gp.model.graspq_dev(*(torch.from_numpy(np.ascontiguousarray(a)).to(gp.model.device) for a in (
            big["cloud_xyz"][2:], big["cloud_normal"][2:], np.stack(bg),
            np.random.randint(0, len(big["cloud_xyz"]) - 2, (2, N_PTS)).astype(np.int32))))
    capsys.readouterr()
    clamp()
    np.random.seed(21)
    loop = [gp.predict_batch(d, g) for d, g in zip(datas, grasps)]
    after = _state()
    printed = capsys.readouterr().out
    assert printed.count("re-running on engine 1") == 1
    clamp()
    np.random.seed(21)
    many = gp.predict_batch_many(datas, grasps)
    assert _same_state(after, _state())
    assert capsys.readouterr().out == printed
    _same_results(loop, many)


def _draw_ids_many_ref(Ms, n_pts, counts, seeds, bases):
    """What cg_draw_ids_many_dev writes, from the CPU restatement of the single-object draw (oracle.draw_ref): object
    o's rows are draw_ids(Ms[o], n_pts, counts[o], seeds[o]) + bases[o], objects in order."""
    from oracle import draw_ref
    parts = [draw_ref.draw_ids(int(M), n_pts, int(c), int(s)) + np.int32(b)
             for M, c, s, b in zip(Ms, counts, seeds, bases) if c > 0]
    return np.concatenate(parts) if parts else np.empty((0, n_pts), np.int32)


def test_draw_ids_many_equals_per_object_draws(predicter):
    net = predicter.model
    Ms, counts = [900, 40, 128, 1, 5000, 77], [3, 1025, 0, 2, 64, 9]
    seeds = [7, 2 ** 40 + 1, 9, 2 ** 63 - 2, 123456789, 0]
    bases = np.concatenate([[0], np.cumsum(Ms)[:-1]])
    got = net.draw_ids_many_dev(Ms, N_PTS, counts, seeds, bases).cpu().numpy()
    first = np.concatenate([[0], np.cumsum(counts)])
    for o in range(len(Ms)):
        if counts[o]:
            one = net.draw_ids_dev(Ms[o], N_PTS, counts[o], seeds[o], first_candidate=0).cpu().numpy()
            assert np.array_equal(got[first[o]:first[o + 1]] - bases[o], one), o
    small = [0, 1, 2, 3, 5]
    args = ([Ms[o] for o in small], N_PTS, [counts[o] for o in small], [seeds[o] for o in small], bases[small])
    got_small = net.draw_ids_many_dev(*args).cpu().numpy()
    assert got_small.dtype == np.int32 and np.array_equal(got_small, _draw_ids_many_ref(*args))
